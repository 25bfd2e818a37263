// SpectralCF (SURVEY.md 8(f) rank 3): the spectral convolution layers forward and backward.
//
// Replaces (reference paths):
//   model/general_recommender/SpectralCF.py:63-83   _create_inference: E_k = act((A_hat E_{k-1}) W_k), concat over layers
//   model/general_recommender/SpectralCF.py:85-91   _create_loss (pairwise_loss on the concatenated rows + reg * l2_loss)
//   util/tool.py:10-33                              activation_function
// and TensorFlow's backward of the same graph (tf.matmul with a constant dense A_hat, tf.concat, embedding_lookup).
//
// A_hat = U U^T + U diag(lamda) U^T is a DENSE (users+items)^2 fp32 matrix built once on the host from
// np.linalg.eig of the normalised Laplacian, exactly as SpectralCF.__init__ does (:37-43,67-69); it is a constant
// of the graph.  Per step the work is 2K products A_hat[N,N] x [N,d] (K layers, forward + backward) plus thin
// [N,d] x [d,d] products -- fp32 GEMMs on the SIMT pipes (TF computes them in fp32; a tensor-core tf32/bf16
// product would change the trained tables beyond the parity tolerance), A_hat stays L2-resident (27 MB on ml-100k).
//
// One register-tiled kernel does every product:  Y[M, n] (+)= act( opA(A)[M, K] * opX(X)[K, n] ),  n <= 128,
// 32 rows x n columns per CTA, K consumed in chunks of 32 through shared memory, each thread 4 rows x n/32 columns.
// gridDim.y > 1 splits K over CTAs (the dW = S^T dZ reduction over all nodes) and adds with RED.
#include "common.cuh"
#include "graph.cuh"
#include "optim.cuh"

namespace nrc {

enum { ACT_IDENTITY = NRC_ACT_IDENTITY, ACT_SIGMOID = NRC_ACT_SIGMOID, ACT_TANH = NRC_ACT_TANH, ACT_RELU = NRC_ACT_RELU,
       ACT_ELU = NRC_ACT_ELU, ACT_SELU = NRC_ACT_SELU };
constexpr float kSeluScale = 1.0507009873554805f, kSeluAlpha = 1.6732632423543772f;

__device__ __forceinline__ float act_fwd(int act, float z) {
    switch (act) {
        case ACT_SIGMOID: return 1.0f / (1.0f + expf(-z));
        case ACT_TANH: return tanhf(z);
        case ACT_RELU: return fmaxf(z, 0.0f);
        case ACT_ELU: return z > 0.0f ? z : expf(z) - 1.0f;
        case ACT_SELU: return kSeluScale * (z > 0.0f ? z : kSeluAlpha * (expf(z) - 1.0f));
        default: return z;
    }
}

// d act / d z in terms of the output y
__device__ __forceinline__ float act_bwd(int act, float y) {
    switch (act) {
        case ACT_SIGMOID: return y * (1.0f - y);
        case ACT_TANH: return 1.0f - y * y;
        case ACT_RELU: return y > 0.0f ? 1.0f : 0.0f;
        case ACT_ELU: return y > 0.0f ? 1.0f : y + 1.0f;
        case ACT_SELU: return y > 0.0f ? kSeluScale : y + kSeluScale * kSeluAlpha;
        default: return 1.0f;
    }
}

struct GemmArgs {
    const float* A; int64_t lda; int trans_a;      // opA(A)[m, k] = trans_a ? A[k * lda + m] : A[m * lda + k]
    const float* X; int64_t ldx; int trans_x;      // opX(X)[k, c] = trans_x ? X[c * ldx + k] : X[k * ldx + c]
    float* Y; int64_t ldy;
    int M, K, n;
    int act;                                        // applied when the K range is not split
    int k_per_cta;                                  // split-K: K range per blockIdx.y (multiple of 32); Y += partials by RED
};

constexpr int kGemmRows = 32, kGemmK = 32, kGemmMaxN = 128;

// Thread (tx, ty): rows 4 ty .. 4 ty + 3 (one LDS.128 of the A tile, broadcast across the warp) x columns
// 4 tx .. 4 tx + 3 (one LDS.128 of the X tile, conflict-free): 16 FMAs per two vector shared-memory reads.
__global__ void __launch_bounds__(256) dense_gemm_kernel(const GemmArgs G) {
    __shared__ __align__(16) float As[kGemmK][kGemmRows + 4];        // [k][row]; row stride 36 floats keeps float4 alignment
    __shared__ __align__(16) float Xs[kGemmK][kGemmMaxN];            // [k][col]; columns >= n stay zero
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int row0 = blockIdx.x * kGemmRows;
    const int k_begin = blockIdx.y * G.k_per_cta;
    const int k_end = min(G.K, k_begin + G.k_per_cta);
    for (int e = threadIdx.x; e < kGemmK * kGemmMaxN; e += 256) (&Xs[0][0])[e] = 0.0f;
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.0f;
    __syncthreads();
    for (int k0 = k_begin; k0 < k_end; k0 += kGemmK) {
        // A tile: 32 rows x 32 k
        for (int e = threadIdx.x; e < kGemmRows * kGemmK; e += 256) {
            int r, kk;
            if (G.trans_a) { r = e & 31; kk = e >> 5; } else { kk = e & 31; r = e >> 5; }     // coalesced along the contiguous axis
            const int gr = row0 + r, gk = k0 + kk;
            float v = 0.0f;
            if (gr < G.M && gk < k_end) v = G.trans_a ? __ldg(G.A + (int64_t)gk * G.lda + gr) : __ldg(G.A + (int64_t)gr * G.lda + gk);
            As[kk][r] = v;
        }
        // X tile: 32 k x n
        for (int e = threadIdx.x; e < kGemmK * G.n; e += 256) {
            int kk, c;
            if (G.trans_x) { kk = e & 31; c = e >> 5; } else { c = e % G.n; kk = e / G.n; }
            const int gk = k0 + kk;
            float v = 0.0f;
            if (gk < k_end) v = G.trans_x ? __ldg(G.X + (int64_t)c * G.ldx + gk) : __ldg(G.X + (int64_t)gk * G.ldx + c);
            Xs[kk][c] = v;
        }
        __syncthreads();
        if (4 * tx < G.n) {
#pragma unroll 8
            for (int kk = 0; kk < kGemmK; ++kk) {
                const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
                const float4 x = *reinterpret_cast<const float4*>(&Xs[kk][tx * 4]);
                const float av[4] = {a.x, a.y, a.z, a.w}, xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(av[r], xv[c], acc[r][c]);
            }
        }
        __syncthreads();
    }
    const bool split = gridDim.y > 1;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int gr = row0 + ty * 4 + r;
        if (gr >= G.M) continue;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int gc = tx * 4 + c;
            if (gc >= G.n) continue;
            float* y = G.Y + (int64_t)gr * G.ldy + gc;
            if (split) atomicAdd(y, acc[r][c]);
            else *y = act_fwd(G.act, acc[r][c]);
        }
    }
}

// dZ[r, c] = (grad_all[r, off + c] + carry[r, c]) * act'(all_emb[r, off + c]); grad_all's block is zeroed for the next step
__global__ void __launch_bounds__(256)
spectral_act_bwd_kernel(float* __restrict__ grad_all, const float* __restrict__ carry, const float* __restrict__ all_emb,
                        int64_t N, int d, int dtot, int off, int act, float* __restrict__ dZ) {
    const int64_t total = N * d;
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / d;
        const int c = (int)(e - r * d);
        const int64_t a = r * dtot + off + c;
        const float g = grad_all[a] + (carry ? carry[e] : 0.0f);
        grad_all[a] = 0.0f;
        dZ[e] = g * act_bwd(act, all_emb[a]);
    }
}

// out[r, c] = grad_all[r, c] + carry[r, c] for the layer-0 block; grad_all's block zeroed
__global__ void __launch_bounds__(256)
spectral_e0_grad_kernel(float* __restrict__ grad_all, const float* __restrict__ carry, int64_t N, int d, int dtot,
                        float* __restrict__ out) {
    const int64_t total = N * d;
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / d;
        const int64_t a = r * dtot + (e - r * d);
        out[e] = grad_all[a] + (carry ? carry[e] : 0.0f);
        grad_all[a] = 0.0f;
    }
}

__global__ void __launch_bounds__(256)
copy_block_kernel(const float* __restrict__ src, int64_t N, int d, int dtot, float* __restrict__ dst) {
    const int64_t total = N * d;
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / d;
        dst[r * dtot + (e - r * d)] = src[e];
    }
}

// route: the g_graph_routes entry that records this product's K split (gridDim.y), or -1
static int gemm(const float* A, int64_t lda, int trans_a, const float* X, int64_t ldx, int trans_x, float* Y, int64_t ldy,
                int M, int K, int n, int act, int split_k, int route, cudaStream_t st) {
    NRC_REQUIRE(n > 0 && n <= kGemmMaxN, NRC_E_LIMIT, "embedding_size %d outside [1, %d]", n, kGemmMaxN);
    GemmArgs G{A, lda, trans_a, X, ldx, trans_x, Y, ldy, M, K, n, act, K};
    unsigned gy = 1;
    // few row tiles and a long reduction (A_hat products on small graphs): two K halves per row tile fill the SMs; the
    // sum of two partials onto zero is exact in either order, so the result stays deterministic
    if (split_k <= 1 && act == ACT_IDENTITY && K >= 1024 && (M + kGemmRows - 1) / kGemmRows < sm_count()) split_k = 2;
    if (split_k > 1) {
        int per = ((K + split_k - 1) / split_k + kGemmK - 1) / kGemmK * kGemmK;
        G.k_per_cta = per;
        gy = (unsigned)((K + per - 1) / per);
        NRC_CUDA_CHECK(cudaMemset2DAsync(Y, (size_t)ldy * sizeof(float), 0, (size_t)n * sizeof(float), (size_t)M, st));
    }
    if (route >= 0) g_graph_routes[route] = (int32_t)gy;
    dim3 grid((unsigned)((M + kGemmRows - 1) / kGemmRows), gy);
    dense_gemm_kernel<<<grid, 256, 0, st>>>(G);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

static unsigned ew_grid(int64_t n) {
    int64_t b = (n + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

static int spectral_forward(int N, int d, int K, const float* a_hat, const float* e0, const float* filters, int act,
                            float* all_emb, float* sides, cudaStream_t st) {
    const int dtot = d * (K + 1);
    copy_block_kernel<<<ew_grid((int64_t)N * d), 256, 0, st>>>(e0, N, d, dtot, all_emb);
    for (int k = 1; k <= K; ++k) {
        float* side = sides + (size_t)(k - 1) * N * d;
        // side = A_hat E_{k-1}   (E_{k-1} is the (k-1)-th column block of all_emb)
        int rc = gemm(a_hat, N, 0, all_emb + (size_t)(k - 1) * d, dtot, 0, side, d, N, N, d, ACT_IDENTITY, 1,
                      kRouteSpecFwdSplit, st);
        if (rc) return rc;
        // E_k = act(side W_k)
        rc = gemm(side, d, 0, filters + (size_t)(k - 1) * d * d, d, 0, all_emb + (size_t)k * d, dtot, N, d, d, act, 1, -1,
                  st);
        if (rc) return rc;
    }
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

static int act_id(int act) { return (act >= ACT_IDENTITY && act <= ACT_SELU) ? act : -1; }

}  // namespace nrc

using namespace nrc;

extern "C" int64_t nrc_spectralcf_work_floats(int32_t num_nodes, int32_t dim, int32_t num_layers) {
    // sides [K, N, d] + dZ [N, d] + dS [N, d] + carry [N, d]
    return (int64_t)num_nodes * dim * ((int64_t)num_layers + 3);
}

extern "C" int nrc_spectralcf_forward(int32_t num_nodes, int32_t dim, int32_t num_layers, const float* a_hat,
                                      const float* e0, const float* filters, int32_t activation, float* all_emb,
                                      float* work, void* stream) {
    NRC_REQUIRE(num_nodes > 0 && dim > 0 && num_layers >= 0 && num_layers <= 8, NRC_E_VALUE, "bad SpectralCF shape");
    // checked before the first launch: the layer-0 copy must not run for a width the products then reject
    NRC_REQUIRE(dim <= kGemmMaxN, NRC_E_LIMIT, "embedding_size %d outside [1, %d]", dim, kGemmMaxN);
    NRC_REQUIRE(act_id(activation) >= 0, NRC_E_NOTIMPL, "ERROR");                        // tool.py:32-33
    g_graph_routes[kRouteSpecFwdSplit] = 0;
    g_graph_routes[kRouteSpecBwdSplit] = g_graph_routes[kRouteSpecDwSplit] = -1;
    return spectral_forward(num_nodes, dim, num_layers, a_hat, e0, filters, activation, all_emb, work, as_stream(stream));
}

extern "C" int nrc_spectralcf_grad(int32_t num_users, int32_t num_items, int32_t dim, int32_t num_layers,
                                   const float* a_hat, const float* a_hat_t, const float* e0, const float* filters,
                                   int32_t activation, const int32_t* users, const int32_t* pos_items,
                                   const int32_t* neg_items, int64_t batch, int32_t loss_kind, float reg, float* all_emb,
                                   float* grad_all, int32_t* touched, float* grad_e0, float* grad_filters, float* work,
                                   float* loss, void* stream) {
    NRC_REQUIRE(num_users > 0 && num_items > 0 && dim > 0 && num_layers >= 0 && num_layers <= 8, NRC_E_VALUE, "bad SpectralCF shape");
    NRC_REQUIRE(dim <= kGemmMaxN, NRC_E_LIMIT, "embedding_size %d outside [1, %d]", dim, kGemmMaxN);
    NRC_REQUIRE(act_id(activation) >= 0, NRC_E_NOTIMPL, "ERROR");
    g_graph_routes[kRouteSpecFwdSplit] = g_graph_routes[kRouteSpecBwdSplit] = g_graph_routes[kRouteSpecDwSplit] = 0;
    cudaStream_t st = as_stream(stream);
    const int N = num_users + num_items, d = dim, K = num_layers, dtot = d * (K + 1);
    float* sides = work;
    float* dZ = work + (size_t)K * N * d;
    float* dS = dZ + (size_t)N * d;
    float* carry = dS + (size_t)N * d;
    int rc = spectral_forward(N, d, K, a_hat, e0, filters, activation, all_emb, sides, st);
    if (rc) return rc;
    // loss + gradient w.r.t. the concatenated rows: the MF pairwise kernel on a table of width d (K + 1)
    rc = nrc_mf_pairwise_grad(all_emb, all_emb + (size_t)num_users * dtot, dtot, users, pos_items, neg_items, batch, loss_kind,
                              reg, grad_all, grad_all + (size_t)num_users * dtot, touched, touched + num_users, 1, loss, stream);
    if (rc) return rc;
    const float* at = a_hat_t ? a_hat_t : a_hat;
    const int at_trans = a_hat_t ? 0 : 1;                   // no explicit transpose given: read A_hat transposed
    const unsigned eg = ew_grid((int64_t)N * d);
    bool have_carry = false;
    for (int k = K; k >= 1; --k) {
        spectral_act_bwd_kernel<<<eg, 256, 0, st>>>(grad_all, have_carry ? carry : nullptr, all_emb, N, d, dtot, k * d, activation, dZ);
        const float* side = sides + (size_t)(k - 1) * N * d;
        const float* W = filters + (size_t)(k - 1) * d * d;
        // dW_k = side^T dZ   (reduction over all N nodes: split over CTAs)
        rc = gemm(side, d, 1, dZ, d, 0, grad_filters + (size_t)(k - 1) * d * d, d, d, N, d, ACT_IDENTITY, 64,
                  kRouteSpecDwSplit, st);
        if (rc) return rc;
        // dS = dZ W_k^T
        rc = gemm(dZ, d, 0, W, d, 1, dS, d, N, d, d, ACT_IDENTITY, 1, -1, st);
        if (rc) return rc;
        // carry = A_hat^T dS
        rc = gemm(at, N, at_trans, dS, d, 0, carry, d, N, N, d, ACT_IDENTITY, 1, kRouteSpecBwdSplit, st);
        if (rc) return rc;
        have_carry = true;
    }
    spectral_e0_grad_kernel<<<eg, 256, 0, st>>>(grad_all, have_carry ? carry : nullptr, N, d, dtot, grad_e0);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}
