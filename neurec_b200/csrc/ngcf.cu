// NGCF: the dense part of the propagation layer around the CSR SpMM, forward and backward.
//
// Replaces (reference paths):
//   model/general_recommender/NGCF.py:160-202  _create_ngcf_embed: per layer
//        side = A_hat . ego                                  (SpMM, lightgcn.cu)
//        sum  = leaky_relu(side . W_gc + b_gc)
//        bi   = leaky_relu((ego * side) . W_bi + b_bi)
//        ego' = dropout(sum + bi, 1 - mess_dropout)          (ALWAYS on, also at evaluation: NGCF.py:193)
//        all += l2_normalize(ego', axis=1);  final = concat(all)
//   model/general_recommender/NGCF.py:94-110   loss: sum softplus(-(pos - neg)) + reg * l2_loss(u, i, j)
// Third-party arithmetic restated (tensorflow==1.12.3, not vendored): tf.nn.leaky_relu alpha 0.2,
// tf.nn.l2_normalize epsilon 1e-12 (x * rsqrt(max(sum x^2, eps))), tf.nn.dropout(x, keep) =
// x * floor(keep + U[0,1)) / keep.  The oracle is oracle/tf_math.py::ngcf_forward /
// ngcf_loss_and_grad (finite-difference pinned; parity unpinned at the TF boundary).
//
// Decomposition.  The layer widths are 16-64, so the two GEMMs per layer are [N, d] x [d, d]
// with d*d weights that live in shared memory; a warp owns a node row (lanes = output columns).
//   ngcf_layer_fwd_kernel   both GEMMs + leaky-relu + dropout + l2-normalise + write into the
//                           concatenated table, keeping z1, z2, ego', |ego'|^2 for the backward
//   ngcf_bpr_grad_kernel    warp per triplet over the concatenated rows, RED into dense G
//   ngcf_layer_bwd_kernel   per 32-row tile: normalise / dropout / leaky-relu backward -> dz1, dz2 in
//                           shared memory; dside = dz1 W_gc^T + (dz2 W_bi^T) * ego and
//                           dego = (dz2 W_bi^T) * side per row; dW = side^T dz1, (ego*side)^T dz2 as
//                           register-tiled outer products accumulated over all tiles of the CTA,
//                           one RED per weight entry and CTA at the end
//   the remaining A_hat^T . dside is nrc_spmm_csr with its fused bias (dego + A^T dside).
#include "common.cuh"
#include "graph.cuh"
#include "learner.cuh"
#include "philox.cuh"

namespace nrc {

constexpr int kNgcfMaxLayers = 4;
constexpr int kNgcfMaxDim = 64;
constexpr float kLeakyAlpha = 0.2f;
constexpr float kL2NormEps = 1e-12f;

struct NgcfDev {
    int n_nodes, n_layers, emb_dim, d_total;
    int din[kNgcfMaxLayers], dout[kNgcfMaxLayers];
    int w_off[kNgcfMaxLayers];        // packed weights: W_gc [din, dout], b_gc [dout], W_bi, b_bi per layer
    int e_off[kNgcfMaxLayers + 1];    // column offset of each block in the concatenated table
    int64_t m_off[kNgcfMaxLayers];    // offset of layer k's [N, dout] block in the caller's packed masks
    // Workspace blocks start on 16 bytes: side, dside and hd blocks are operands of the SpMM, whose float2 / float4
    // forms need aligned rows (N * width floats is not a multiple of 4 for an odd N and an odd width).
    int64_t a_off[kNgcfMaxLayers];    // offset of layer k's [N, dout] block in z1 / z2 / hd
    int64_t side_off[kNgcfMaxLayers]; // offset of layer k's [N, din] block in side / dside buffers
    int weights_size;
    int64_t act_floats, in_floats;
};

static int64_t round4(int64_t n) { return (n + 3) & ~(int64_t)3; }

static int ngcf_make(NgcfDev& S, const nrc_ngcf_shape* sh) {
    NRC_REQUIRE(sh != nullptr, NRC_E_VALUE, "shape is NULL");
    NRC_REQUIRE(sh->n_layers >= 1 && sh->n_layers <= kNgcfMaxLayers, NRC_E_LIMIT, "n_layers %d outside [1, %d]",
                sh->n_layers, kNgcfMaxLayers);
    NRC_REQUIRE(sh->emb_dim >= 1 && sh->emb_dim <= kNgcfMaxDim, NRC_E_LIMIT, "embedding_size %d outside [1, %d]",
                sh->emb_dim, kNgcfMaxDim);
    S.n_nodes = sh->num_users + sh->num_items;
    S.n_layers = sh->n_layers; S.emb_dim = sh->emb_dim;
    int in = sh->emb_dim, woff = 0, eoff = sh->emb_dim;
    int64_t moff = 0, aoff = 0, soff = 0;
    S.e_off[0] = 0;
    for (int k = 0; k < kNgcfMaxLayers; ++k) {
        if (k >= S.n_layers) {
            S.din[k] = S.dout[k] = S.w_off[k] = 0; S.e_off[k + 1] = eoff; S.m_off[k] = moff; S.a_off[k] = aoff;
            S.side_off[k] = soff;
            continue;
        }
        const int out = sh->layers[k];
        NRC_REQUIRE(out >= 1 && out <= kNgcfMaxDim, NRC_E_LIMIT, "layer width %d outside [1, %d]", out, kNgcfMaxDim);
        S.din[k] = in; S.dout[k] = out;
        S.w_off[k] = woff; woff += 2 * (in * out + out);
        S.e_off[k + 1] = eoff; eoff += out;
        S.m_off[k] = moff; moff += (int64_t)S.n_nodes * out;
        S.a_off[k] = aoff; aoff += round4((int64_t)S.n_nodes * out);
        S.side_off[k] = soff; soff += round4((int64_t)S.n_nodes * in);
        in = out;
    }
    S.weights_size = woff; S.d_total = eoff; S.act_floats = aoff; S.in_floats = soff;
    return NRC_OK;
}

__device__ __forceinline__ float leaky(float x) { return x > 0.0f ? x : x * kLeakyAlpha; }

struct NgcfLayerArgs {
    const float* ego; const float* side;      // [N, din]
    const float* W;                           // packed W_gc, b_gc, W_bi, b_bi of this layer
    const float* mask; float keep;            // [N, dout] 0/1 or NULL
    float* z1; float* z2; float* hd;          // [N, dout]
    float* sq;                                // [N]
    float* all_emb; int d_total, e_off;       // normalised output -> all_emb[:, e_off : e_off + dout]
    int n, din, dout;
};

__global__ void __launch_bounds__(256) ngcf_layer_fwd_kernel(const NgcfLayerArgs A) {
    extern __shared__ float sm[];
    const int din = A.din, dout = A.dout;
    float* sWgc = sm;                        // [din][dout]
    float* sWbi = sWgc + din * dout;
    float* sB = sWbi + din * dout;           // b_gc [dout], b_bi [dout]
    float* sRow = sB + 2 * dout;             // per warp: side [din], bi [din]
    const float* Wgc = A.W; const float* bgc = Wgc + din * dout; const float* Wbi = bgc + dout; const float* bbi = Wbi + din * dout;
    for (int e = threadIdx.x; e < din * dout; e += blockDim.x) { sWgc[e] = Wgc[e]; sWbi[e] = Wbi[e]; }
    for (int e = threadIdx.x; e < dout; e += blockDim.x) { sB[e] = bgc[e]; sB[dout + e] = bbi[e]; }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    float* s_side = sRow + warp * 2 * din;
    float* s_bi = s_side + din;
    for (int row = blockIdx.x * wpb + warp; row < A.n; row += gridDim.x * wpb) {
        for (int k = lane; k < din; k += kWarp) {
            const float sd = A.side[(size_t)row * din + k];
            s_side[k] = sd;
            s_bi[k] = A.ego[(size_t)row * din + k] * sd;
        }
        __syncwarp();
        float hv[2], sqp = 0.0f;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int j = lane + 32 * t;
            hv[t] = 0.0f;
            if (j < dout) {
                float a1 = 0.0f, a2 = 0.0f;
                for (int k = 0; k < din; ++k) {
                    a1 = fmaf(s_side[k], sWgc[k * dout + j], a1);
                    a2 = fmaf(s_bi[k], sWbi[k * dout + j], a2);
                }
                a1 += sB[j]; a2 += sB[dout + j];
                const size_t o = (size_t)row * dout + j;
                A.z1[o] = a1; A.z2[o] = a2;
                float h = leaky(a1) + leaky(a2);
                if (A.mask) h = h * A.mask[o] / A.keep;          // tf.nn.dropout: x * mask / keep
                A.hd[o] = h;
                hv[t] = h;
                sqp += h * h;
            }
        }
        const float sq = warp_sum(sqp);
        const float inv = rsqrtf(fmaxf(sq, kL2NormEps));        // tf.nn.l2_normalize
        if (lane == 0) A.sq[row] = sq;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int j = lane + 32 * t;
            if (j < dout) A.all_emb[(size_t)row * A.d_total + A.e_off + j] = hv[t] * inv;
        }
        __syncwarp();
    }
}

// all_emb[:, 0:emb_dim] = e0
__global__ void ngcf_copy_e0_kernel(const float* __restrict__ e0, float* __restrict__ all_emb, int64_t n, int d, int d_total) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n * d; e += (int64_t)gridDim.x * blockDim.x)
        all_emb[(e / d) * d_total + (e % d)] = e0[e];
}

// BPR-softplus loss and its gradient on the concatenated embeddings (NGCF.py:94-110)
__global__ void __launch_bounds__(256)
ngcf_bpr_grad_kernel(const float* __restrict__ E, int D, int num_users, const int32_t* __restrict__ users,
                     const int32_t* __restrict__ pos, const int32_t* __restrict__ neg, int64_t batch, float reg,
                     float* __restrict__ G, float* __restrict__ loss2) {
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    float mf_acc = 0.0f, emb_acc = 0.0f;
    for (int64_t b = (int64_t)blockIdx.x * wpb + wib; b < batch; b += (int64_t)gridDim.x * wpb) {
        const size_t ru = (size_t)users[b] * D, ri = (size_t)(num_users + pos[b]) * D, rj = (size_t)(num_users + neg[b]) * D;
        float di = 0.f, dj = 0.f, sq = 0.f;
        for (int k = lane; k < D; k += kWarp) {
            const float a = E[ru + k], bi = E[ri + k], bj = E[rj + k];
            di = fmaf(a, bi, di); dj = fmaf(a, bj, dj);
            sq += a * a + bi * bi + bj * bj;
        }
        di = warp_sum(di); dj = warp_sum(dj); sq = warp_sum(sq);
        const float x = di - dj;
        mf_acc += neg_log_sigmoid(x);     // softplus(-x)
        emb_acc += reg * 0.5f * sq;
        const float g = neg_log_sigmoid_grad(x);
        for (int k = lane; k < D; k += kWarp) {
            const float a = E[ru + k], bi = E[ri + k], bj = E[rj + k];
            atomicAdd(G + ru + k, g * (bi - bj) + reg * a);
            atomicAdd(G + ri + k, g * a + reg * bi);
            atomicAdd(G + rj + k, -g * a + reg * bj);
        }
    }
    if (lane == 0 && loss2) { atomicAdd(loss2, mf_acc); atomicAdd(loss2 + 1, emb_acc); }
}

struct NgcfBwdArgs {
    const float* G; int d_total, e_off;       // gradient w.r.t. the concatenated table
    const float* d_next;                      // [N, dout] gradient flowing into this layer's raw output from layer k+1, or NULL
    const float* ego; const float* side;      // [N, din]
    const float* W;
    const float* mask; float keep;
    const float* z1; const float* z2; const float* hd; const float* sq;
    float* dside; float* dego;                // [N, din]: dego = (dz2 W_bi^T) * side (A^T dside is added by the SpMM)
    float* gW;                                // packed like W: accumulated with RED
    int n, din, dout;
};

constexpr int kBwdRows = 32;

__global__ void __launch_bounds__(256) ngcf_layer_bwd_kernel(const NgcfBwdArgs A) {
    extern __shared__ float sm[];
    const int din = A.din, dout = A.dout, dp = dout + 1;
    float* sWgc = sm;                          // [din][dout + 1] (conflict-free when lanes walk k)
    float* sWbi = sWgc + din * dp;
    float* s_side = sWbi + din * dp;           // [R][din]
    float* s_bi = s_side + kBwdRows * din;
    float* s_dz1 = s_bi + kBwdRows * din;      // [R][dout]
    float* s_dz2 = s_dz1 + kBwdRows * dout;
    const float* Wgc = A.W; const float* Wbi = Wgc + din * dout + dout;
    for (int e = threadIdx.x; e < din * dout; e += blockDim.x) {
        sWgc[(e / dout) * dp + (e % dout)] = Wgc[e];
        sWbi[(e / dout) * dp + (e % dout)] = Wbi[e];
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int kAcc = (kNgcfMaxDim * kNgcfMaxDim + 255) / 256;     // weight entries per thread and matrix
    float acc1[kAcc], acc2[kAcc], accb1 = 0.0f, accb2 = 0.0f;
#pragma unroll
    for (int i = 0; i < kAcc; ++i) acc1[i] = acc2[i] = 0.0f;
    __syncthreads();
    const int tiles = (A.n + kBwdRows - 1) / kBwdRows;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int row0 = tile * kBwdRows;
        // (i) element-wise backward of normalise / dropout / leaky-relu: dz1, dz2 of the tile's rows
        for (int r = warp; r < kBwdRows; r += 8) {
            const int row = row0 + r;
            const bool live_row = row < A.n;
            float gn[2] = {0.f, 0.f}, hdv[2] = {0.f, 0.f}, dotp = 0.0f;
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const int j = lane + 32 * t;
                if (live_row && j < dout) {
                    gn[t] = A.G[(size_t)row * A.d_total + A.e_off + j];
                    hdv[t] = A.hd[(size_t)row * dout + j];
                    dotp += gn[t] * hdv[t];
                }
            }
            const float dot = warp_sum(dotp);
            const float sq = live_row ? A.sq[row] : 1.0f;
            const float inv = rsqrtf(fmaxf(sq, kL2NormEps));
            const float lv = (sq > kL2NormEps) ? 1.0f : 0.0f;
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const int j = lane + 32 * t;
                if (j < dout) {
                    float d1 = 0.0f, d2 = 0.0f;
                    if (live_row) {
                        const size_t o = (size_t)row * dout + j;
                        float dhd = gn[t] * inv - lv * hdv[t] * dot * inv * inv * inv;
                        if (A.d_next) dhd += A.d_next[o];
                        const float dh = A.mask ? dhd * A.mask[o] / A.keep : dhd;
                        d1 = dh * (A.z1[o] > 0.0f ? 1.0f : kLeakyAlpha);
                        d2 = dh * (A.z2[o] > 0.0f ? 1.0f : kLeakyAlpha);
                    }
                    s_dz1[r * dout + j] = d1; s_dz2[r * dout + j] = d2;
                }
            }
            for (int k = lane; k < din; k += kWarp) {
                const float sd = live_row ? A.side[(size_t)row * din + k] : 0.0f;
                const float eg = live_row ? A.ego[(size_t)row * din + k] : 0.0f;
                s_side[r * din + k] = sd; s_bi[r * din + k] = eg * sd;
            }
            __syncwarp();
            // dside = dz1 W_gc^T + (dz2 W_bi^T) * ego ; dego = (dz2 W_bi^T) * side
            if (live_row) {
                for (int k = lane; k < din; k += kWarp) {
                    float a = 0.0f, b = 0.0f;
                    for (int j = 0; j < dout; ++j) {
                        a = fmaf(s_dz1[r * dout + j], sWgc[k * dp + j], a);
                        b = fmaf(s_dz2[r * dout + j], sWbi[k * dp + j], b);
                    }
                    const float sd = s_side[r * din + k];
                    const float eg = A.ego[(size_t)row * din + k];
                    A.dside[(size_t)row * din + k] = a + b * eg;
                    A.dego[(size_t)row * din + k] = b * sd;
                }
            }
        }
        __syncthreads();
        // (ii) weight gradients of the tile: dW_gc += side^T dz1, dW_bi += bi^T dz2, db += colsum(dz)
#pragma unroll
        for (int i = 0; i < kAcc; ++i) {
            const int e = threadIdx.x + 256 * i;
            if (e < din * dout) {
                const int k = e / dout, j = e - k * dout;
                float a = acc1[i], b = acc2[i];
#pragma unroll 8
                for (int r = 0; r < kBwdRows; ++r) {
                    a = fmaf(s_side[r * din + k], s_dz1[r * dout + j], a);
                    b = fmaf(s_bi[r * din + k], s_dz2[r * dout + j], b);
                }
                acc1[i] = a; acc2[i] = b;
            }
        }
        if ((int)threadIdx.x < dout) {
            for (int r = 0; r < kBwdRows; ++r) { accb1 += s_dz1[r * dout + threadIdx.x]; accb2 += s_dz2[r * dout + threadIdx.x]; }
        }
        __syncthreads();
    }
    float* gWgc = A.gW; float* gbgc = gWgc + din * dout; float* gWbi = gbgc + dout; float* gbbi = gWbi + din * dout;
#pragma unroll
    for (int i = 0; i < kAcc; ++i) {
        const int e = threadIdx.x + 256 * i;
        if (e < din * dout) { atomicAdd(gWgc + e, acc1[i]); atomicAdd(gWbi + e, acc2[i]); }
    }
    if ((int)threadIdx.x < dout) { atomicAdd(gbgc + threadIdx.x, accb1); atomicAdd(gbbi + threadIdx.x, accb2); }
}

// tf.nn.dropout's keep mask: floor(keep + U[0,1)); U from Philox4x32-10 keyed by (seed, stream), one
// 32-bit word per element (4 elements per counter).
__global__ void dropout_mask_kernel(int64_t n, float keep, uint64_t seed, uint64_t stream_id, float* __restrict__ out) {
    for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q * 4 < n; q += (int64_t)gridDim.x * blockDim.x) {
        const Philox4 r = philox4x32_10((uint32_t)q, (uint32_t)(q >> 32), 0x44524F50u /* 'DROP' */, (uint32_t)stream_id,
                                        (uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(stream_id >> 32));
        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int t = 0; t < 4; ++t)
            if (q * 4 + t < n) out[q * 4 + t] = ((float)(w[t] >> 8) * (1.0f / 16777216.0f) < keep) ? 1.0f : 0.0f;
    }
}

// dE0 = G[:, 0:emb_dim] + d_ego of layer 0
__global__ void ngcf_finish_e0_kernel(const float* __restrict__ G, const float* __restrict__ d0, float* __restrict__ out,
                                      int64_t n, int d, int dt) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n * d; e += (int64_t)gridDim.x * blockDim.x)
        out[e] = G[(e / d) * dt + (e % d)] + d0[e];
}

static int grid_for(int64_t work_items, int per_block) {
    int64_t blocks = (work_items + per_block - 1) / per_block;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    return blocks < 1 ? 1 : (int)blocks;
}

static int32_t per_worker(int64_t work_items, int64_t workers) {
    return (int32_t)((work_items + workers - 1) / workers);
}

}  // namespace nrc

using namespace nrc;

extern "C" int nrc_ngcf_weights_size(const nrc_ngcf_shape* shape) {
    NgcfDev S;
    if (ngcf_make(S, shape)) return NRC_E_VALUE;
    return S.weights_size;
}

extern "C" int64_t nrc_ngcf_work_floats(const nrc_ngcf_shape* shape) {
    NgcfDev S;
    if (ngcf_make(S, shape)) return NRC_E_VALUE;
    // side + dside (in_floats each), z1 + z2 + hd (act_floats each), d_next ping-pong x2 and dego
    // ([N, 64] each), sq [layers * N]
    return 2 * S.in_floats + 3 * S.act_floats + (int64_t)S.n_nodes * kNgcfMaxDim * 3 + (int64_t)S.n_layers * S.n_nodes + 1024;
}

extern "C" int nrc_dropout_mask(int64_t n, float keep, uint64_t seed, uint64_t stream_id, float* out, void* stream) {
    NRC_REQUIRE(n >= 0 && keep > 0.0f && keep <= 1.0f, NRC_E_VALUE, "n >= 0 and keep in (0, 1] required");
    if (n == 0) return NRC_OK;
    dropout_mask_kernel<<<grid_for((n + 3) / 4, 256), 256, 0, as_stream(stream)>>>(n, keep, seed, stream_id, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

namespace {
struct Work {
    float *side, *dside, *z1, *z2, *hd, *dnA, *dnB, *dego, *sq;
};
Work carve(const NgcfDev& S, float* w) {
    Work W;
    W.side = w; w += S.in_floats;
    W.dside = w; w += S.in_floats;
    W.z1 = w; w += S.act_floats;
    W.z2 = w; w += S.act_floats;
    W.hd = w; w += S.act_floats;
    W.dnA = w; w += (int64_t)S.n_nodes * kNgcfMaxDim;
    W.dnB = w; w += (int64_t)S.n_nodes * kNgcfMaxDim;
    W.dego = w; w += (int64_t)S.n_nodes * kNgcfMaxDim;
    W.sq = w;
    return W;
}

int forward_impl(const NgcfDev& S, const int64_t* indptr, const int32_t* indices, const float* values,
                 const int32_t* row_order, const float* e0, const float* weights, const float* masks, float keep,
                 float* all_emb, const Work& W, cudaStream_t st) {
    const int N = S.n_nodes;
    g_graph_routes[kRouteNgcfFwdRows] = per_worker(N, (int64_t)grid_for(N, 8) * 8);
    g_graph_routes[kRouteNgcfBwdTiles] = g_graph_routes[kRouteNgcfBprTriplets] = -1;
    ngcf_copy_e0_kernel<<<grid_for((int64_t)N * S.emb_dim, 256), 256, 0, st>>>(e0, all_emb, N, S.emb_dim, S.d_total);
    NRC_CUDA_CHECK(cudaGetLastError());
    const float* ego = e0;
    for (int k = 0; k < S.n_layers; ++k) {
        float* side = W.side + S.side_off[k];
        int rc = nrc_spmm_csr(indptr, indices, values, row_order, N, ego, S.din[k], nullptr, side, nullptr, 0.0f, st);
        if (rc) return rc;
        NgcfLayerArgs A{ego, side, weights + S.w_off[k], masks ? masks + S.m_off[k] : nullptr, keep,
                        W.z1 + S.a_off[k], W.z2 + S.a_off[k], W.hd + S.a_off[k], W.sq + (int64_t)k * N,
                        all_emb, S.d_total, S.e_off[k + 1], N, S.din[k], S.dout[k]};
        const size_t smem = ((size_t)2 * S.din[k] * S.dout[k] + 2 * S.dout[k] + 8 * 2 * S.din[k]) * 4;
        ngcf_layer_fwd_kernel<<<grid_for(N, 8), 256, smem, st>>>(A);
        NRC_CUDA_CHECK(cudaGetLastError());
        ego = W.hd + S.a_off[k];
    }
    return NRC_OK;
}
}  // namespace

// _create_ngcf_embed, NGCF.py:160-202: all_emb f32 [N, emb_dim + sum(layers)] (users first).
extern "C" int nrc_ngcf_forward(const nrc_ngcf_shape* shape, const int64_t* indptr, const int32_t* indices,
                                const float* values, const int32_t* row_order, const float* e0, const float* weights,
                                const float* masks, float keep, float* all_emb, float* work, void* stream) {
    NgcfDev S;
    int rc = ngcf_make(S, shape);
    if (rc) return rc;
    NRC_REQUIRE(masks == nullptr || (keep > 0.0f && keep <= 1.0f), NRC_E_VALUE, "keep must be in (0, 1]");
    return forward_impl(S, indptr, indices, values, row_order, e0, weights, masks, keep, all_emb, carve(S, work),
                        as_stream(stream));
}

// One `sess.run((loss, optimizer))` of NGCF.train_model (NGCF.py:125-135) up to the gradients: forward
// with the given dropout masks, BPR-softplus loss on the batch, backward through every layer.
//   t_*        CSR of A_hat^T ('norm' = D^-1 (A + I) is NOT symmetric); NULL -> A_hat itself
//   grad_all   f32 [N, d_total], zero on entry, zero on return
//   grad_e0    f32 [N, emb_dim] out; grad_weights f32 [weights_size] out (both overwritten)
//   loss2      f32 [2] += {mf_loss, emb_loss}
extern "C" int nrc_ngcf_grad(const nrc_ngcf_shape* shape, const int64_t* indptr, const int32_t* indices,
                             const float* values, const int32_t* row_order, const int64_t* t_indptr,
                             const int32_t* t_indices, const float* t_values, const int32_t* t_row_order,
                             const float* e0, const float* weights, const float* masks, float keep,
                             const int32_t* users, const int32_t* pos_items, const int32_t* neg_items, int64_t batch,
                             float reg, float* all_emb, float* grad_all, float* grad_e0, float* grad_weights,
                             float* work, float* loss2, void* stream) {
    NgcfDev S;
    int rc = ngcf_make(S, shape);
    if (rc) return rc;
    NRC_REQUIRE(batch >= 0, NRC_E_VALUE, "batch must be >= 0");
    cudaStream_t st = as_stream(stream);
    const Work W = carve(S, work);
    const int N = S.n_nodes;
    rc = forward_impl(S, indptr, indices, values, row_order, e0, weights, masks, keep, all_emb, W, st);
    if (rc) return rc;
    if (!t_indptr) { t_indptr = indptr; t_indices = indices; t_values = values; t_row_order = row_order; }
    NRC_CUDA_CHECK(cudaMemsetAsync(grad_weights, 0, (size_t)S.weights_size * sizeof(float), st));
    const int tiles = (N + kBwdRows - 1) / kBwdRows;
    const int bwd_grid = tiles < sm_count() * 2 ? tiles : sm_count() * 2;
    g_graph_routes[kRouteNgcfBprTriplets] = batch > 0 ? per_worker(batch, (int64_t)grid_for(batch, 8) * 8) : 0;
    g_graph_routes[kRouteNgcfBwdTiles] = per_worker(tiles, bwd_grid);
    if (batch > 0) {
        ngcf_bpr_grad_kernel<<<grid_for(batch, 8), 256, 0, st>>>(all_emb, S.d_total, shape->num_users, users, pos_items,
                                                                neg_items, batch, reg, grad_all, loss2);
        NRC_CUDA_CHECK(cudaGetLastError());
    }
    const float* d_next = nullptr;
    float* pp[2] = {W.dnA, W.dnB};
    for (int k = S.n_layers - 1; k >= 0; --k) {
        const float* ego = (k == 0) ? e0 : W.hd + S.a_off[k - 1];
        NgcfBwdArgs A{grad_all, S.d_total, S.e_off[k + 1], d_next, ego, W.side + S.side_off[k], weights + S.w_off[k],
                      masks ? masks + S.m_off[k] : nullptr, keep, W.z1 + S.a_off[k], W.z2 + S.a_off[k], W.hd + S.a_off[k],
                      W.sq + (int64_t)k * N, W.dside + S.side_off[k], W.dego, grad_weights + S.w_off[k], N, S.din[k], S.dout[k]};
        const size_t smem = ((size_t)2 * S.din[k] * (S.dout[k] + 1) + (size_t)2 * kBwdRows * S.din[k] +
                             (size_t)2 * kBwdRows * S.dout[k]) * 4;
        static bool attr_done = false;
        if (!attr_done) {
            NRC_CUDA_CHECK(cudaFuncSetAttribute(ngcf_layer_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
            attr_done = true;
        }
        ngcf_layer_bwd_kernel<<<bwd_grid, 256, smem, st>>>(A);
        NRC_CUDA_CHECK(cudaGetLastError());
        // d_ego (input of this layer) = dego + A_hat^T . dside
        float* out = pp[k & 1];
        rc = nrc_spmm_csr(t_indptr, t_indices, t_values, t_row_order, N, W.dside + S.side_off[k], S.din[k], W.dego, out,
                          nullptr, 0.0f, st);
        if (rc) return rc;
        d_next = out;
    }
    ngcf_finish_e0_kernel<<<grid_for((int64_t)N * S.emb_dim, 256), 256, 0, st>>>(grad_all, d_next, grad_e0, N, S.emb_dim,
                                                                                 S.d_total);
    NRC_CUDA_CHECK(cudaGetLastError());
    NRC_CUDA_CHECK(cudaMemsetAsync(grad_all, 0, (size_t)N * S.d_total * sizeof(float), st));
    return NRC_OK;
}
