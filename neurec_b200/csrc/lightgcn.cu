// CSR SpMM (A_hat . E propagation) and the LightGCN training step built on it.
//
// Replaces (reference paths):
//   model/general_recommender/LightGCN.py:132-149  _create_lightgcn_embed: E_{k+1} = A_hat E_k via
//                                                  tf.sparse_tensor_dense_matmul, E = mean_k E_k
//   model/general_recommender/LightGCN.py:156-166  create_bpr_loss (sum BPR + reg on layer-0 rows)
//   model/general_recommender/LightGCN.py:130      AdamOptimizer(lr).minimize(loss)
//   model/general_recommender/NGCF.py:170-179      the same SpMM (n_fold row slabs are a TF memory
//                                                  work-around; one CSR pass is equivalent)
// Third-party arithmetic restated (tensorflow==1.12.3 sparse_tensor_dense_matmul CPU kernel, not
// vendored): out(m, :) += a_value * b(k, :) for every nnz in row-major COO order, i.e. each
// output row is a SEQUENTIAL sum over its nnz with separately rounded multiply and add (the
// pip wheels carry no FMA).  scipy's csr_matvecs does exactly the same, which is what the oracle
// uses; this kernel keeps that order and rounding => bit-exact SpMM.  The adjoint product of
// the backward pass (A_hat^T . g) visits the nnz of a column in ascending row order, which for
// a symmetric A_hat ('pre', LightGCN.py:63-72) is again this kernel on the same CSR.
//
// Work decomposition: one warp per row, rows visited in caller-supplied (degree-descending)
// order; lane owns dim/32 consecutive columns so every gathered E row is one coalesced
// 128/256/512 B request; (col, val) pairs are fetched 32 at a time and shuffled out.  The graph
// and E (18 MB for gowalla) are L2-resident; the bound is L2 gather bandwidth.
#include <stdlib.h>

#include "common.cuh"
#include "extras.cuh"
#include "graph.cuh"
#include "learner.cuh"
#include "optim.cuh"

namespace nrc {

int32_t g_graph_routes[kGraphRoutes] = {-1, -1, -1, -1, -1, -1, -1, -1, -1};

template <int V> struct VecT;
template <> struct VecT<1> { using T = float; };
template <> struct VecT<2> { using T = float2; };
template <> struct VecT<4> { using T = float4; };

__device__ __forceinline__ void vload(float (&o)[1], const float* p) { o[0] = __ldg(p); }
__device__ __forceinline__ void vload(float (&o)[2], const float* p) {
    const float2 t = __ldg(reinterpret_cast<const float2*>(p)); o[0] = t.x; o[1] = t.y;
}
__device__ __forceinline__ void vload(float (&o)[4], const float* p) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p)); o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w;
}
__device__ __forceinline__ void vload_rw(float (&o)[1], const float* p) { o[0] = *p; }
__device__ __forceinline__ void vload_rw(float (&o)[2], const float* p) {
    const float2 t = *reinterpret_cast<const float2*>(p); o[0] = t.x; o[1] = t.y;
}
__device__ __forceinline__ void vload_rw(float (&o)[4], const float* p) {
    const float4 t = *reinterpret_cast<const float4*>(p); o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w;
}
__device__ __forceinline__ void vstore(float* p, const float (&v)[1]) { *p = v[0]; }
__device__ __forceinline__ void vstore(float* p, const float (&v)[2]) {
    *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
}
__device__ __forceinline__ void vstore(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}

struct SpmmArgs {
    const int64_t* indptr; const int32_t* indices; const float* values; const int32_t* row_order;
    int n_rows; int dim;
    const float* X;      // [*, dim] gathered operand
    const float* bias;   // optional [n_rows, dim]: y = bias + A.x   (backward: g + A^T t)
    float* Y;            // optional output
    float* sum;          // optional running layer sum: sum = (sum + y) [/ div]
    float div;           // 0 = no division; LightGCN.py:147 reduce_mean divides by n_layers+1
    const float* sum_in; // optional: the running sum is READ from here instead of `sum` (first layer: sum = E0 + y
                         // without a copy of E0 into the accumulator first)
};

// V = columns per lane (dim == 32*V).  V == 0: generic dim (lane strides over columns).
template <int V>
__global__ void __launch_bounds__(256) spmm_csr_kernel(const SpmmArgs A) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    constexpr int VV = (V == 0) ? 8 : V;  // generic path: up to 256 columns
    for (int rr = gw; rr < A.n_rows; rr += warps) {
        const int r = A.row_order ? A.row_order[rr] : rr;
        const int64_t beg = A.indptr[r], end = A.indptr[r + 1];
        float acc[VV];
#pragma unroll
        for (int j = 0; j < VV; ++j) acc[j] = 0.0f;
        for (int64_t p = beg; p < end; p += 32) {
            const int cnt = (int)((end - p < 32) ? (end - p) : 32);
            const int my_c = (lane < cnt) ? __ldg(A.indices + p + lane) : 0;
            const float my_v = (lane < cnt) ? __ldg(A.values + p + lane) : 0.0f;
            if constexpr (V != 0) {
                // kDepth gathered rows in flight per warp, then the sequential (order-preserving)
                // accumulation; padding lanes carry c = 0 (a valid row) and are skipped in the sum
                constexpr int kDepth = (V == 4) ? 8 : 16;
#pragma unroll 1
                for (int q0 = 0; q0 < cnt; q0 += kDepth) {
                    float x[kDepth][V];
#pragma unroll
                    for (int j = 0; j < kDepth; ++j) {
                        const int c = __shfl_sync(kFull, my_c, (q0 + j) & 31);
                        vload(x[j], A.X + (size_t)c * A.dim + lane * V);
                    }
#pragma unroll
                    for (int j = 0; j < kDepth; ++j) {
                        const float v = __shfl_sync(kFull, my_v, (q0 + j) & 31);
                        if (q0 + j < cnt) {
#pragma unroll
                            for (int t = 0; t < V; ++t) acc[t] = __fadd_rn(acc[t], __fmul_rn(v, x[j][t]));
                        }
                    }
                }
            } else {
#pragma unroll 4
                for (int q = 0; q < cnt; ++q) {
                    const int c = __shfl_sync(kFull, my_c, q);
                    const float v = __shfl_sync(kFull, my_v, q);
#pragma unroll
                    for (int j = 0; j < VV; ++j) {
                        const int col = lane + 32 * j;
                        if (col < A.dim)
                            acc[j] = __fadd_rn(acc[j], __fmul_rn(v, __ldg(A.X + (size_t)c * A.dim + col)));
                    }
                }
            }
        }
        if constexpr (V != 0) {
            const size_t o = (size_t)r * A.dim + lane * V;
            float (&a)[V] = acc;
            if (A.bias) {
                float b[V];
                vload(b, A.bias + o);
#pragma unroll
                for (int j = 0; j < V; ++j) a[j] = __fadd_rn(b[j], a[j]);
            }
            if (A.Y) vstore(A.Y + o, a);
            if (A.sum) {
                float s[V];
                vload_rw(s, const_cast<float*>(A.sum_in ? A.sum_in : A.sum) + o);
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    s[j] = __fadd_rn(s[j], a[j]);
                    if (A.div != 0.0f) s[j] = __fdiv_rn(s[j], A.div);
                }
                vstore(A.sum + o, s);
            }
        } else {
#pragma unroll
            for (int j = 0; j < VV; ++j) {
                const int col = lane + 32 * j;
                if (col < A.dim) {
                    const size_t o = (size_t)r * A.dim + col;
                    float y = acc[j];
                    if (A.bias) y = __fadd_rn(A.bias[o], y);
                    if (A.Y) A.Y[o] = y;
                    if (A.sum) {
                        float s = __fadd_rn((A.sum_in ? A.sum_in : A.sum)[o], y);
                        if (A.div != 0.0f) s = __fdiv_rn(s, A.div);
                        A.sum[o] = s;
                    }
                }
            }
        }
    }
}

// ----------------------------------------------------------------------------------------
// Default ("fast") SpMM: same product, accumulation order free (north_star's tolerance for this
// path is NDCG within 1e-5, not a bit-exact SpMM; the sequential kernel above stays available
// through nrc_spmm_set_exact for bit-level parity tests).
//   * a gathered row is dim/4 float4 loads, so a warp fetches 32/(dim/4) non-zeros per load
//     instruction (2 for dim 64, 4 for dim 32, 1 for dim 128) -- half the instructions per nnz;
//   * FFMA into two independent accumulator sets (no serial FADD chain), groups reduced by shuffle;
//   * 8 load instructions in flight per warp (16-32 gathered rows);
//   * rows longer than kLongRow are not left to one warp: the CTA's 8 warps stride over the row's
//     32-nnz segments and combine through shared memory in fixed order (deterministic).  A CTA
//     works on units of 8 rows of the caller's (degree-descending) order, so long rows are met by
//     whole units and the decision is one __syncthreads_or per unit.
// ----------------------------------------------------------------------------------------
constexpr int kLongRow = 192;

template <int G, int UNMAX>   // lanes per gathered row: dim == 4 * G, G in {8, 16, 32}; load instructions in flight
__device__ __forceinline__ void spmm_accumulate(const SpmmArgs& A, int64_t beg, int64_t end, int64_t seg_stride,
                                                int lane, float4& acc) {
    constexpr int NPI = 32 / G;            // non-zeros per load instruction
    constexpr int STEPS = 32 / NPI;        // load instructions per 32-nnz segment
    constexpr int UN = (STEPS < UNMAX) ? STEPS : UNMAX;
    const int grp = lane / G, sub = lane % G;
    float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
    for (int64_t p = beg; p < end; p += seg_stride) {
        const int cnt = (int)((end - p < 32) ? (end - p) : 32);
        const int my_c = (lane < cnt) ? __ldg(A.indices + p + lane) : 0;
        const float my_v = (lane < cnt) ? __ldg(A.values + p + lane) : 0.0f;   // padding: 0 * row 0
#pragma unroll 1
        for (int j0 = 0; j0 * NPI < cnt; j0 += UN) {
            float4 x[UN];
            float v[UN];
#pragma unroll
            for (int j = 0; j < UN; ++j) {
                const int src = (j0 + j) * NPI + grp;
                const int c = __shfl_sync(kFull, my_c, src & 31);
                v[j] = __shfl_sync(kFull, my_v, src & 31);
                x[j] = __ldg(reinterpret_cast<const float4*>(A.X + (size_t)c * A.dim) + sub);
            }
#pragma unroll
            for (int j = 0; j < UN; ++j) {
                if ((j0 + j) * NPI + grp < cnt) {          // padding slots gathered row 0: never accumulate them
                    float4& a = (j & 1) ? a1 : a0;
                    a.x = fmaf(v[j], x[j].x, a.x); a.y = fmaf(v[j], x[j].y, a.y);
                    a.z = fmaf(v[j], x[j].z, a.z); a.w = fmaf(v[j], x[j].w, a.w);
                }
            }
        }
    }
    acc.x = a0.x + a1.x; acc.y = a0.y + a1.y; acc.z = a0.z + a1.z; acc.w = a0.w + a1.w;
#pragma unroll
    for (int o = G; o < 32; o <<= 1) {     // sum the 32/G groups (fixed tree)
        acc.x += __shfl_xor_sync(kFull, acc.x, o); acc.y += __shfl_xor_sync(kFull, acc.y, o);
        acc.z += __shfl_xor_sync(kFull, acc.z, o); acc.w += __shfl_xor_sync(kFull, acc.w, o);
    }
}

template <int G>
__device__ __forceinline__ void spmm_epilogue(const SpmmArgs& A, int r, int sub, float4 a) {
    const size_t o = (size_t)r * A.dim + sub * 4;
    if (A.bias) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(A.bias + o));
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    if (A.Y) *reinterpret_cast<float4*>(A.Y + o) = a;
    if (A.sum) {
        float4 s = *reinterpret_cast<const float4*>((A.sum_in ? A.sum_in : A.sum) + o);
        s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
        if (A.div != 0.0f) { s.x = __fdiv_rn(s.x, A.div); s.y = __fdiv_rn(s.y, A.div); s.z = __fdiv_rn(s.z, A.div); s.w = __fdiv_rn(s.w, A.div); }
        *reinterpret_cast<float4*>(A.sum + o) = s;
    }
}

// UNMAX = 4: 4 loads in flight per warp, 64 registers, 4 CTAs per SM (default); UNMAX = 8: 8 in flight, 3 CTAs per SM
template <int G, int UNMAX>
__global__ void __launch_bounds__(256, UNMAX == 4 ? 4 : 3) spmm_csr_fast_kernel(const SpmmArgs A) {
    __shared__ float4 s_part[8][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int units = (A.n_rows + 7) >> 3;
    // this warp's row of the NEXT unit is fetched while the current one is processed (the
    // row_order -> indptr -> indices -> X chain is four dependent L2 round trips otherwise)
    auto fetch = [&](int w, int& r, int64_t& beg, int64_t& end, bool& lng) {
        const int rr = w * 8 + warp;
        const bool live = w < units && rr < A.n_rows;
        r = live ? (A.row_order ? __ldg(A.row_order + rr) : rr) : 0;
        beg = live ? __ldg(A.indptr + r) : 0;
        end = live ? __ldg(A.indptr + r + 1) : 0;
        if (A.row_order) {      // degree-descending order: a unit holds a long row iff its FIRST row is long
            const int r0 = (w < units) ? __ldg(A.row_order + w * 8) : 0;
            lng = (w < units) && (__ldg(A.indptr + r0 + 1) - __ldg(A.indptr + r0)) > kLongRow;
        } else {
            lng = false;        // decided per unit with a CTA vote below
        }
    };
    int r, rn; int64_t beg, end, begn, endn; bool lng, lngn;
    fetch(blockIdx.x, r, beg, end, lng);
    for (int w = blockIdx.x; w < units; w += gridDim.x) {
        fetch(w + gridDim.x, rn, begn, endn, lngn);
        const bool live = w * 8 + warp < A.n_rows;
        const bool any_long = A.row_order ? lng : (bool)__syncthreads_or(live && (end - beg) > kLongRow);
        if (!any_long) {
            if (live) {
                float4 acc;
                spmm_accumulate<G, UNMAX>(A, beg, end, 32, lane, acc);
                if (lane < G) spmm_epilogue<G>(A, r, lane, acc);
            }
        } else {
            // a unit with a long row: every row of the unit by the whole CTA, one after the other
            for (int k = 0; k < 8; ++k) {
                const int rk = w * 8 + k;
                if (rk >= A.n_rows) break;
                const int row = A.row_order ? __ldg(A.row_order + rk) : rk;
                const int64_t b0 = __ldg(A.indptr + row), e0 = __ldg(A.indptr + row + 1);
                float4 acc;
                spmm_accumulate<G, UNMAX>(A, b0 + 32 * warp, e0, 32 * 8, lane, acc);
                s_part[warp][lane] = acc;
                __syncthreads();
                if (warp == 0 && lane < G) {
                    float4 t = s_part[0][lane];
#pragma unroll
                    for (int q = 1; q < 8; ++q) {
                        const float4 u = s_part[q][lane];
                        t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
                    }
                    spmm_epilogue<G>(A, row, lane, t);
                }
                __syncthreads();
            }
        }
        r = rn; beg = begn; end = endn; lng = lngn;
    }
}

static bool g_spmm_exact = false;

static int spmm_launch(const SpmmArgs& A, cudaStream_t st) {
    if (A.n_rows <= 0) return NRC_OK;
    NRC_REQUIRE(A.dim > 0 && A.dim <= 256, NRC_E_LIMIT, "dim %d outside [1, 256]", A.dim);
    const int threads = 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    // both kernels need ceil(n_rows / 8) CTAs of 8 warps for one unit (fast) or one row (exact) per warp; beyond the
    // cap a CTA walks several units, a warp several rows
    g_graph_routes[kRouteSpmmCapped] = ((int64_t)A.n_rows + 7) / 8 > cap ? 1 : 0;
    if (!g_spmm_exact && (A.dim == 32 || A.dim == 64 || A.dim == 128)) {
        int64_t blocks = ((int64_t)A.n_rows + 7) / 8;
        if (blocks > cap) blocks = cap;
        g_graph_routes[kRouteSpmmFast] = 1;
        g_graph_routes[kRouteSpmmWidth] = A.dim / 4;
        static int un = -1;
        // 8 row loads in flight per warp by default (NRC_SPMM_UN=4: four)
        if (un < 0) { const char* e = getenv("NRC_SPMM_UN"); un = (e && atoi(e) == 4) ? 4 : 8; }
        if (un == 8) {
            if (A.dim == 32) spmm_csr_fast_kernel<8, 8><<<(unsigned)blocks, threads, 0, st>>>(A);
            else if (A.dim == 64) spmm_csr_fast_kernel<16, 8><<<(unsigned)blocks, threads, 0, st>>>(A);
            else spmm_csr_fast_kernel<32, 8><<<(unsigned)blocks, threads, 0, st>>>(A);
        } else {
            if (A.dim == 32) spmm_csr_fast_kernel<8, 4><<<(unsigned)blocks, threads, 0, st>>>(A);
            else if (A.dim == 64) spmm_csr_fast_kernel<16, 4><<<(unsigned)blocks, threads, 0, st>>>(A);
            else spmm_csr_fast_kernel<32, 4><<<(unsigned)blocks, threads, 0, st>>>(A);
        }
        NRC_CUDA_CHECK(cudaGetLastError());
        return NRC_OK;
    }
    int64_t blocks = ((int64_t)A.n_rows * 32 + threads - 1) / threads;
    if (blocks > cap) blocks = cap;
    g_graph_routes[kRouteSpmmFast] = 0;
    g_graph_routes[kRouteSpmmWidth] = (A.dim == 32 || A.dim == 64 || A.dim == 128) ? A.dim / 32 : 0;
    if (A.dim == 32) spmm_csr_kernel<1><<<(unsigned)blocks, threads, 0, st>>>(A);
    else if (A.dim == 64) spmm_csr_kernel<2><<<(unsigned)blocks, threads, 0, st>>>(A);
    else if (A.dim == 128) spmm_csr_kernel<4><<<(unsigned)blocks, threads, 0, st>>>(A);
    else spmm_csr_kernel<0><<<(unsigned)blocks, threads, 0, st>>>(A);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// BPR gradient on the propagated table (LightGCN.py:99-104, 156-166): one warp per triplet.
//   x = <E[u], E[U+i]> - <E[u], E[U+j]>;  mf_loss = sum -log_sigmoid(x)
//   emb_loss = reg * sum 1/2 (|E0[u]|^2 + |E0[U+i]|^2 + |E0[U+j]|^2)
// Adds dL/dE (times `scale` = 1/(n_layers+1), the reduce_mean factor) into G and the
// regulariser's gradient reg*E0[row] into R; both dense [N, dim].
__global__ void __launch_bounds__(256)
lightgcn_grad_kernel(const float* __restrict__ E, const float* __restrict__ E0, int num_users,
                     int D, const int32_t* __restrict__ users, const int32_t* __restrict__ pos,
                     const int32_t* __restrict__ neg, int64_t batch, float reg, float scale,
                     float* __restrict__ G, float* __restrict__ R, float* __restrict__ loss) {
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    float mf_acc = 0.0f, emb_acc = 0.0f;
    for (int64_t b = (int64_t)blockIdx.x * wpb + wib; b < batch; b += (int64_t)gridDim.x * wpb) {
        const size_t ru = (size_t)users[b] * D, ri = (size_t)(num_users + pos[b]) * D,
                     rj = (size_t)(num_users + neg[b]) * D;
        float di = 0.f, dj = 0.f, sq = 0.f;
        for (int k = lane; k < D; k += kWarp) {
            const float a = E[ru + k];
            di = fmaf(a, E[ri + k], di);
            dj = fmaf(a, E[rj + k], dj);
            const float a0 = E0[ru + k], b0 = E0[ri + k], c0 = E0[rj + k];
            sq += a0 * a0 + b0 * b0 + c0 * c0;
        }
        di = warp_sum(di); dj = warp_sum(dj); sq = warp_sum(sq);
        const float x = di - dj;
        mf_acc += neg_log_sigmoid(x);
        emb_acc += reg * 0.5f * sq;
        const float g = neg_log_sigmoid_grad(x) * scale;
        for (int k = lane; k < D; k += kWarp) {
            const float a = E[ru + k], bi = E[ri + k], bj = E[rj + k];
            atomicAdd(G + ru + k, g * (bi - bj));
            atomicAdd(G + ri + k, g * a);
            atomicAdd(G + rj + k, -g * a);
            if (reg != 0.0f) {
                atomicAdd(R + ru + k, reg * E0[ru + k]);
                atomicAdd(R + ri + k, reg * E0[ri + k]);
                atomicAdd(R + rj + k, reg * E0[rj + k]);
            }
        }
    }
    if (lane == 0 && loss) {
        atomicAdd(loss, mf_acc);
        atomicAdd(loss + 1, emb_acc);
    }
}

}  // namespace nrc

using namespace nrc;

// 1: every SpMM of this process uses the sequential, separately-rounded accumulation that is
// bit-identical to scipy / TF's CPU kernel (parity tests); 0 (default): the fast order.
extern "C" int nrc_spmm_set_exact(int32_t on) {
    g_spmm_exact = on != 0;
    return NRC_OK;
}

// Host bookkeeping of the routes the most recent graph calls launched (see the header); no device work.
extern "C" int nrc_graph_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "NULL output");
    for (int r = 0; r < kGraphRoutes; ++r) out[r] = g_graph_routes[r];
    return NRC_OK;
}

extern "C" int nrc_spmm_csr(const int64_t* indptr, const int32_t* indices, const float* values,
                            const int32_t* row_order, int32_t n_rows, const float* x, int32_t dim,
                            const float* bias, float* y, float* sum, float div, void* stream) {
    SpmmArgs A{indptr, indices, values, row_order, n_rows, dim, x, bias, y, sum, div};
    return spmm_launch(A, as_stream(stream));
}

extern "C" int nrc_lightgcn_propagate(const int64_t* indptr, const int32_t* indices,
                                      const float* values, const int32_t* row_order,
                                      int32_t n_nodes, int32_t dim, int32_t n_layers,
                                      const float* e0, float* e_final, float* work_a, float* work_b,
                                      void* stream) {
    NRC_REQUIRE(n_layers >= 0, NRC_E_VALUE, "n_layers must be >= 0");
    cudaStream_t st = as_stream(stream);
    const size_t bytes = (size_t)n_nodes * dim * sizeof(float);
    if (n_layers == 0) NRC_CUDA_CHECK(cudaMemcpyAsync(e_final, e0, bytes, cudaMemcpyDeviceToDevice, st));
    const float* x = e0;
    float* bufs[2] = {work_a, work_b};
    for (int k = 0; k < n_layers; ++k) {
        float* y = bufs[k & 1];
        const bool last = (k == n_layers - 1);
        // LightGCN.py:139-147: running sum of the stacked layers, mean at the end
        SpmmArgs A{indptr, indices, values, row_order, n_nodes, dim, x, nullptr, last ? nullptr : y,
                   e_final, last ? (float)(n_layers + 1) : 0.0f, k == 0 ? e0 : nullptr};   // layer 0: e_final = E0 + y
        int rc = spmm_launch(A, st);
        if (rc) return rc;
        x = y;
    }
    return NRC_OK;
}

extern "C" int nrc_lightgcn_bpr_grad(const float* e_final, const float* e0, int32_t num_users,
                                     int32_t dim, const int32_t* users, const int32_t* pos_items,
                                     const int32_t* neg_items, int64_t batch, float reg, float scale,
                                     float* grad_final, float* grad_reg, float* loss2,
                                     void* stream) {
    NRC_REQUIRE(dim > 0 && batch >= 0, NRC_E_VALUE, "dim must be positive, batch >= 0");
    if (batch == 0) return NRC_OK;
    int64_t blocks = (batch + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 8;
    const int capped = blocks > cap ? 1 : 0;
    if (blocks > cap) blocks = cap;
    extras_route(kExLightgcnGrad, blocks, capped);
    lightgcn_grad_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(
        e_final, e0, num_users, dim, users, pos_items, neg_items, batch, reg, scale, grad_final,
        grad_reg, loss2);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_lightgcn_train_epoch(const int64_t* indptr, const int32_t* indices,
                                        const float* values, const int64_t* t_indptr,
                                        const int32_t* t_indices, const float* t_values,
                                        const int32_t* row_order, int32_t num_users,
                                        int32_t num_items, int32_t dim, int32_t n_layers, float* e0,
                                        float* adam_m, float* adam_v, const int32_t* users,
                                        const int32_t* pos_items, const int32_t* neg_items, int64_t n,
                                        int32_t batch_size, float reg, const float* lr_t_host,
                                        const float* hyper_host, float* e_final, float* grad_final,
                                        float* grad_e0, float* work_a, float* work_b,
                                        float* step_loss2, void* stream) {
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    NRC_REQUIRE(n_layers >= 1, NRC_E_LIMIT, "n_layers must be >= 1");
    cudaStream_t st = as_stream(stream);
    const int n_nodes = num_users + num_items;
    const int64_t steps = (n + batch_size - 1) / batch_size;
    if (steps == 0) return NRC_OK;
    if (!t_indptr) { t_indptr = indptr; t_indices = indices; t_values = values; }  // symmetric A_hat
    NRC_CUDA_CHECK(cudaMemsetAsync(step_loss2, 0, (size_t)steps * 2 * sizeof(float), st));
    const size_t bytes = (size_t)n_nodes * dim * sizeof(float);
    float hyper[4] = {hyper_host[0], hyper_host[1], hyper_host[2], hyper_host[3]};
    const float scale = 1.0f / (float)(n_layers + 1);
    for (int64_t s = 0; s < steps; ++s) {
        const int64_t off = s * batch_size;
        const int64_t bs = (n - off < batch_size) ? (n - off) : batch_size;
        int rc = nrc_lightgcn_propagate(indptr, indices, values, row_order, n_nodes, dim, n_layers, e0,
                                        e_final, work_a, work_b, stream);
        if (rc) return rc;
        // grad_final and grad_e0 are zero here (zeroed by the previous step's tail)
        rc = nrc_lightgcn_bpr_grad(e_final, e0, num_users, dim, users + off, pos_items + off,
                                   neg_items + off, bs, reg, scale, grad_final, grad_e0,
                                   step_loss2 + 2 * s, stream);
        if (rc) return rc;
        // backward through the propagation: t_L = g; t_k = g + A^T t_{k+1}; dE0 = R + t_0
        const float* t = grad_final;
        float* bufs[2] = {work_a, work_b};
        for (int k = 0; k < n_layers; ++k) {
            const bool last = (k == n_layers - 1);
            float* y = bufs[k & 1];
            SpmmArgs A{t_indptr, t_indices, t_values, row_order, n_nodes, dim, t, grad_final,
                       last ? nullptr : y, last ? grad_e0 : nullptr, 0.0f};
            rc = spmm_launch(A, st);
            if (rc) return rc;
            t = y;
        }
        hyper[0] = lr_t_host[s];
        OptLaunch L;
        rc = opt_launch_init(L, NRC_OPT_ADAM, hyper);
        if (rc) return rc;
        // dense gradient (it flowed through tf.concat + SpMM): ApplyAdam formulas, every element
        opt_launch_add(L, e0, grad_e0, adam_m, adam_v, nullptr, n_nodes, dim, 1);
        rc = opt_launch_run(L, 0, st);
        if (rc) return rc;
        NRC_CUDA_CHECK(cudaMemsetAsync(grad_final, 0, bytes, st));
    }
    return NRC_OK;
}
