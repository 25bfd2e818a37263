// WRMF (Hu, Koren and Volinsky, ICDM 2008): one ALS half-step of the implicit-feedback objective.
//
// Replaces (reference paths):
//   model/general_recommender/WRMF.py:27-33   the dense Cui / Pui host matrices (the CSR is the sparsity pattern)
//   model/general_recommender/WRMF.py:51-61   per row: x = solve(Y^T Y + Y^T diag(Cu) Y + lambda I, Y^T ((Cu + 1) * Pu))
//   model/general_recommender/WRMF.py:69-85   one sess.run per user and one per item, every epoch
//
// For every row r of the CSR (a user over the item table, or an item over the user table) with entries J(r):
//   A_r = G + alpha * sum_{j in J(r)} y_j y_j^T + reg * I,   G = Y^T Y over the whole fixed table
//   b_r = (1 + alpha) * sum_{j in J(r)} y_j,                 x_r = A_r^{-1} b_r  (Cholesky, forward and back solve)
// The fixed table does not change during a half, so solving every row in one launch is exactly the reference's loop.
//
// Kernels (fp32 on the SIMT pipes; every sum has one fixed order, so a half-step is bit-reproducible and a row's
// result does not depend on which other rows are in the launch):
//   wrmf_gram_partial_kernel<R>  G's upper triangle over fixed slices of rows, one slice per CTA (slice count depends
//                                only on num_fixed)
//   wrmf_gram_finish_kernel      sums the slices in ascending order and mirrors the triangle: G is exactly symmetric
//   wrmf_solve_warp_kernel<DP>   dim <= 32: one warp per row; A lives in registers, lane j owns column j
//   wrmf_solve_cta_kernel<R>     32 < dim <= 128: one CTA per row; A (padded) in shared memory, right-looking Cholesky
// A pivot that is not positive and finite leaves the row untouched and counts it in *not_spd.
#include <float.h>

#include "common.cuh"

namespace nrc {

constexpr int kWrmfThreads = 256;
constexpr int kWrmfStage = 32;           // rows gathered into shared memory at a time
constexpr int kGramMaxSlices = 256;
constexpr int kGramMinRows = 128;        // rows per Gram slice, at least

static int gram_slices(int64_t n) {
    const int64_t s = (n + kGramMinRows - 1) / kGramMinRows;
    return (int)(s < kGramMaxSlices ? s : kGramMaxSlices);
}

__device__ __forceinline__ bool pivot_ok(float p) { return p > 0.0f && p <= FLT_MAX; }

// Gather up to kWrmfStage rows of the fixed table into Ys[r][0:P) (columns >= dim are zero).  Row r is
// fixed[idx ? idx[first + r] : first + r]; the whole CTA takes part.
__device__ __forceinline__ void stage_rows(float* Ys, int P, const float* __restrict__ fixed, int dim,
                                           const int32_t* __restrict__ idx, int64_t first, int nrows) {
    for (int e = threadIdx.x; e < nrows * P; e += blockDim.x) {
        const int r = e / P, c = e - r * P;
        float v = 0.0f;
        if (c < dim) {
            const int64_t row = idx ? (int64_t)__ldg(idx + first + r) : first + r;
            v = __ldg(fixed + row * dim + c);
        }
        Ys[e] = v;
    }
}

// acc[a][b] += sum_r Ys[r][ty R + a] * Ys[r][tx R + b] over the staged rows in ascending order.  Thread (tx, ty) of
// a 16 x 16 grid owns one R x R block; only blocks on or above the diagonal (ty <= tx) are computed.
template <int R>
__device__ __forceinline__ void outer_accumulate(const float* Ys, int P, int nrows, int tx, int ty,
                                                 float (&acc)[R][R]) {
    for (int r = 0; r < nrows; ++r) {
        const float* y = Ys + r * P;
        float a[R], b[R];
#pragma unroll
        for (int q = 0; q < R; ++q) { a[q] = y[ty * R + q]; b[q] = y[tx * R + q]; }
#pragma unroll
        for (int p = 0; p < R; ++p)
#pragma unroll
            for (int q = 0; q < R; ++q) acc[p][q] = fmaf(a[p], b[q], acc[p][q]);
    }
}

// partial[s] = sum over rows [s * rows_per, min(n, (s + 1) * rows_per)) of y y^T, blocks on or above the diagonal.
template <int R>
__global__ void __launch_bounds__(kWrmfThreads)
wrmf_gram_partial_kernel(const float* __restrict__ fixed, int64_t n, int dim, int64_t rows_per, float* __restrict__ partial) {
    extern __shared__ __align__(16) float smem[];
    constexpr int P = 16 * R;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const bool mine = ty <= tx && ty * R < dim && tx * R < dim;
    float acc[R][R];
#pragma unroll
    for (int p = 0; p < R; ++p)
#pragma unroll
        for (int q = 0; q < R; ++q) acc[p][q] = 0.0f;
    const int64_t begin = blockIdx.x * rows_per;
    const int64_t end = begin + rows_per < n ? begin + rows_per : n;
    for (int64_t r0 = begin; r0 < end; r0 += kWrmfStage) {
        const int nr = (int)(end - r0 < kWrmfStage ? end - r0 : kWrmfStage);
        __syncthreads();
        stage_rows(smem, P, fixed, dim, nullptr, r0, nr);
        __syncthreads();
        if (mine) outer_accumulate<R>(smem, P, nr, tx, ty, acc);
    }
    if (!mine) return;
    float* out = partial + (int64_t)blockIdx.x * dim * dim;
#pragma unroll
    for (int p = 0; p < R; ++p)
#pragma unroll
        for (int q = 0; q < R; ++q) {
            const int i = ty * R + p, j = tx * R + q;
            if (i < dim && j < dim) out[i * dim + j] = acc[p][q];
        }
}

// G[i][j] = G[j][i] = sum_{s ascending} partial[s][i][j] for i <= j
__global__ void __launch_bounds__(kWrmfThreads)
wrmf_gram_finish_kernel(const float* __restrict__ partial, int slices, int dim, float* __restrict__ G) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= dim * dim) return;
    const int i = e / dim, j = e - i * dim;
    if (i > j) return;
    float s = 0.0f;
    for (int k = 0; k < slices; ++k) s += __ldg(partial + (int64_t)k * dim * dim + e);
    G[i * dim + j] = s;
    G[j * dim + i] = s;
}

struct SolveArgs {
    const float* fixed; const int64_t* indptr; const int32_t* indices; const int32_t* row_order;
    const float* G; int num_rows, dim; float alpha, reg; float* out; int32_t* not_spd;
};

// dim <= DP <= 32: one warp per row.  Lane j holds column j of A in a[0:DP) (rows and columns >= dim are the
// identity).  After the factorisation a[i] = L[max(i, j)][min(i, j)]: row j of L below the diagonal and column j on
// and below it, which is what lane j needs in the forward (row) and back (column) solves.
template <int DP>
__global__ void __launch_bounds__(kWrmfThreads)
wrmf_solve_warp_kernel(const SolveArgs S) {
    constexpr int kWarps = kWrmfThreads / kWarp;
    __shared__ __align__(16) float stage[kWarps][kWrmfStage * DP];
    __shared__ int32_t sidx[kWarps][kWrmfStage];
    __shared__ __align__(16) float col[kWarps][DP];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * kWarps + w;
    if (t >= S.num_rows) return;                        // warp-uniform
    const int row = S.row_order ? __ldg(S.row_order + t) : t;
    const int d = S.dim;
    const int64_t p0 = __ldg(S.indptr + row), p1 = __ldg(S.indptr + row + 1);
    float a[DP];
#pragma unroll
    for (int i = 0; i < DP; ++i) a[i] = 0.0f;
    float bb = 0.0f;
    float* Ys = stage[w];
    for (int64_t q0 = p0; q0 < p1; q0 += kWrmfStage) {
        const int nr = (int)(p1 - q0 < kWrmfStage ? p1 - q0 : kWrmfStage);
        __syncwarp();
        if (lane < nr) sidx[w][lane] = __ldg(S.indices + q0 + lane);
        __syncwarp();
        for (int e = lane; e < nr * DP; e += kWarp) {
            const int r = e / DP, c = e - r * DP;
            Ys[e] = c < d ? __ldg(S.fixed + (int64_t)sidx[w][r] * d + c) : 0.0f;
        }
        __syncwarp();
        if (lane < DP) {
            for (int r = 0; r < nr; ++r) {
                const float* y = Ys + r * DP;
                const float yl = y[lane];
                bb += yl;
#pragma unroll
                for (int i = 0; i < DP; i += 4) {
                    const float4 v = *reinterpret_cast<const float4*>(y + i);
                    a[i] = fmaf(v.x, yl, a[i]); a[i + 1] = fmaf(v.y, yl, a[i + 1]);
                    a[i + 2] = fmaf(v.z, yl, a[i + 2]); a[i + 3] = fmaf(v.w, yl, a[i + 3]);
                }
            }
        }
    }
    // A = G + alpha * S + reg * I,  b = (1 + alpha) * sum y
#pragma unroll
    for (int i = 0; i < DP; ++i) {
        if (lane < d && i < d) a[i] = __ldg(S.G + i * d + lane) + S.alpha * a[i] + (i == lane ? S.reg : 0.0f);
        else a[i] = i == lane ? 1.0f : 0.0f;
    }
    bb = lane < d ? (1.0f + S.alpha) * bb : 0.0f;
    bool ok = true;
    float* cs = col[w];
#pragma unroll
    for (int k = 0; k < DP; ++k) {
        const float piv = __shfl_sync(kFull, a[k], k);
        ok = ok && pivot_ok(piv);
        const float ukk = sqrtf(piv);
        const float c = lane == k ? ukk : a[k] / ukk;   // lane j > k: L[j][k]
        if (lane >= k) a[k] = c;
        if (lane > k && lane < DP) cs[lane] = c;
        __syncwarp();
        if (lane > k) {
#pragma unroll
            for (int i = k + 1; i < DP; ++i) a[i] = fmaf(-cs[i], c, a[i]);
        } else if (lane == k) {
#pragma unroll
            for (int i = k + 1; i < DP; ++i) a[i] = cs[i];
        }
        __syncwarp();
    }
    if (!ok) {
        if (lane == 0) atomicAdd(S.not_spd, 1);
        return;
    }
    // L z = b (lane j > k uses L[j][k] = a[k]), then L^T x = z (lane j < k uses L[k][j] = a[k])
#pragma unroll
    for (int k = 0; k < DP; ++k) {
        if (lane == k) bb = bb / a[k];
        const float z = __shfl_sync(kFull, bb, k);
        if (lane > k) bb = fmaf(-a[k], z, bb);
    }
#pragma unroll
    for (int k = DP - 1; k >= 0; --k) {
        if (lane == k) bb = bb / a[k];
        const float x = __shfl_sync(kFull, bb, k);
        if (lane < k) bb = fmaf(-a[k], x, bb);
    }
    if (lane < d) S.out[(int64_t)row * d + lane] = bb;
}

// 32 < dim <= P = 16 R: one CTA per row.  The rows are gathered into the region that later holds A; the outer
// products accumulate in the R x R register blocks of outer_accumulate.  A's upper triangle M[i][j] (i <= j, row
// stride P + 1) is factored in place as A = U^T U, then U^T z = b and U x = z.
template <int R>
__global__ void __launch_bounds__(kWrmfThreads, 2)
wrmf_solve_cta_kernel(const SolveArgs S) {
    constexpr int P = 16 * R, LD = P + 1, kGroups = kWrmfThreads / P;
    extern __shared__ __align__(16) float smem[];
    float* M = smem;                                    // [P][LD]; the staging area before A is formed
    float* bs = smem + P * LD;                          // [P]
    __shared__ int ok_flag;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int row = S.row_order ? __ldg(S.row_order + blockIdx.x) : blockIdx.x;
    const int d = S.dim;
    const bool mine = ty <= tx && ty * R < d && tx * R < d;
    const int64_t p0 = __ldg(S.indptr + row), p1 = __ldg(S.indptr + row + 1);
    float acc[R][R];
#pragma unroll
    for (int p = 0; p < R; ++p)
#pragma unroll
        for (int q = 0; q < R; ++q) acc[p][q] = 0.0f;
    float bsum = 0.0f;
    for (int64_t q0 = p0; q0 < p1; q0 += kWrmfStage) {
        const int nr = (int)(p1 - q0 < kWrmfStage ? p1 - q0 : kWrmfStage);
        __syncthreads();
        stage_rows(M, P, S.fixed, d, S.indices, q0, nr);
        __syncthreads();
        if (mine) outer_accumulate<R>(M, P, nr, tx, ty, acc);
        if (tid < d)
            for (int r = 0; r < nr; ++r) bsum += M[r * P + tid];
    }
    __syncthreads();
    if (mine) {
#pragma unroll
        for (int p = 0; p < R; ++p)
#pragma unroll
            for (int q = 0; q < R; ++q) {
                const int i = ty * R + p, j = tx * R + q;
                if (i <= j && j < d) M[i * LD + j] = __ldg(S.G + i * d + j) + S.alpha * acc[p][q] + (i == j ? S.reg : 0.0f);
            }
    }
    if (tid < d) bs[tid] = (1.0f + S.alpha) * bsum;
    if (tid == 0) ok_flag = 1;
    const int j = tid % P, g = tid / P;
    for (int k = 0; k < d; ++k) {
        __syncthreads();
        const float piv = M[k * LD + k];
        if (!pivot_ok(piv)) {                           // the same value for every thread: a uniform exit
            if (tid == 0) ok_flag = 0;
            break;
        }
        const float ukk = sqrtf(piv);
        if (g == 0 && j > k && j < d) M[k * LD + j] = M[k * LD + j] / ukk;
        __syncthreads();
        if (g == 0 && j == k) M[k * LD + k] = ukk;      // after the barrier: every thread has read the pivot
        if (j > k && j < d) {
            const float ukj = M[k * LD + j];
            for (int i = k + 1 + g; i <= j; i += kGroups) M[i * LD + j] = fmaf(-M[k * LD + i], ukj, M[i * LD + j]);
        }
    }
    __syncthreads();
    if (!ok_flag) {
        if (tid == 0) atomicAdd(S.not_spd, 1);
        return;
    }
    if (tid >= kWarp) return;
    // U^T z = b: z_k = b_k / U[k][k], then b_j -= U[k][j] z_k for j > k (row k of U)
    for (int k = 0; k < d; ++k) {
        const float z = bs[k] / M[k * LD + k];
        __syncwarp();
        for (int jj = k + 1 + tid; jj < d; jj += kWarp) bs[jj] = fmaf(-M[k * LD + jj], z, bs[jj]);
        if (tid == 0) bs[k] = z;
        __syncwarp();
    }
    // U x = z: x_k = z_k / U[k][k], then z_j -= U[j][k] x_k for j < k (column k of U)
    for (int k = d - 1; k >= 0; --k) {
        const float x = bs[k] / M[k * LD + k];
        __syncwarp();
        for (int jj = tid; jj < k; jj += kWarp) bs[jj] = fmaf(-M[jj * LD + k], x, bs[jj]);
        if (tid == 0) bs[k] = x;
        __syncwarp();
    }
    for (int jj = tid; jj < d; jj += kWarp) S.out[(int64_t)row * d + jj] = bs[jj];
}

template <int R>
static int launch_gram(const float* fixed, int64_t n, int dim, float* partial, int slices, int64_t rows_per,
                       cudaStream_t st) {
    const size_t smem = (size_t)kWrmfStage * 16 * R * sizeof(float);
    wrmf_gram_partial_kernel<R><<<slices, kWrmfThreads, smem, st>>>(fixed, n, dim, rows_per, partial);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

template <int R>
static int launch_cta_solve(const SolveArgs& S, cudaStream_t st) {
    constexpr int P = 16 * R;
    const size_t smem = ((size_t)P * (P + 1) + P) * sizeof(float);
    static bool attr = false;
    if (!attr) {
        NRC_CUDA_CHECK(cudaFuncSetAttribute(wrmf_solve_cta_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    wrmf_solve_cta_kernel<R><<<S.num_rows, kWrmfThreads, smem, st>>>(S);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

template <int DP>
static int launch_warp_solve(const SolveArgs& S, cudaStream_t st) {
    constexpr int kWarps = kWrmfThreads / kWarp;
    wrmf_solve_warp_kernel<DP><<<(S.num_rows + kWarps - 1) / kWarps, kWrmfThreads, 0, st>>>(S);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

}  // namespace nrc

using namespace nrc;

extern "C" int64_t nrc_wrmf_work_floats(int32_t num_rows_max, int32_t dim) {
    if (num_rows_max < 0 || dim < 1) return 0;
    return (int64_t)dim * dim * (1 + gram_slices(num_rows_max));
}

extern "C" int nrc_wrmf_half_step(const float* fixed, int32_t num_fixed, const int64_t* indptr, const int32_t* indices,
                                  const int32_t* row_order, int32_t num_rows, int32_t dim, float alpha, float reg,
                                  float* out, float* work, int32_t* not_spd, void* stream) {
    NRC_REQUIRE(dim >= 1 && dim <= 128, NRC_E_LIMIT, "WRMF embedding_size %d outside [1, 128]", dim);
    NRC_REQUIRE(isfinite(alpha) && alpha >= 0.0f, NRC_E_VALUE, "WRMF alpha must be finite and >= 0, got %g", alpha);
    NRC_REQUIRE(isfinite(reg) && reg >= 0.0f, NRC_E_VALUE, "WRMF reg_mf must be finite and >= 0, got %g", reg);
    NRC_REQUIRE(num_fixed >= 0 && num_rows >= 0, NRC_E_VALUE, "bad WRMF shape");
    cudaStream_t st = as_stream(stream);
    NRC_CUDA_CHECK(cudaMemsetAsync(not_spd, 0, sizeof(int32_t), st));
    float* G = work;
    float* partial = work + (int64_t)dim * dim;
    const int slices = gram_slices(num_fixed);
    if (slices == 0) {
        NRC_CUDA_CHECK(cudaMemsetAsync(G, 0, sizeof(float) * dim * dim, st));
    } else {
        const int64_t rows_per = ((int64_t)num_fixed + slices - 1) / slices;
        int rc = dim <= 16 ? launch_gram<1>(fixed, num_fixed, dim, partial, slices, rows_per, st)
               : dim <= 32 ? launch_gram<2>(fixed, num_fixed, dim, partial, slices, rows_per, st)
               : dim <= 64 ? launch_gram<4>(fixed, num_fixed, dim, partial, slices, rows_per, st)
                           : launch_gram<8>(fixed, num_fixed, dim, partial, slices, rows_per, st);
        if (rc) return rc;
        wrmf_gram_finish_kernel<<<(dim * dim + kWrmfThreads - 1) / kWrmfThreads, kWrmfThreads, 0, st>>>(partial, slices, dim, G);
        NRC_CUDA_CHECK(cudaGetLastError());
    }
    if (num_rows == 0) return NRC_OK;
    const SolveArgs S{fixed, indptr, indices, row_order, G, num_rows, dim, alpha, reg, out, not_spd};
    if (dim <= 8) return launch_warp_solve<8>(S, st);
    if (dim <= 16) return launch_warp_solve<16>(S, st);
    if (dim <= 32) return launch_warp_solve<32>(S, st);
    if (dim <= 64) return launch_cta_solve<4>(S, st);
    return launch_cta_solve<8>(S, st);
}
