// ItemKNN: item-item similarity, the best `neighbor` items of every column, and ratings = R . W.
//
// Replaces (reference paths):
//   model/general_recommender/ItemKNN.py:11-214    Compute_Similarity_Euclidean (similarity_from_distance_mode "lin")
//   model/general_recommender/ItemKNN.py:240-547   Compute_Similarity_Python (cosine, adjusted, asymmetric, pearson,
//                                                  jaccard / tanimoto, dice, tversky)
//   model/general_recommender/ItemKNN.py:568-589   build_graph's ratings = train.dot(W) and predict(users, None)
//
// The data X [U, I] come as a CSR (rows = users) and the same matrix as a CSC (users ascending in every column), with
// values as double: the host has already centred them (adjusted, pearson), made them binary (tanimoto, dice, tversky)
// and computed the per-item vectors va, vb with numpy exactly as the reference does.  For column c:
//   w_k   = sum over users u of X[u, k] * X[u, c], users ascending (scipy's csr_matvecs order), w_c = 0
//   NORM      (cosine, adjusted, pearson, asymmetric):  w * (1 / (va_c * vb_k + shrink + 1e-6))
//   TANIMOTO  w * (1 / (va_c + va_k - w + shrink + 1e-6))                       (va = un-rooted sums of squares)
//   DICE      w * (1 / (va_c + va_k + shrink + 1e-6))
//   TVERSKY   w * (1 / (w + (va_c - w) * ta + (va_k - w) * tb + shrink + 1e-6))
//   EUCLIDEAN 1 / (sqrt(((va_k + va_c) - 2 w) / (vb_c * vb_k)) + shrink + 1e-9), 0 on the diagonal (vb = sqrt(va))
// each sum and product in the reference's order, every operation a correctly rounded __d*_rn (nothing contracted into
// an FMA), so the float64 values are numpy's bit for bit.  The top min(K, I) values of the column are selected by
// (value descending, row ascending, NaN last) and the ones != 0.0 kept; numpy's introselect breaks ties at the K-th
// value in an order of its own, so the row-ascending rule is the one deviation.
//
// Routes (chosen from the shapes and what the caller vouches for):
//   accumulator  int32 with shared / global atomics when the data are integral and the caller's bound on |w| fits
//                int32 (an integer sum is the same in any order); else float64, one barrier per user of the column so
//                every w_k is summed in ascending user order;
//   tier 0       the CTA's row (I x 8 B: accumulator, then the selection keys in place) in shared memory;
//   tier 1       an int32 accumulator in shared memory, the keys in a per-CTA global row (I above the tier-0 limit);
//   tier 2       accumulator and keys in a per-CTA global row.
// The selection is a block-wide radix select over 64-bit order keys, 8 bits per pass, with warp-aggregated shared
// histogram adds; the survivors are written in ascending row order by a block scan.
#include "common.cuh"

namespace nrc {

constexpr int kKnnThreads = 512;
constexpr int kKnnWarps = kKnnThreads / kWarp;
constexpr int kKnnCtasPerSm = 4;                       // grid cap: 4 x 512 threads fill an SM
constexpr size_t kKnnRowSmem = 220 * 1024;             // dynamic shared memory a CTA's row may take
constexpr int kKnnScoreThreads = 256;
constexpr int kKnnScoreCtasPerSm = 8;

// Order key of a value: larger key = ranked first.  -0.0 ranks as +0.0 (numpy's comparisons do not tell them
// apart), NaN below everything (numpy's sorts put it last).
__device__ __forceinline__ uint64_t knn_key(double v) {
    if (v != v) return 0ull;
    const uint64_t b = (uint64_t)__double_as_longlong(v == 0.0 ? 0.0 : v);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}

__device__ __forceinline__ double knn_unkey(uint64_t key) {
    return __longlong_as_double((long long)((key >> 63) ? (key & ~(1ull << 63)) : ~key));
}

// The similarity of row k in column c from its dot w (already 0 on the diagonal), in the reference's order.
__device__ __forceinline__ double knn_value(int kind, double w, int k, int c, double va_c, double vb_c,
                                            const double* __restrict__ va, const double* __restrict__ vb,
                                            double shrink, double ta, double tb) {
    double den;
    switch (kind) {
    case NRC_ITEMKNN_NORM:
        den = __dmul_rn(va_c, vb[k]);
        break;
    case NRC_ITEMKNN_TANIMOTO:
        den = __dsub_rn(__dadd_rn(va_c, va[k]), w);
        break;
    case NRC_ITEMKNN_DICE:
        den = __dadd_rn(va_c, va[k]);
        break;
    case NRC_ITEMKNN_TVERSKY:
        den = __dadd_rn(__dadd_rn(w, __dmul_rn(__dsub_rn(va_c, w), ta)), __dmul_rn(__dsub_rn(va[k], w), tb));
        break;
    default: {  // NRC_ITEMKNN_EUCLIDEAN
        if (k == c) return 0.0;
        double d = __dsub_rn(__dadd_rn(va[k], va_c), __dmul_rn(2.0, w));
        d = __dsqrt_rn(__ddiv_rn(d, __dmul_rn(vb_c, vb[k])));
        return __ddiv_rn(1.0, __dadd_rn(__dadd_rn(d, shrink), 1e-9));
    }
    }
    return __dmul_rn(w, __ddiv_rn(1.0, __dadd_rn(__dadd_rn(den, shrink), 1e-6)));
}

// Exclusive block-wide prefix sum of x in thread order; *total gets the block's sum.  Every thread must call it.
__device__ __forceinline__ int knn_block_scan(int x, int* total, int32_t* s_warp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = x;
#pragma unroll
    for (int o = 1; o < kWarp; o <<= 1) {
        const int y = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == kWarp - 1) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int t = lane < (int)(blockDim.x >> 5) ? s_warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < kWarp; o <<= 1) {
            const int y = __shfl_up_sync(kFull, t, o);
            if (lane >= o) t += y;
        }
        if (lane < (int)(blockDim.x >> 5)) s_warp[lane] = t;
    }
    __syncthreads();
    const int before = warp ? s_warp[warp - 1] : 0;
    *total = s_warp[(blockDim.x >> 5) - 1];
    __syncthreads();
    return before + incl - x;
}

// One CTA per column c (grid-strided).  Output, slot-major: column c's kept rows and values at [t * I + c] for
// t < counts[c], rows ascending.
__global__ void __launch_bounds__(kKnnThreads, kKnnCtasPerSm)
itemknn_similarity_kernel(int32_t ni, const int64_t* __restrict__ rptr, const int32_t* __restrict__ ridx,
                          const double* __restrict__ rval, const int64_t* __restrict__ cptr,
                          const int32_t* __restrict__ cidx, const double* __restrict__ cval, int kind,
                          const double* __restrict__ va, const double* __restrict__ vb, double shrink, double ta,
                          double tb, int32_t K, int int_acc, int tier, uint64_t* __restrict__ work,
                          int32_t* __restrict__ counts, int32_t* __restrict__ out_rows, float* __restrict__ out_vals) {
    extern __shared__ __align__(16) unsigned char knn_smem[];
    __shared__ int32_t s_hist[256];
    __shared__ int32_t s_warp[kKnnWarps];
    __shared__ int32_t s_pick[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint64_t* row;
    int32_t* acc_i;
    int stride;
    if (tier == 0) {
        row = reinterpret_cast<uint64_t*>(knn_smem);
        acc_i = reinterpret_cast<int32_t*>(row);
        stride = 2;  // the int32 accumulator of row k is the low half of key slot k, so keys replace it in place
    } else if (tier == 1) {
        row = work + (size_t)blockIdx.x * ni;
        acc_i = reinterpret_cast<int32_t*>(knn_smem);
        stride = 1;
    } else {
        row = work + (size_t)blockIdx.x * ni;
        acc_i = reinterpret_cast<int32_t*>(row);
        stride = 2;
    }
    double* acc_d = reinterpret_cast<double*>(row);
    const int Ke = K < ni ? K : ni;

    for (int c = blockIdx.x; c < ni; c += gridDim.x) {
        if (int_acc)
            for (int k = tid; k < ni; k += blockDim.x) acc_i[(size_t)k * stride] = 0;
        else
            for (int k = tid; k < ni; k += blockDim.x) acc_d[k] = 0.0;
        __syncthreads();
        const int64_t cb = cptr[c], ce = cptr[c + 1];
        if (int_acc) {
            // a warp per user of the column, lanes over the user's row
            for (int64_t e = cb + warp; e < ce; e += kKnnWarps) {
                const int u = cidx[e];
                const int xc = (int)cval[e];
                const int64_t rb = rptr[u], re = rptr[u + 1];
                for (int64_t q = rb + lane; q < re; q += kWarp)
                    atomicAdd(acc_i + (size_t)ridx[q] * stride, (int)rval[q] * xc);
            }
        } else {
            // users in ascending order; within one user's row every k is distinct, so plain stores
            for (int64_t e = cb; e < ce; ++e) {
                const int u = cidx[e];
                const double xc = cval[e];
                const int64_t rb = rptr[u], re = rptr[u + 1];
                for (int64_t q = rb + tid; q < re; q += blockDim.x) {
                    const int k = ridx[q];
                    acc_d[k] = __dadd_rn(acc_d[k], __dmul_rn(rval[q], xc));
                }
                __syncthreads();
            }
        }
        __syncthreads();
        const double va_c = va[c], vb_c = vb[c];
        for (int k = tid; k < ni; k += blockDim.x) {
            double w = int_acc ? (double)acc_i[(size_t)k * stride] : acc_d[k];
            if (k == c) w = 0.0;
            row[k] = knn_key(knn_value(kind, w, k, c, va_c, vb_c, va, vb, shrink, ta, tb));
        }
        __syncthreads();

        // radix select of the Ke-th largest key: after the loop every key whose masked bits exceed `pre` is taken,
        // and of the keys equal to `pre` in the masked bits, all (whole) or the first `need` in row order
        uint64_t pre = 0, msk = 0;
        int need = Ke;
        bool whole = Ke >= ni;
        for (int shift = 56; !whole && shift >= 0; shift -= 8) {
            for (int i = tid; i < 256; i += blockDim.x) s_hist[i] = 0;
            __syncthreads();
            for (int base = 0; base < ni; base += blockDim.x) {
                const int k = base + tid;
                int bin = 256;
                if (k < ni) {
                    const uint64_t key = row[k];
                    if ((key & msk) == pre) bin = (int)((key >> shift) & 255);
                }
                const unsigned peers = __match_any_sync(kFull, bin);
                if (bin < 256 && lane == __ffs(peers) - 1) atomicAdd(&s_hist[bin], __popc(peers));
            }
            __syncthreads();
            if (tid == 0) {
                int above = 0, d = 255;
                for (; d > 0 && above + s_hist[d] < need; --d) above += s_hist[d];
                s_pick[0] = d;
                s_pick[1] = need - above;
            }
            __syncthreads();
            const int d = s_pick[0];
            const bool all = s_hist[d] == s_pick[1];
            need = s_pick[1];
            pre |= (uint64_t)d << shift;
            msk |= 255ull << shift;
            whole = all;
            __syncthreads();
        }

        int seen_eq = 0, n_out = 0;
        for (int base = 0; base < ni; base += blockDim.x) {
            const int k = base + tid;
            bool gt = false, eq = false;
            uint64_t key = 0;
            if (k < ni) {
                key = row[k];
                const uint64_t m = key & msk;
                gt = m > pre || (whole && m == pre);
                eq = !whole && m == pre;
            }
            if (!__syncthreads_or(gt || eq)) continue;
            int n_eq;
            const int r_eq = seen_eq + knn_block_scan(eq ? 1 : 0, &n_eq, s_warp);
            seen_eq += n_eq;
            const bool sel = gt || (eq && r_eq < need);
            const double v = knn_unkey(key);
            const bool keep = sel && v != 0.0;  // NaN != 0.0: a NaN the selection reaches is kept, as in numpy
            int n_keep;
            const int pos = n_out + knn_block_scan(keep ? 1 : 0, &n_keep, s_warp);
            n_out += n_keep;
            if (keep) {
                out_rows[(size_t)pos * ni + c] = k;
                out_vals[(size_t)pos * ni + c] = __double2float_rn(v);
            }
        }
        if (tid == 0) counts[c] = n_out;
        __syncthreads();
    }
}

// ratings[b, j] = sum over column j's kept rows k (ascending) with X[u, k] != 0 of X[u, k] * W[k, j] in float64,
// u = users[b], from 0 as scipy's csr_matmat sums, rounded once to float32.  One CTA per user (grid-strided): the
// user's row becomes a bitmap with per-word prefix counts in shared memory, so X[u, k] is found in O(1).
__global__ void __launch_bounds__(kKnnScoreThreads)
itemknn_scores_kernel(int32_t ni, const int64_t* __restrict__ rptr, const int32_t* __restrict__ ridx,
                      const double* __restrict__ rval, const int32_t* __restrict__ counts,
                      const int32_t* __restrict__ wrows, const float* __restrict__ wvals,
                      const int32_t* __restrict__ users, int64_t B, float* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char knn_smem[];
    __shared__ int32_t s_warp[kKnnScoreThreads / kWarp];
    const int words = (ni + 31) >> 5;
    uint32_t* bits = reinterpret_cast<uint32_t*>(knn_smem);
    int32_t* rank = reinterpret_cast<int32_t*>(bits + words);
    const int tid = threadIdx.x;
    for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
        const int u = users[b];
        const int64_t beg = rptr[u], end = rptr[u + 1];
        for (int w = tid; w < words; w += blockDim.x) bits[w] = 0u;
        __syncthreads();
        for (int64_t q = beg + tid; q < end; q += blockDim.x) {
            const int k = ridx[q];
            atomicOr(&bits[k >> 5], 1u << (k & 31));
        }
        __syncthreads();
        int run = 0;
        for (int base = 0; base < words; base += blockDim.x) {
            const int w = base + tid;
            int tot;
            const int p = knn_block_scan(w < words ? __popc(bits[w]) : 0, &tot, s_warp);
            if (w < words) rank[w] = run + p;
            run += tot;
        }
        __syncthreads();
        for (int j = tid; j < ni; j += blockDim.x) {
            double acc = 0.0;
            const int n = counts[j];
            for (int t = 0; t < n; ++t) {
                const size_t s = (size_t)t * ni + j;
                const int k = wrows[s];
                const uint32_t word = bits[k >> 5], bit = 1u << (k & 31);
                if (word & bit) {
                    const double x = rval[beg + rank[k >> 5] + __popc(word & (bit - 1u))];
                    acc = __dadd_rn(acc, __dmul_rn(x, (double)wvals[s]));
                }
            }
            out[(size_t)b * ni + j] = __double2float_rn(acc);
        }
        __syncthreads();
    }
}

}  // namespace nrc

using namespace nrc;

// Host record of ItemKNN's launches, for nrc_itemknn_last_routes (see the header); -1 = no such launch yet, or a field
// the kernel does not decide.  Written just before the launch.
enum KnnKernel { kKnSim, kKnScores, kKnKernels };
enum KnnField { kKnAcc, kKnTier, kKnGrid, kKnCapped, kKnK, kKnSmem, kKnFields };
static struct KnnRoutes {
    int32_t r[kKnKernels][kKnFields];
    KnnRoutes() { for (auto& k : r) for (auto& f : k) f = -1; }
} g_knn_routes;

static void knn_route(int kernel, int acc, int tier, int64_t grid, int capped, int k, int64_t smem) {
    int32_t* r = g_knn_routes.r[kernel];
    r[kKnAcc] = acc; r[kKnTier] = tier; r[kKnGrid] = (int32_t)grid; r[kKnCapped] = capped; r[kKnK] = k;
    r[kKnSmem] = (int32_t)smem;
}

static int64_t knn_grid(int64_t work, int per_sm, int* capped) {
    const int64_t cap = (int64_t)sm_count() * per_sm;
    *capped = work > cap ? 1 : 0;
    return work > cap ? cap : (work < 1 ? 1 : work);
}

static bool knn_global_row(int32_t num_items) { return (size_t)num_items * 8 > kKnnRowSmem; }

extern "C" int64_t nrc_itemknn_work_bytes(int32_t num_items) {
    if (num_items < 1 || !knn_global_row(num_items)) return 0;
    int capped;
    return knn_grid(num_items, kKnnCtasPerSm, &capped) * (int64_t)num_items * 8;
}

extern "C" int nrc_itemknn_similarity(int32_t num_users, int32_t num_items, const int64_t* csr_ptr,
                                      const int32_t* csr_idx, const double* csr_val, const int64_t* csc_ptr,
                                      const int32_t* csc_idx, const double* csc_val, int32_t kind, const double* va,
                                      const double* vb, double shrink, double tversky_alpha, double tversky_beta,
                                      int32_t neighbor, int32_t integral, double gram_bound, void* work,
                                      int64_t work_bytes, int32_t* counts, int32_t* rows, float* vals,
                                      void* stream) {
    NRC_REQUIRE(num_users >= 0 && num_items >= 1, NRC_E_VALUE, "num_users >= 0 and num_items >= 1 required");
    NRC_REQUIRE(kind >= NRC_ITEMKNN_NORM && kind <= NRC_ITEMKNN_EUCLIDEAN, NRC_E_VALUE,
                "similarity kind %d outside [0, 4]", kind);
    NRC_REQUIRE(neighbor >= 1, NRC_E_VALUE, "neighbor >= 1 required");
    NRC_REQUIRE(shrink == shrink && tversky_alpha == tversky_alpha && tversky_beta == tversky_beta, NRC_E_VALUE,
                "shrink and the tversky coefficients must not be NaN");
    NRC_REQUIRE(csr_ptr && csc_ptr && va && vb && counts && rows && vals, NRC_E_VALUE,
                "the CSR, the CSC, the item vectors and the outputs are required");
    const int64_t need = nrc_itemknn_work_bytes(num_items);
    NRC_REQUIRE(work_bytes >= need && (need == 0 || work), NRC_E_VALUE,
                "work of %lld bytes required (nrc_itemknn_work_bytes)", (long long)need);
    const int int_acc = integral && gram_bound >= 0.0 && gram_bound <= 2147483647.0 ? 1 : 0;
    int tier = 0;
    size_t smem = (size_t)num_items * 8;
    if (knn_global_row(num_items)) {
        tier = int_acc && (size_t)num_items * 4 <= kKnnRowSmem ? 1 : 2;
        smem = tier == 1 ? (size_t)num_items * 4 : 0;
    }
    int capped;
    const int64_t grid = knn_grid(num_items, kKnnCtasPerSm, &capped);
    const int Ke = neighbor < num_items ? neighbor : num_items;
    NRC_CUDA_CHECK(cudaFuncSetAttribute(itemknn_similarity_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)kKnnRowSmem));
    knn_route(kKnSim, int_acc ? 0 : 1, tier, grid, capped, Ke, (int64_t)smem);
    itemknn_similarity_kernel<<<(unsigned)grid, kKnnThreads, smem, as_stream(stream)>>>(
        num_items, csr_ptr, csr_idx, csr_val, csc_ptr, csc_idx, csc_val, kind, va, vb, shrink, tversky_alpha,
        tversky_beta, neighbor, int_acc, tier, static_cast<uint64_t*>(work), counts, rows, vals);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_itemknn_scores(int32_t num_items, const int64_t* csr_ptr, const int32_t* csr_idx,
                                  const double* csr_val, int32_t neighbor, const int32_t* counts, const int32_t* rows,
                                  const float* vals, const int32_t* users, int64_t batch, float* out, void* stream) {
    NRC_REQUIRE(num_items >= 1 && batch >= 0 && neighbor >= 1, NRC_E_VALUE,
                "num_items >= 1, neighbor >= 1 and batch >= 0 required");
    const size_t smem = (size_t)((num_items + 31) / 32) * 8;
    NRC_REQUIRE(smem <= kKnnRowSmem, NRC_E_LIMIT, "num_items %d above %d", num_items, (int)(kKnnRowSmem / 8 * 32));
    NRC_REQUIRE(batch == 0 || (csr_ptr && counts && users && out), NRC_E_VALUE,
                "the CSR, W, users and out are required");
    if (batch == 0) return NRC_OK;
    int capped;
    const int64_t grid = knn_grid(batch, kKnnScoreCtasPerSm, &capped);
    NRC_CUDA_CHECK(cudaFuncSetAttribute(itemknn_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)kKnnRowSmem));
    knn_route(kKnScores, -1, -1, grid, capped, neighbor < num_items ? neighbor : num_items, (int64_t)smem);
    itemknn_scores_kernel<<<(unsigned)grid, kKnnScoreThreads, smem, as_stream(stream)>>>(
        num_items, csr_ptr, csr_idx, csr_val, counts, rows, vals, users, batch, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// Host bookkeeping of the routes the most recent ItemKNN launches took (see the header); no device work.
extern "C" int nrc_itemknn_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "out is NULL");
    for (int k = 0; k < kKnKernels; ++k)
        for (int f = 0; f < kKnFields; ++f) out[k * kKnFields + f] = g_knn_routes.r[k][f];
    return NRC_OK;
}
