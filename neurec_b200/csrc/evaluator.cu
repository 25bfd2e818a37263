// Evaluator kernels: top-K selection with libstdc++-identical tie order + ranking metrics.
//
// Replaces (reference paths):
//   evaluator/backend/cpp/include/evaluate.h:23-72   eval_one_user / cpp_evaluate_matrix
//   evaluator/backend/cpp/include/metric.h:17-117    precision / recall / ap / ndcg / mrr
//   util/cython/include/arg_topk.h:15-45             arg_top_k_1d / arg_top_k_2d
//   evaluator/backend/cpp/uni_evaluator.py:132-146   predict -> mask -> eval (fused path)
//
// Selection semantics.  The reference ranks with std::partial_sort_copy(index, ..., L slots,
// comp = ratings[a] > ratings[b]).  libstdc++ implements it as: copy the first L indices,
// make_heap (root = smallest rating), then for every later index i: if ratings[i] >
// ratings[root] replace the root (__adjust_heap), finally sort_heap.  Which of several equal
// ratings survives and in what order is an artefact of those heap operations, so to be
// bit-exact we run EXACTLY those heap operations -- but only on the few elements that beat the
// current root.  The root value never decreases, so a warp can test 32 elements at a time
// against a (possibly stale, hence lower) threshold with one ballot, and hand the rare
// survivors, in ascending index order, to lane 0 which replays the sequential heap update.
// Expected survivors per row: ~L*ln(N/L), e.g. ~280 of 40 981 items for L = 40.
#include <float.h>
#include <math.h>

#include "common.cuh"
#include "tc_eval.cuh"

namespace nrc {

constexpr int kMaxTopK = 512;       // top_k limit of this build (L = 2*top_k <= 1024)
constexpr int kMaxMetrics = 8;

// Position-only tables, computed on the host with the host libm so that they carry the same
// bits as the reference's `1.0/log2(i+2)` (metric.h:77-82) evaluated on the host.
__constant__ double c_inv_log2[kMaxTopK];   // 1.0 / log2(i + 2)
__constant__ float c_idcg[kMaxTopK];        // float running sum of the above (iDCG after i+1 terms)
__constant__ int c_metric[kMaxMetrics];

static bool g_tables_ready = false;
static bool g_force_exact = false;   // nrc_eval_force_exact: skip the tie-free fast passes

// __constant__ tables live per device: remember which device holds them and upload again when the
// calling thread has switched devices (one process per GPU is the supported model; this keeps a
// process that touches a second device correct instead of silently reading zeros).
static int g_tables_dev = -1;

static int upload_tables() {
    int dev = 0;
    NRC_CUDA_CHECK(cudaGetDevice(&dev));
    if (g_tables_ready && dev == g_tables_dev) return NRC_OK;
    g_tables_dev = dev;
    static double inv[kMaxTopK];
    static float idcg[kMaxTopK];
    float acc = 0.0f;
    for (int i = 0; i < kMaxTopK; ++i) {
        inv[i] = 1.0 / log2((double)(i + 2));
        acc = (float)((double)acc + inv[i]);  // metric.h:82  iDCG += 1.0/log2(i+2)
        idcg[i] = acc;
    }
    NRC_CUDA_CHECK(cudaMemcpyToSymbol(c_inv_log2, inv, sizeof(inv)));
    NRC_CUDA_CHECK(cudaMemcpyToSymbol(c_idcg, idcg, sizeof(idcg)));
    g_tables_ready = true;
    return NRC_OK;
}

// ----------------------------------------------------------------------------------------
// libstdc++ heap primitives (bits/stl_heap.h) on parallel (index, value) arrays.
// comp(a, b) := value[a] > value[b].  Executed by ONE lane.
// ----------------------------------------------------------------------------------------
struct Heap {
    int* idx;
    float* val;
};

__device__ __forceinline__ void heap_push(Heap h, int hole, int top, int vi, float vv) {
    int parent = (hole - 1) / 2;
    while (hole > top && h.val[parent] > vv) {
        h.idx[hole] = h.idx[parent];
        h.val[hole] = h.val[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    h.idx[hole] = vi;
    h.val[hole] = vv;
}

__device__ __forceinline__ void heap_adjust(Heap h, int hole, int len, int vi, float vv) {
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (h.val[child] > h.val[child - 1]) child--;
        h.idx[hole] = h.idx[child];
        h.val[hole] = h.val[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        h.idx[hole] = h.idx[child - 1];
        h.val[hole] = h.val[child - 1];
        hole = child - 1;
    }
    heap_push(h, hole, top, vi, vv);
}

__device__ __forceinline__ void heap_make(Heap h, int len) {
    if (len < 2) return;
    int parent = (len - 2) / 2;
    for (;;) {
        heap_adjust(h, parent, len, h.idx[parent], h.val[parent]);
        if (parent == 0) return;
        parent--;
    }
}

__device__ __forceinline__ void heap_sort(Heap h, int len) {
    while (len > 1) {
        --len;
        int vi = h.idx[len];
        float vv = h.val[len];
        h.idx[len] = h.idx[0];
        h.val[len] = h.val[0];
        heap_adjust(h, 0, len, vi, vv);
    }
}

// Offer the warp's 32 candidates (v, idx) -- idx ascending with the lane id -- to the heap.
// Returns the current root value (the new threshold) in every lane.
__device__ __forceinline__ float offer_candidates(Heap h, int L, float v, int idx, bool valid,
                                                  float thr, int lane) {
    unsigned m = __ballot_sync(kFull, valid && v > thr);
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const float cv = __shfl_sync(kFull, v, src);
        const int ci = __shfl_sync(kFull, idx, src);
        if (lane == 0 && cv > h.val[0]) heap_adjust(h, 0, L, ci, cv);  // evaluate.h:40-41
        __syncwarp();
        thr = h.val[0];
    }
    return thr;
}

// evaluate.h:40: the first L indices, with their scores score(i), seed the heap; then make_heap.
// Returns the root value (the first threshold) in every lane.
template <class Score>
__device__ __forceinline__ float heap_seed(Heap h, int L, int lane, Score score) {
    for (int i = lane; i < L; i += kWarp) {
        h.idx[i] = i;
        h.val[i] = score(i);
    }
    __syncwarp();
    if (lane == 0) heap_make(h, L);
    __syncwarp();
    return h.val[0];
}

// ----------------------------------------------------------------------------------------
// Tie-free selection (see eval_mf_fast_kernel): the running top-(K+1) of a user as a sorted list
// over the warp's lanes, lane r holding the rank-r entry (tv, ti); thr = the (K+1)-th value.
// ----------------------------------------------------------------------------------------

// Offer the warp's 32 candidates (v, idx; ok = eligible), in lane order.  An entry goes after every
// entry >= it, so among equal values the one offered first keeps the better rank.  kLaneLinear: idx is
// (idx of lane 0) + lane, so a winner's index is computed rather than shuffled (fewer live registers).
template <bool kLaneLinear = true>
__device__ __forceinline__ void topk_offer(float v, int idx, bool ok, float& tv, int& ti, float& thr, int K,
                                           int lane) {
    unsigned c = __ballot_sync(kFull, ok && v > thr);
    while (c) {
        const int src = __ffs(c) - 1;
        c &= c - 1;
        const float cv = __shfl_sync(kFull, v, src);
        const int ci = kLaneLinear ? idx - lane + src : __shfl_sync(kFull, idx, src);
        if (!(cv > thr)) continue;   // the threshold rose since the ballot
        const int pos = __popc(__ballot_sync(kFull, lane <= K && tv >= cv));
        const float up_v = __shfl_up_sync(kFull, tv, 1);
        const int up_i = __shfl_up_sync(kFull, ti, 1);
        if (lane > pos) { tv = up_v; ti = up_i; }
        if (lane == pos) { tv = cv; ti = ci; }
        thr = __shfl_sync(kFull, tv, K);
    }
}

// Whether the list decides the user without the heap: its K+1 values are strictly decreasing and the
// last is above -inf, and no lane reports a NaN among the L items that seed the reference's heap
// (every heap comparison with a NaN fails, which reorders the heap; the list never holds a NaN).
__device__ __forceinline__ bool topk_decided(float tv, bool seed_nan, int K, int lane) {
    const float nxt = __shfl_down_sync(kFull, tv, 1);
    const bool bad = (lane < K && !(tv > nxt)) || (lane == K && !(tv > -INFINITY)) || seed_nan;
    return !__ballot_sync(kFull, bad);
}

// ----------------------------------------------------------------------------------------
// metric.h:17-109 for one user, executed by one warp.
//   rank: smem, top_k ranked item ids; truth: sorted global row; scratch: 3*K words of smem.
// Float/double expression shapes follow metric.h literally (see oracle/neurec_oracle.c).
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void metrics_for_user(const int* rank, int K, const int32_t* truth,
                                                 int T, int* s_cnt, float* s_sum_pre,
                                                 float* s_dcg, int M, float* out_row, int lane) {
    // hit flags -> stash as 0/1 in s_cnt, prefix-summed serially below
    for (int i = lane; i < K; i += kWarp) s_cnt[i] = sorted_contains(truth, T, rank[i]) ? 1 : 0;
    __syncwarp();
    int first_hit = K;
    if (lane == 0) {
        int hits = 0;
        float sum_pre = 0.0f, dcg = 0.0f;
        int fh = K;
        for (int i = 0; i < K; ++i) {
            if (s_cnt[i]) {
                if (hits == 0) fh = i;
                hits += 1;
                const float pre = (float)__ddiv_rn((double)hits, (double)(i + 1));  // metric.h:59
                sum_pre = __fadd_rn(sum_pre, pre);                                  // metric.h:60
                dcg = (float)__dadd_rn((double)dcg, c_inv_log2[i]);                 // metric.h:78
            }
            s_cnt[i] = hits;
            s_sum_pre[i] = sum_pre;
            s_dcg[i] = dcg;
        }
        first_hit = fh;
    }
    first_hit = __shfl_sync(kFull, first_hit, 0);
    __syncwarp();
    const float Tf = (float)T;
    for (int i = lane; i < K; i += kWarp) {
        const int hits = s_cnt[i];
        for (int m = 0; m < M; ++m) {
            float r;
            switch (c_metric[m]) {
                case NRC_METRIC_PRECISION:  // metric.h:26
                    r = (float)__ddiv_rn((double)hits, (double)(i + 1));
                    break;
                case NRC_METRIC_RECALL:  // metric.h:41
                    r = (float)__ddiv_rn((double)hits, (double)T);
                    break;
                case NRC_METRIC_MAP: {  // metric.h:62-63
                    const float den = (Tf < (float)(i + 1)) ? Tf : (float)(i + 1);
                    r = (hits == 0) ? 0.0f : __fdiv_rn(s_sum_pre[i], den);
                    break;
                }
                case NRC_METRIC_NDCG: {  // metric.h:80-84
                    const float idcg = (T == 0) ? 0.0f : c_idcg[(i < T ? i : T - 1)];
                    r = __fdiv_rn(s_dcg[i], idcg);
                    break;
                }
                default:  // NRC_METRIC_MRR, metric.h:92-106
                    r = (i >= first_hit) ? (float)__ddiv_rn(1.0, (double)(first_hit + 1)) : 0.0f;
                    break;
            }
            out_row[m * K + i] = r;
        }
    }
}

// Per-user epilogue, one warp.  rank: the user's K ranked item ids in shared memory; scratch: 3K words
// of shared memory.  Writes the ranks row `row` (if ranks) and the metric row `row` against the test
// items of CSR row `test_row` (if results).  Every kernel keeps, per user, the ranked ids followed by
// the scratch: [rank K][scratch 3K] when it selects with the top-(K+1) list, [heap idx L][heap val L]
// [scratch 3K] when it replays the heap (rank = heap idx after heap_sort).
__device__ __forceinline__ void user_epilogue(const int* rank, int* scratch, int K, int row, int test_row,
                                              const int64_t* test_ptr, const int32_t* test_idx, int M,
                                              float* results, int32_t* ranks, int lane) {
    __syncwarp();
    if (ranks)
        for (int i = lane; i < K; i += kWarp) ranks[(size_t)row * K + i] = rank[i];
    if (results) {
        const int64_t t0 = test_ptr[test_row];
        const int T = (int)(test_ptr[test_row + 1] - t0);
        float* s_sum_pre = reinterpret_cast<float*>(scratch + K);
        metrics_for_user(rank, K, test_idx + t0, T, scratch, s_sum_pre, s_sum_pre + K, M,
                         results + (size_t)row * M * K, lane);
    }
}

// ----------------------------------------------------------------------------------------
// Kernel A: score matrix given.  One warp per row; coalesced streaming read of the row.
// ----------------------------------------------------------------------------------------
constexpr int kRowUnroll = 8;

template <bool kMetrics>
__global__ void __launch_bounds__(256)
eval_rows_kernel(const float* __restrict__ scores, int N, int rows, int K, int L,
                 const int64_t* __restrict__ tptr, const int32_t* __restrict__ tidx, int M,
                 float* __restrict__ results, int32_t* __restrict__ ranks, int fast) {
    extern __shared__ int smem[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int row = blockIdx.x * (blockDim.x >> 5) + warp;
    if (row >= rows) return;
    Heap h;
    h.idx = smem + warp * (2 * L + 3 * K);
    h.val = reinterpret_cast<float*>(h.idx + L);
    int* scratch = h.idx + 2 * L;
    if (!kMetrics) results = nullptr;

    const float* __restrict__ r = scores + (size_t)row * N;
    bool decided = false;
    if (fast) {
        // tie-free fast pass: if the top-(K+1) list decides the row, the reference's first K ranks
        // are exactly this list, otherwise the exact heap replay below ranks the row.
        float tv = -INFINITY, fthr = -INFINITY;
        int ti = -1;
        for (int base = 0; base < N; base += kWarp * kRowUnroll) {
            float v[kRowUnroll];
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) {
                const int i = base + u * kWarp + lane;
                v[u] = (i < N) ? __ldcs(r + i) : -INFINITY;
            }
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) topk_offer(v[u], base + u * kWarp + lane, true, tv, ti, fthr, K, lane);
        }
        // A NaN at i >= L is never admitted by the reference either.  L <= 2K <= 62 here.
        const bool seed_nan = (lane < L && isnan(r[lane])) || (lane + kWarp < L && isnan(r[lane + kWarp]));
        decided = topk_decided(tv, seed_nan, K, lane);
        if (decided && lane < K) h.idx[lane] = ti;
    }
    if (!decided) {
        float thr = heap_seed(h, L, lane, [&](int i) { return r[i]; });
        for (int base = L; base < N; base += kWarp * kRowUnroll) {
            float v[kRowUnroll];
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) {
                const int i = base + u * kWarp + lane;
                v[u] = (i < N) ? __ldcs(r + i) : -INFINITY;
            }
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) {
                const int i = base + u * kWarp + lane;
                thr = offer_candidates(h, L, v[u], i, i < N, thr, lane);
            }
        }
        if (lane == 0) heap_sort(h, L);
    }
    user_epilogue(h.idx, scratch, K, row, row, tptr, tidx, M, results, ranks, lane);
}

// ----------------------------------------------------------------------------------------
// Kernel B: fused predict (U.V^T, fp32 FMA chain over k) -> train mask -> select -> metrics.
//
// CTA = kWarps warps; each warp owns TM users and, per item tile, each lane owns TN items
// (item = tile_base + n*32 + lane).  The V tile sits in shared memory as [item][dim+4] floats
// (row stride = odd multiple of 16 B => conflict-free LDS.128 by item), the CTA's user rows
// as [user][dim] (LDS.128 broadcast).  Per 4 consecutive k: TN + TM LDS.128 feed 4*TM*TN FFMA.
// Every (user, item) accumulator sees acc = fma(u[k], v[k], acc) for k = 0..dim-1 in order,
// the oracle's definition of the score, so scores are bit-identical to the oracle's.
//
// Train masking: a masked score is -inf and -inf never beats the heap root, so masked items
// only need explicit treatment (a) among the first L items that seed the heap and (b) so
// that they do not pass the threshold test: the warp walks each user's sorted train row in
// step with the item tiles and builds a TN*32-bit mask per tile.
//
// The four steps below are the tile core of both eval_mf_kernel and eval_mf_fast_kernel.
// ----------------------------------------------------------------------------------------

// Stage the CTA's user rows as [kWarps*TM][D4] floats, zero past D (fma(0,0,acc) == acc): batch
// row b < num_eval is user users[row_map ? row_map[b] : b].
template <int TM, int kWarps>
__device__ __forceinline__ void mf_stage_users(float* sU, const float* __restrict__ Utab, int D, int D4,
                                               const int32_t* __restrict__ users,
                                               const int32_t* __restrict__ row_map, int num_eval) {
    for (int idx = threadIdx.x; idx < kWarps * TM * D4; idx += blockDim.x) {
        const int us = idx / D4, k = idx - us * D4;
        const int b = blockIdx.x * (kWarps * TM) + us;
        float val = 0.0f;
        if (b < num_eval && k < D) val = Utab[(size_t)users[row_map ? row_map[b] : b] * D + k];
        sU[idx] = val;
    }
    __syncthreads();
}

// Load the V tile of items [base, base + TN*32) as [item][VS] floats, zero past N and past D
// (coalesced float4 when dim % 4 == 0, scalar otherwise), once the previous tile is consumed.
template <int TN>
__device__ __forceinline__ void mf_load_tile(float* sV, const float* __restrict__ Vtab, int D, int D4, int VS,
                                             int N, int base) {
    constexpr int TILE = TN * 32;
    __syncthreads();  // previous tile fully consumed
    if ((D & 3) == 0) {
        const int q_per_row = D >> 2;
        for (int idx = threadIdx.x; idx < TILE * q_per_row; idx += blockDim.x) {
            const int it = idx / q_per_row, q = idx - it * q_per_row;
            const int item = base + it;
            float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (item < N) val = __ldg(reinterpret_cast<const float4*>(Vtab + (size_t)item * D) + q);
            *reinterpret_cast<float4*>(sV + it * VS + q * 4) = val;
        }
    } else {
        for (int idx = threadIdx.x; idx < TILE * D4; idx += blockDim.x) {
            const int it = idx / D4, k = idx - it * D4;
            const int item = base + it;
            sV[it * VS + k] = (item < N && k < D) ? __ldg(Vtab + (size_t)item * D + k) : 0.0f;
        }
    }
    __syncthreads();
}

// acc[m][n] = score of the warp's user m (row m of su) and the lane's item n*32 + lane of the tile.
template <int TM, int TN>
__device__ __forceinline__ void mf_tile_fma(float (&acc)[TM][TN], const float* su, const float* sV, int D4, int VS,
                                            int lane) {
#pragma unroll
    for (int m = 0; m < TM; ++m)
#pragma unroll
        for (int n = 0; n < TN; ++n) acc[m][n] = 0.0f;
    for (int k = 0; k < D4; k += 4) {
        float4 vv[TN], uu[TM];
#pragma unroll
        for (int n = 0; n < TN; ++n)
            vv[n] = *reinterpret_cast<const float4*>(sV + (n * 32 + lane) * VS + k);
#pragma unroll
        for (int m = 0; m < TM; ++m) uu[m] = *reinterpret_cast<const float4*>(su + m * D4 + k);
#pragma unroll
        for (int m = 0; m < TM; ++m)
#pragma unroll
            for (int n = 0; n < TN; ++n) {
                float a = acc[m][n];
                a = __fmaf_rn(uu[m].x, vv[n].x, a);
                a = __fmaf_rn(uu[m].y, vv[n].y, a);
                a = __fmaf_rn(uu[m].z, vv[n].z, a);
                a = __fmaf_rn(uu[m].w, vv[n].w, a);
                acc[m][n] = a;
            }
    }
}

// Train items of one user inside the tile [base, base + TN*32): item base + n*32 + j sets bit j of
// maskbits[n].  Walks the sorted train row tr[0, tr_len) from tr_pos (>= base there) and advances it.
template <int TN>
__device__ __forceinline__ void mf_tile_mask(unsigned (&maskbits)[TN], const int32_t* __restrict__ tr, int tr_len,
                                             int& tr_pos, int base, int lane) {
    constexpr int TILE = TN * 32;
#pragma unroll
    for (int n = 0; n < TN; ++n) maskbits[n] = 0u;
    for (;;) {
        const int p = tr_pos + lane;
        const int t = (p < tr_len) ? __ldg(tr + p) : INT32_MAX;
        const bool in_tile = t < base + TILE;
        const int off = t - base;  // >= 0 by construction when in_tile
#pragma unroll
        for (int n = 0; n < TN; ++n) {
            const unsigned bit = (in_tile && (off >> 5) == n) ? (1u << (off & 31)) : 0u;
            maskbits[n] |= __reduce_or_sync(kFull, bit);
        }
        const int c = __popc(__ballot_sync(kFull, in_tile));
        tr_pos += c;
        if (c < kWarp) break;
    }
}

template <int TM, int TN, int kWarps>
__global__ void __launch_bounds__(kWarps * 32)
eval_mf_kernel(const float* __restrict__ Utab, const float* __restrict__ Vtab, int D, int N,
               const int32_t* __restrict__ users, int num_eval_arg,
               const int64_t* __restrict__ train_ptr, const int32_t* __restrict__ train_idx,
               const int64_t* __restrict__ test_ptr, const int32_t* __restrict__ test_idx,
               int K, int L, int M, float* __restrict__ results, int32_t* __restrict__ ranks,
               const int32_t* __restrict__ row_map, const int32_t* __restrict__ count_ptr) {
    // row_map / count_ptr (optional): evaluate only the batch rows listed in row_map[0, *count_ptr)
    // -- the users the tie-free fast kernel could not decide.
    constexpr int TILE = TN * 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int num_eval = count_ptr ? *count_ptr : num_eval_arg;
    if ((int)(blockIdx.x * (kWarps * TM)) >= num_eval) return;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int D4 = (D + 3) & ~3;       // padded dim
    const int VS = D4 + 4;             // V tile row stride in floats
    float* sU = reinterpret_cast<float*>(smem_raw);                 // [kWarps*TM][D4]
    float* sV = sU + kWarps * TM * D4;                              // [TILE][VS]
    int* sHeap = reinterpret_cast<int*>(sV + TILE * VS);            // per user 2L+3K words
    auto heap_of = [&](int m) {
        Heap h;
        h.idx = sHeap + (warp * TM + m) * (2 * L + 3 * K);
        h.val = reinterpret_cast<float*>(h.idx + L);
        return h;
    };

    const int user_slot0 = blockIdx.x * (kWarps * TM) + warp * TM;  // first batch row of warp
    mf_stage_users<TM, kWarps>(sU, Utab, D, D4, users, row_map, num_eval);

    // ---- per-user state (warp-uniform) ---------------------------------------------
    int64_t tr_beg[TM];
    int tr_len[TM], tr_pos[TM];
    float thr[TM];
    bool live[TM];
#pragma unroll
    for (int m = 0; m < TM; ++m) {
        const int b = user_slot0 + m;
        live[m] = b < num_eval;
        const int u = live[m] ? users[row_map ? row_map[b] : b] : 0;
        tr_beg[m] = live[m] ? train_ptr[u] : 0;
        tr_len[m] = live[m] ? (int)(train_ptr[u + 1] - tr_beg[m]) : 0;
        tr_pos[m] = 0;
        thr[m] = INFINITY;
    }

    // ---- seed the heaps with items [0, L), masked exactly -----------------------------
#pragma unroll
    for (int m = 0; m < TM; ++m) {
        if (!live[m]) continue;
        const int32_t* tr = train_idx + tr_beg[m];
        int cnt = 0;   // first train position >= L
        for (int p = lane; p < tr_len[m]; p += kWarp) cnt += (__ldg(tr + p) < L);
        tr_pos[m] = __reduce_add_sync(kFull, cnt);
        const float* su = sU + (warp * TM + m) * D4;
        thr[m] = heap_seed(heap_of(m), L, lane, [&](int i) {
            const float* vr = Vtab + (size_t)i * D;
            float acc = 0.0f;
            for (int k = 0; k < D; ++k) acc = __fmaf_rn(su[k], __ldg(vr + k), acc);
            return sorted_contains(tr, tr_len[m], i) ? -INFINITY : acc;
        });
    }

    // ---- main loop over item tiles ---------------------------------------------------
    for (int base = L; base < N; base += TILE) {
        mf_load_tile<TN>(sV, Vtab, D, D4, VS, N, base);
        float acc[TM][TN];
        mf_tile_fma<TM, TN>(acc, sU + warp * TM * D4, sV, D4, VS, lane);
#pragma unroll
        for (int m = 0; m < TM; ++m) {
            if (!live[m]) continue;
            unsigned maskbits[TN];
            mf_tile_mask<TN>(maskbits, train_idx + tr_beg[m], tr_len[m], tr_pos[m], base, lane);
            const Heap h = heap_of(m);
#pragma unroll
            for (int n = 0; n < TN; ++n) {
                const int item = base + n * 32 + lane;
                const bool ok = item < N && !((maskbits[n] >> lane) & 1u);
                thr[m] = offer_candidates(h, L, acc[m][n], item, ok, thr[m], lane);
            }
        }
    }

    // ---- finalise: sort_heap, ranks, metrics ------------------------------------------
#pragma unroll
    for (int m = 0; m < TM; ++m) {
        if (!live[m]) continue;
        const int b = row_map ? row_map[user_slot0 + m] : (user_slot0 + m);
        const Heap h = heap_of(m);
        if (lane == 0) heap_sort(h, L);
        user_epilogue(h.idx, h.idx + 2 * L, K, b, users[b], test_ptr, test_idx, M, results, ranks, lane);
        __syncwarp();
    }
}

// ----------------------------------------------------------------------------------------
// Kernel B-fast: the same fused scoring, but selection WITHOUT the heap replay.
//
// std::partial_sort_copy's output is ambiguous only where scores tie: if the K+1 largest scores
// of a row are pairwise distinct, the first K entries of the reference's ranking are exactly
// those K items in descending score order, whatever the heap did (the heap always holds the L
// largest values; sort_heap orders distinct values uniquely; ties below rank K+1 cannot move
// anything above them).  So each warp keeps, per user, the running top-(K+1) as a sorted list
// spread over its lanes (lane r = rank r; K+1 <= 32): an insertion is one ballot + two
// shuffles instead of ~150 single-lane heap instructions.  At the end the warp checks that the
// K+1 values are strictly decreasing and finite; users that fail the check (exact ties in the
// top K+1, fewer than K+1 unmasked items, or an unmasked NaN among the first L items, which the
// reference's heap holds from the start) are appended to a list and re-done by the exact
// heap-replay kernel above, so the result stays bit-identical to the reference for every input.
// ----------------------------------------------------------------------------------------
template <int TM, int TN, int kWarps>
__global__ void __launch_bounds__(kWarps * 32)
eval_mf_fast_kernel(const float* __restrict__ Utab, const float* __restrict__ Vtab, int D, int N,
                    const int32_t* __restrict__ users, int num_eval,
                    const int64_t* __restrict__ train_ptr, const int32_t* __restrict__ train_idx,
                    const int64_t* __restrict__ test_ptr, const int32_t* __restrict__ test_idx,
                    int K, int M, float* __restrict__ results, int32_t* __restrict__ ranks,
                    int32_t* __restrict__ slow_count, int32_t* __restrict__ slow_rows) {
    constexpr int TILE = TN * 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int D4 = (D + 3) & ~3;
    const int VS = D4 + 4;
    float* sU = reinterpret_cast<float*>(smem_raw);                 // [kWarps*TM][D4]
    float* sV = sU + kWarps * TM * D4;                              // [TILE][VS]
    int* sMet = reinterpret_cast<int*>(sV + TILE * VS);             // per user 4K words
    const int user_slot0 = blockIdx.x * (kWarps * TM) + warp * TM;
    mf_stage_users<TM, kWarps>(sU, Utab, D, D4, users, nullptr, num_eval);

    int64_t tr_beg[TM];
    int tr_len[TM], tr_pos[TM];
    float top_v[TM], thr[TM];   // lane r holds the rank-r entry of user m's running top-(K+1)
    int top_i[TM];
    bool live[TM];
    const int L = (2 * K < N) ? 2 * K : N;   // the reference's heap size (evaluate.h:38)
    unsigned seed_nan = 0u;                  // bit m: user m has an unmasked NaN score in [0, L)
#pragma unroll
    for (int m = 0; m < TM; ++m) {
        const int b = user_slot0 + m;
        live[m] = b < num_eval;
        const int u = live[m] ? users[b] : 0;
        tr_beg[m] = live[m] ? train_ptr[u] : 0;
        tr_len[m] = live[m] ? (int)(train_ptr[u + 1] - tr_beg[m]) : 0;
        tr_pos[m] = 0;
        top_v[m] = -INFINITY;
        top_i[m] = -1;
        thr[m] = -INFINITY;
    }

    for (int base = 0; base < N; base += TILE) {
        mf_load_tile<TN>(sV, Vtab, D, D4, VS, N, base);
        float acc[TM][TN];
        mf_tile_fma<TM, TN>(acc, sU + warp * TM * D4, sV, D4, VS, lane);
#pragma unroll
        for (int m = 0; m < TM; ++m) {
            if (!live[m]) continue;
            unsigned maskbits[TN];
            mf_tile_mask<TN>(maskbits, train_idx + tr_beg[m], tr_len[m], tr_pos[m], base, lane);
            if (base == 0) {   // the heap seed [0, L) lies in the first tile (L <= 62 < TILE)
#pragma unroll
                for (int n = 0; n < TN; ++n) {
                    const int item = n * 32 + lane;
                    if (__any_sync(kFull, item < L && !((maskbits[n] >> lane) & 1u) && isnan(acc[m][n])))
                        seed_nan |= 1u << m;
                }
            }
#pragma unroll
            for (int n = 0; n < TN; ++n) {
                const int item = base + n * 32 + lane;
                const bool ok = item < N && !((maskbits[n] >> lane) & 1u);
                topk_offer(acc[m][n], item, ok, top_v[m], top_i[m], thr[m], K, lane);
            }
        }
    }

#pragma unroll
    for (int m = 0; m < TM; ++m) {
        if (!live[m]) continue;
        const int b = user_slot0 + m;
        if (!topk_decided(top_v[m], (seed_nan >> m) & 1u, K, lane)) {
            if (lane == 0) slow_rows[atomicAdd(slow_count, 1)] = b;
            continue;
        }
        int* rank = sMet + (warp * TM + m) * 4 * K;
        if (lane < K) rank[lane] = top_i[m];
        user_epilogue(rank, rank + K, K, b, users[b], test_ptr, test_idx, M, results, ranks, lane);
        __syncwarp();
    }
}

// np.mean(axis=0) of a C-contiguous [rows, cols] fp32 matrix: numpy adds row after row into
// the fp32 output (no pairwise blocking along a non-contiguous reduction axis), then divides
// by the row count in fp32.  One thread per column, rows in order.
// Block = 256 threads owning 32 columns: tiles of 256 rows x 32 columns are staged through
// shared memory by all threads (many loads in flight), then lanes 0..31 add their column's 256
// values strictly in row order -- the same sequence of fp32 additions as numpy.
constexpr int kMeanTileRows = 128;
__global__ void __launch_bounds__(256)
mean_rows_kernel(const float* __restrict__ a, int64_t rows, int cols, float* __restrict__ out) {
    __shared__ float tile[2][kMeanTileRows][33];
    const int c0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // ty: 8 row groups
    const int c = c0 + tx;
    float acc = 0.0f;
    bool first = true;
    const int64_t n_tiles = (rows + kMeanTileRows - 1) / kMeanTileRows;
    auto load = [&](int buf, int64_t t) {
        const int64_t r0 = t * kMeanTileRows;
#pragma unroll 8
        for (int rr = ty; rr < kMeanTileRows; rr += 8) {
            const int64_t r = r0 + rr;
            tile[buf][rr][tx] = (r < rows && c < cols) ? __ldg(a + r * cols + c) : 0.0f;
        }
    };
    if (n_tiles > 0) load(0, 0);
    __syncthreads();
    for (int64_t t = 0; t < n_tiles; ++t) {
        const int buf = (int)(t & 1);
        if (t + 1 < n_tiles && ty != 0) load(buf ^ 1, t + 1);     // warps 1..7 prefetch
        if (ty == 0) {
            const int64_t r0 = t * kMeanTileRows;
            const int n = (int)((rows - r0 < kMeanTileRows) ? (rows - r0) : kMeanTileRows);
            int rr = 0;
            if (first) { acc = tile[buf][0][tx]; rr = 1; first = false; }
            for (; rr < n; ++rr) acc = __fadd_rn(acc, tile[buf][rr][tx]);
            if (t + 1 < n_tiles) {                                 // warp 0's share of the prefetch
                const int64_t r1 = (t + 1) * kMeanTileRows;
#pragma unroll 8
                for (int q = 0; q < kMeanTileRows; q += 8) {
                    const int64_t r = r1 + q;
                    tile[buf ^ 1][q][tx] = (r < rows && c < cols) ? __ldg(a + r * cols + c) : 0.0f;
                }
            }
        }
        __syncthreads();
    }
    if (ty == 0 && c < cols) out[c] = __fdiv_rn(acc, (float)rows);
}

// A one-column matrix is contiguous along axis 0, and there numpy reduces with its pairwise_sum
// (numpy/_core/src/umath/loops_utils.h.src), starting from 0: below 8 values in order, up to 128
// values in 8 interleaved partial sums, above that split at an even multiple of 8 and add the halves.
__device__ float np_pairwise_leaf(const float* __restrict__ a, int64_t n) {   // n <= 128
    if (n < 8) {
        float r = 0.0f;
        for (int64_t i = 0; i < n; ++i) r = __fadd_rn(r, __ldg(a + i));
        return r;
    }
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __ldg(a + j);
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], __ldg(a + i + j));
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                          __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __fadd_rn(res, __ldg(a + i));
    return res;
}

// The split tree walked without recursion (a recursive kernel's stack would outgrow the default
// per-thread limit on long columns): the left child first, each pending right child's length on an
// explicit stack, a node's sum = left + right as numpy adds them.  Leaves are visited in order, so the
// next subtree always starts where the last leaf ended.  Every split roughly halves n, so the depth
// stays below log2(2^63 / 128) + 2 < 64 for any int64 n (a 768-byte stack frame).
constexpr int kPairwiseDepth = 64;
__device__ float np_pairwise_sum(const float* __restrict__ a, int64_t n) {
    int64_t s_len[kPairwiseDepth];   // length of the pending right child; -1 once it runs
    float s_left[kPairwiseDepth];    // the node's left sum, once known
    int sp = 0;
    int64_t off = 0, len = n;
    for (;;) {
        while (len > 128) {
            int64_t half = len / 2;
            half -= half % 8;
            s_len[sp++] = len - half;
            len = half;
        }
        float r = np_pairwise_leaf(a + off, len);
        off += len;
        for (;;) {
            if (sp == 0) return r;
            if (s_len[sp - 1] >= 0) {
                s_left[sp - 1] = r;
                len = s_len[sp - 1];
                s_len[sp - 1] = -1;
                break;
            }
            r = __fadd_rn(s_left[sp - 1], r);
            --sp;
        }
    }
}

__global__ void mean_column_kernel(const float* __restrict__ a, int64_t rows, float* __restrict__ out) {
    out[0] = __fdiv_rn(np_pairwise_sum(a, rows), (float)rows);
}

static int check_metrics(const int32_t* metric_host, int metric_num) {
    NRC_REQUIRE(metric_num >= 0 && metric_num <= kMaxMetrics, NRC_E_LIMIT,
                "metric_num %d outside [0, %d]", metric_num, kMaxMetrics);
    int ids[kMaxMetrics] = {0};
    for (int i = 0; i < metric_num; ++i) {
        // cpp/uni_evaluator.py:71-73 raises ValueError for an unknown metric
        NRC_REQUIRE(metric_host[i] >= 1 && metric_host[i] <= 5, NRC_E_VALUE,
                    "There is not the metric id '%d'!", metric_host[i]);
        ids[i] = metric_host[i];
    }
    static int cached[kMaxMetrics] = {-1, -1, -1, -1, -1, -1, -1, -1};
    static int cached_dev = -1;
    int dev = 0;
    NRC_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev != cached_dev || memcmp(cached, ids, sizeof(ids)) != 0) {
        cached_dev = dev;
        // a previous launch may still be reading the old ids on another stream
        NRC_CUDA_CHECK(cudaDeviceSynchronize());
        NRC_CUDA_CHECK(cudaMemcpyToSymbol(c_metric, ids, sizeof(ids)));
        memcpy(cached, ids, sizeof(ids));
    }
    return upload_tables();
}

// nrc_eval_last_routes: [0] form of the last nrc_eval_mf, [1] fast pass and [2] warps per CTA of the
// last eval_rows_kernel launch; -1 until a call has decided them.  Process-wide (a test hook), so with
// several host threads it holds whichever thread launched last.
static int32_t g_routes[3] = {-1, -1, -1};

constexpr int kMfWarps = 8;   // warps per CTA of every eval_mf_kernel / eval_mf_fast_kernel form

// Dynamic shared memory of eval_mf_kernel / eval_mf_fast_kernel<TM, TN, kMfWarps>: the CTA's user
// rows, one V tile and user_words per user (heap form: 2L + 3K; tie-free form: 4K).
static size_t mf_smem_bytes(int TM, int TN, int D, int user_words) {
    const size_t D4 = (D + 3) & ~3;
    return ((size_t)kMfWarps * TM * D4 + (size_t)TN * 32 * (D4 + 4) + (size_t)kMfWarps * TM * user_words) * 4;
}

// Dynamic shared-memory limits of every evaluator kernel form launched above 48 KB, once per device.
static int set_smem_limits() {
    static int done_dev = -1;
    int dev = 0;
    NRC_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev == done_dev) return NRC_OK;
    const cudaFuncAttribute a = cudaFuncAttributeMaxDynamicSharedMemorySize;
    NRC_CUDA_CHECK(cudaFuncSetAttribute(eval_rows_kernel<true>, a, 100 * 1024));
    NRC_CUDA_CHECK(cudaFuncSetAttribute(eval_rows_kernel<false>, a, 100 * 1024));
    NRC_CUDA_CHECK(cudaFuncSetAttribute(eval_mf_kernel<8, 2, kMfWarps>, a, 227 * 1024));
    NRC_CUDA_CHECK(cudaFuncSetAttribute(eval_mf_kernel<1, 2, kMfWarps>, a, 227 * 1024));
    NRC_CUDA_CHECK(cudaFuncSetAttribute(eval_mf_fast_kernel<8, 4, kMfWarps>, a, 227 * 1024));
    NRC_CUDA_CHECK(cudaFuncSetAttribute(eval_mf_fast_kernel<8, 2, kMfWarps>, a, 227 * 1024));
    NRC_CUDA_CHECK(cudaFuncSetAttribute(eval_mf_fast_kernel<2, 2, kMfWarps>, a, 227 * 1024));
    done_dev = dev;
    return NRC_OK;
}

static int launch_rows(const float* scores, int N, int rows, int K, int L, const int64_t* tptr,
                       const int32_t* tidx, int M, float* results, int32_t* ranks, bool metrics,
                       cudaStream_t st) {
    if (rows == 0) return NRC_OK;
    int rc = set_smem_limits();
    if (rc) return rc;
    const int stride_bytes = (2 * L + 3 * K) * 4;
    int warps = 8;
    while (warps > 1 && warps * stride_bytes > 96 * 1024) warps >>= 1;
    const size_t smem = (size_t)warps * stride_bytes;
    const int grid = (rows + warps - 1) / warps;
    const int fast = (K + 1 <= 32 && K < N && !g_force_exact) ? 1 : 0;
    g_routes[1] = fast;
    g_routes[2] = warps;
    if (metrics)
        eval_rows_kernel<true><<<grid, warps * 32, smem, st>>>(scores, N, rows, K, L, tptr, tidx, M,
                                                              results, ranks, fast);
    else
        eval_rows_kernel<false><<<grid, warps * 32, smem, st>>>(scores, N, rows, K, L, tptr, tidx,
                                                               M, results, ranks, fast);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

}  // namespace nrc

using namespace nrc;

extern "C" int nrc_eval_score_matrix(const float* scores, int32_t rating_len, int32_t num_users,
                                     const int64_t* test_indptr, const int32_t* test_indices,
                                     const int32_t* metric_host, int32_t metric_num,
                                     int32_t top_k, float* results, int32_t* ranks,
                                     void* stream) {
    NRC_REQUIRE(top_k > 0 && top_k <= kMaxTopK, NRC_E_LIMIT, "top_k %d outside [1, %d]", top_k,
                kMaxTopK);
    NRC_REQUIRE(rating_len >= top_k, NRC_E_VALUE,
                "rating_len (%d) must be >= top_k (%d)", rating_len, top_k);
    NRC_REQUIRE(num_users >= 0, NRC_E_VALUE, "num_users must be >= 0");
    int rc = check_metrics(metric_host, metric_num);
    if (rc) return rc;
    const int L = (2 * top_k < rating_len) ? 2 * top_k : rating_len;  // evaluate.h:38
    return launch_rows(scores, rating_len, num_users, top_k, L, test_indptr, test_indices,
                       metric_num, results, ranks, true, as_stream(stream));
}

extern "C" int nrc_arg_topk(const float* scores, int32_t rating_len, int32_t rows_num,
                            int32_t top_k, int32_t* results, void* stream) {
    NRC_REQUIRE(top_k > 0 && top_k <= 2 * kMaxTopK, NRC_E_LIMIT, "top_k %d outside [1, %d]", top_k,
                2 * kMaxTopK);
    NRC_REQUIRE(rating_len >= top_k, NRC_E_VALUE, "rating_len (%d) must be >= top_k (%d)",
                rating_len, top_k);
    // arg_topk.h:22: exactly top_k slots.  (K = L = top_k; no metric scratch is touched.)
    return launch_rows(scores, rating_len, rows_num, top_k, top_k, nullptr, nullptr, 0, nullptr,
                       results, false, as_stream(stream));
}

// Host-buffer variants: stream row chunks through two device staging buffers.
static int rows_host(const float* scores, int N, int rows, const int64_t* tptr_h,
                     const int32_t* tidx_h, const int32_t* metric_host, int M, int K, int L,
                     float* results_h, int32_t* ranks_h, bool metrics) {
    if (rows == 0) return NRC_OK;
    const size_t row_bytes = (size_t)N * sizeof(float);
    size_t chunk_rows = (64u << 20) / (row_bytes ? row_bytes : 1);
    if (chunk_rows < 1) chunk_rows = 1;
    if (chunk_rows > (size_t)rows) chunk_rows = rows;
    cudaStream_t st[2] = {nullptr, nullptr};
    float* d_scores[2] = {nullptr, nullptr};
    float* d_res[2] = {nullptr, nullptr};
    int32_t* d_rank[2] = {nullptr, nullptr};
    int64_t* d_tptr = nullptr;
    int32_t* d_tidx = nullptr;
    int rc = NRC_OK;
    auto cleanup = [&]() {
        for (int i = 0; i < 2; ++i) {
            if (d_scores[i]) cudaFree(d_scores[i]);
            if (d_res[i]) cudaFree(d_res[i]);
            if (d_rank[i]) cudaFree(d_rank[i]);
        }
        if (d_tptr) cudaFree(d_tptr);
        if (d_tidx) cudaFree(d_tidx);
        if (st[0]) cudaStreamDestroy(st[0]);
        if (st[1]) cudaStreamDestroy(st[1]);
    };
    NRC_CUDA_CHECK(cudaStreamCreateWithFlags(&st[0], cudaStreamNonBlocking));
    NRC_CUDA_CHECK(cudaStreamCreateWithFlags(&st[1], cudaStreamNonBlocking));
#define NRC_TRY(expr)                                                                    \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            set_error("%s failed: %s", #expr, cudaGetErrorString(_e));                   \
            cleanup();                                                                   \
            return NRC_E_CUDA;                                                           \
        }                                                                                \
    } while (0)
    for (int i = 0; i < 2; ++i) {
        NRC_TRY(cudaMalloc(&d_scores[i], chunk_rows * row_bytes));
        if (metrics) NRC_TRY(cudaMalloc(&d_res[i], chunk_rows * (size_t)M * K * sizeof(float)));
        if (ranks_h || !metrics) NRC_TRY(cudaMalloc(&d_rank[i], chunk_rows * (size_t)K * sizeof(int32_t)));
    }
    if (metrics) {
        const int64_t nnz = tptr_h[rows];
        NRC_TRY(cudaMalloc(&d_tptr, (size_t)(rows + 1) * sizeof(int64_t)));
        NRC_TRY(cudaMalloc(&d_tidx, (size_t)(nnz > 0 ? nnz : 1) * sizeof(int32_t)));
        NRC_TRY(cudaMemcpy(d_tptr, tptr_h, (size_t)(rows + 1) * sizeof(int64_t), cudaMemcpyHostToDevice));
        NRC_TRY(cudaMemcpy(d_tidx, tidx_h, (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice));
    }
    int buf = 0;
    for (size_t r0 = 0; r0 < (size_t)rows; r0 += chunk_rows, buf ^= 1) {
        const size_t nr = ((size_t)rows - r0 < chunk_rows) ? (size_t)rows - r0 : chunk_rows;
        NRC_TRY(cudaMemcpyAsync(d_scores[buf], scores + r0 * N, nr * row_bytes, cudaMemcpyHostToDevice, st[buf]));
        rc = launch_rows(d_scores[buf], N, (int)nr, K, L, metrics ? d_tptr + r0 : nullptr, d_tidx, M,
                         d_res[buf], d_rank[buf], metrics, st[buf]);
        if (rc) { cleanup(); return rc; }
        if (metrics)
            NRC_TRY(cudaMemcpyAsync(results_h + r0 * (size_t)M * K, d_res[buf], nr * (size_t)M * K * sizeof(float),
                                    cudaMemcpyDeviceToHost, st[buf]));
        if (ranks_h)
            NRC_TRY(cudaMemcpyAsync(ranks_h + r0 * (size_t)K, d_rank[buf], nr * (size_t)K * sizeof(int32_t),
                                    cudaMemcpyDeviceToHost, st[buf]));
    }
    NRC_TRY(cudaStreamSynchronize(st[0]));
    NRC_TRY(cudaStreamSynchronize(st[1]));
#undef NRC_TRY
    cleanup();
    return NRC_OK;
}

extern "C" int nrc_eval_score_matrix_host(const float* scores, int32_t rating_len,
                                          int32_t num_users, const int64_t* test_indptr,
                                          const int32_t* test_indices, const int32_t* metric_host,
                                          int32_t metric_num, int32_t top_k, float* results,
                                          int32_t* ranks) {
    NRC_REQUIRE(top_k > 0 && top_k <= kMaxTopK, NRC_E_LIMIT, "top_k %d outside [1, %d]", top_k,
                kMaxTopK);
    NRC_REQUIRE(rating_len >= top_k, NRC_E_VALUE, "rating_len (%d) must be >= top_k (%d)",
                rating_len, top_k);
    int rc = check_metrics(metric_host, metric_num);
    if (rc) return rc;
    const int L = (2 * top_k < rating_len) ? 2 * top_k : rating_len;
    return rows_host(scores, rating_len, num_users, test_indptr, test_indices, metric_host,
                     metric_num, top_k, L, results, ranks, true);
}

extern "C" int nrc_arg_topk_host(const float* scores, int32_t rating_len, int32_t rows_num,
                                 int32_t top_k, int32_t* results) {
    NRC_REQUIRE(top_k > 0 && top_k <= 2 * kMaxTopK, NRC_E_LIMIT, "top_k %d outside [1, %d]", top_k,
                2 * kMaxTopK);
    NRC_REQUIRE(rating_len >= top_k, NRC_E_VALUE, "rating_len (%d) must be >= top_k (%d)",
                rating_len, top_k);
    return rows_host(scores, rating_len, rows_num, nullptr, nullptr, nullptr, 0, top_k, top_k,
                     nullptr, results, false);
}

// library-owned list of batch rows the fast kernel could not decide: [count, rows...]
static int32_t* g_slow = nullptr;
static size_t g_slow_cap = 0;
static int32_t* g_und = nullptr;      // tensor-core path: users with ties (second, heap-replay pass)
static size_t g_und_cap = 0;
static int32_t g_last_replays = 0;
static bool g_last_was_tc = false;

// Grows a library-owned list [count, per_user * n words] (with room for larger batches later).
static int grow_list(int32_t*& list, size_t& cap, int n, int per_user) {
    if ((size_t)per_user * n + 1 <= cap) return NRC_OK;
    if (list) NRC_CUDA_CHECK(cudaFree(list));
    list = nullptr;
    cap = 0;
    const size_t c = (size_t)(per_user + 1) * n + 1024;
    NRC_CUDA_CHECK(cudaMalloc(&list, c * sizeof(int32_t)));
    cap = c;
    return NRC_OK;
}

// Full-catalogue heap replay of the batch rows in list = [count, rows...]: eval_mf_kernel with one
// user per warp, so that the few listed users spread over many SMs.
static int launch_mf_replay(const float* U, const float* V, int D, int N, const int32_t* users, int num_eval,
                            const int64_t* train_ptr, const int32_t* train_idx, const int64_t* test_ptr,
                            const int32_t* test_idx, int K, int L, int M, float* results, int32_t* ranks,
                            const int32_t* list, cudaStream_t st) {
    constexpr int TM = 1, TN = 2;
    const int grid = (num_eval + kMfWarps * TM - 1) / (kMfWarps * TM);
    eval_mf_kernel<TM, TN, kMfWarps><<<grid, kMfWarps * 32, mf_smem_bytes(TM, TN, D, 2 * L + 3 * K), st>>>(
        U, V, D, N, users, num_eval, train_ptr, train_idx, test_ptr, test_idx, K, L, M, results, ranks, list + 1,
        list);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// Test hook: 1 = always use the exact heap-replay kernel (no tie-free fast pass).
extern "C" int nrc_eval_force_exact(int32_t on) {
    g_force_exact = on != 0;
    return NRC_OK;
}

// Number of users of the last nrc_eval_mf call that the tie-free pass could not decide (ties
// among the K+1 best scores, or fewer than K+1 unmasked items) and that were re-ranked by the
// heap replay.  Synchronises the device.
extern "C" int nrc_eval_last_undecided(int32_t* count_host) {
    NRC_REQUIRE(count_host != nullptr, NRC_E_VALUE, "count_host is NULL");
    *count_host = 0;
    if (g_slow) NRC_CUDA_CHECK(cudaMemcpy(count_host, g_slow, sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (g_last_was_tc) *count_host += g_last_replays;
    return NRC_OK;
}

// Host bookkeeping of which kernel forms the last calls launched (see g_routes); no device work.
extern "C" int nrc_eval_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "out is NULL");
    for (int i = 0; i < 3; ++i) out[i] = g_routes[i];
    return NRC_OK;
}

// Routes of the last nrc_eval_mf_tc call: users re-ranked by the candidate-list heap replay (ties) and users
// re-ranked by the full-catalogue eval_mf_kernel (an overflowed candidate list in either pass).  The second
// count lives on the device, so this synchronises.
extern "C" int nrc_eval_tc_last_fallbacks(int32_t* replayed, int32_t* full_replays) {
    NRC_REQUIRE(replayed != nullptr && full_replays != nullptr, NRC_E_VALUE, "NULL output");
    NRC_REQUIRE(g_last_was_tc && g_slow != nullptr, NRC_E_VALUE, "the last evaluation was not nrc_eval_mf_tc");
    *replayed = g_last_replays;
    NRC_CUDA_CHECK(cudaDeviceSynchronize());   // whatever stream the call ran on
    NRC_CUDA_CHECK(cudaMemcpy(full_replays, g_slow, sizeof(int32_t), cudaMemcpyDeviceToHost));
    return NRC_OK;
}

extern "C" int nrc_eval_mf(const float* user_table, const float* item_table, int32_t dim,
                           int32_t num_items, const int32_t* users, int32_t num_eval_users,
                           const int64_t* train_indptr, const int32_t* train_indices,
                           const int64_t* test_indptr, const int32_t* test_indices,
                           const int32_t* metric_host, int32_t metric_num, int32_t top_k,
                           float* results, int32_t* ranks, void* stream) {
    NRC_REQUIRE(top_k > 0 && top_k <= kMaxTopK, NRC_E_LIMIT, "top_k %d outside [1, %d]", top_k,
                kMaxTopK);
    NRC_REQUIRE(num_items >= top_k, NRC_E_VALUE, "num_items (%d) must be >= top_k (%d)", num_items,
                top_k);
    NRC_REQUIRE(dim > 0 && dim <= 512, NRC_E_LIMIT, "dim %d outside [1, 512]", dim);
    int rc = check_metrics(metric_host, metric_num);
    if (rc) return rc;
    if (num_eval_users <= 0) return NRC_OK;
    g_last_was_tc = false;
    const int K = top_k;
    const int L = (2 * K < num_items) ? 2 * K : num_items;
    constexpr int TM = 8, W = kMfWarps;
    const size_t smem = mf_smem_bytes(TM, 2, dim, 2 * L + 3 * K);
    NRC_REQUIRE(smem <= 227 * 1024, NRC_E_LIMIT,
                "dim %d / top_k %d need %zu B of shared memory (> 227 KB)", dim, top_k, smem);
    rc = set_smem_limits();
    if (rc) return rc;
    cudaStream_t st = as_stream(stream);
    const int grid = (num_eval_users + W * TM - 1) / (W * TM);
    const bool fast = (K + 1 <= 32) && !g_force_exact;
    if (!fast) {
        g_routes[0] = 0;
        eval_mf_kernel<TM, 2, W><<<grid, W * 32, smem, st>>>(
            user_table, item_table, dim, num_items, users, num_eval_users, train_indptr, train_indices, test_indptr,
            test_indices, K, L, metric_num, results, ranks, nullptr, nullptr);
        NRC_CUDA_CHECK(cudaGetLastError());
        return NRC_OK;
    }
    // tie-free fast pass, then the exact heap replay for the users it could not decide
    rc = grow_list(g_slow, g_slow_cap, num_eval_users, 1);
    if (rc) return rc;
    NRC_CUDA_CHECK(cudaMemsetAsync(g_slow, 0, sizeof(int32_t), st));
    const size_t smem4 = mf_smem_bytes(TM, 4, dim, 4 * K);
    if (num_eval_users <= sm_count() * 16) {   // few users: 2 per warp => 4x the CTAs
        constexpr int TMs = 2;
        g_routes[0] = 1;
        eval_mf_fast_kernel<TMs, 2, W><<<(num_eval_users + W * TMs - 1) / (W * TMs), W * 32,
                                         mf_smem_bytes(TMs, 2, dim, 4 * K), st>>>(
            user_table, item_table, dim, num_items, users, num_eval_users, train_indptr, train_indices,
            test_indptr, test_indices, K, metric_num, results, ranks, g_slow, g_slow + 1);
    } else if (smem4 <= 200 * 1024) {   // 128-item tiles while they fit (measured 15 % faster than 64)
        g_routes[0] = 2;
        eval_mf_fast_kernel<TM, 4, W><<<grid, W * 32, smem4, st>>>(
            user_table, item_table, dim, num_items, users, num_eval_users, train_indptr, train_indices,
            test_indptr, test_indices, K, metric_num, results, ranks, g_slow, g_slow + 1);
    } else {
        g_routes[0] = 3;
        eval_mf_fast_kernel<TM, 2, W><<<grid, W * 32, mf_smem_bytes(TM, 2, dim, 4 * K), st>>>(
            user_table, item_table, dim, num_items, users, num_eval_users, train_indptr, train_indices,
            test_indptr, test_indices, K, metric_num, results, ranks, g_slow, g_slow + 1);
    }
    NRC_CUDA_CHECK(cudaGetLastError());
    return launch_mf_replay(user_table, item_table, dim, num_items, users, num_eval_users, train_indptr,
                            train_indices, test_indptr, test_indices, K, L, metric_num, results, ranks, g_slow, st);
}

namespace nrc {
// uni_evaluator.py:140-143: ranking_score[idx][train_items] = -inf, one warp per batch row.
__global__ void mask_rows_kernel(float* __restrict__ scores, int N, int rows,
                                 const int32_t* __restrict__ users,
                                 const int64_t* __restrict__ tptr,
                                 const int32_t* __restrict__ tidx) {
    const int lane = threadIdx.x & 31;
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= rows) return;
    const int u = users[row];
    const int64_t beg = tptr[u], end = tptr[u + 1];
    for (int64_t p = beg + lane; p < end; p += kWarp) {
        const int it = tidx[p];
        if (it >= 0 && it < N) scores[(size_t)row * N + it] = -INFINITY;
    }
}
}  // namespace nrc

namespace nrc {
// MF.predict / LightGCN.predict (MF.py:120-122, LightGCN.py:187-189) materialised: the same
// fp32 FMA chain over k as the fused evaluator, so predict() returns exactly the scores the
// fused path ranks.  One thread per (row, item); a warp covers 32 consecutive items.
__global__ void mf_scores_kernel(const float* __restrict__ U, const float* __restrict__ V, int D,
                                 int N, const int32_t* __restrict__ users, int rows,
                                 float* __restrict__ out) {
    const int64_t total = (int64_t)rows * N;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total;
         e += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(e / N), i = (int)(e - (int64_t)b * N);
        const float* u = U + (size_t)users[b] * D;
        const float* v = V + (size_t)i * D;
        float acc = 0.0f;
        for (int k = 0; k < D; ++k) acc = __fmaf_rn(__ldg(u + k), __ldg(v + k), acc);
        out[e] = acc;
    }
}
}  // namespace nrc

extern "C" int nrc_mf_scores(const float* user_table, const float* item_table, int32_t dim,
                             int32_t num_items, const int32_t* users, int32_t num_rows,
                             float* scores, void* stream) {
    NRC_REQUIRE(dim > 0 && num_items > 0 && num_rows >= 0, NRC_E_VALUE, "bad shape");
    if (num_rows == 0) return NRC_OK;
    const int64_t total = (int64_t)num_rows * num_items;
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    mf_scores_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(user_table, item_table, dim,
                                                                      num_items, users, num_rows, scores);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_mask_rows(float* scores, int32_t rating_len, int32_t num_rows,
                             const int32_t* users, const int64_t* train_indptr,
                             const int32_t* train_indices, void* stream) {
    NRC_REQUIRE(rating_len > 0 && num_rows >= 0, NRC_E_VALUE, "bad shape");
    if (num_rows == 0) return NRC_OK;
    const int threads = 256;
    const int blocks = (int)(((int64_t)num_rows * 32 + threads - 1) / threads);
    mask_rows_kernel<<<blocks, threads, 0, as_stream(stream)>>>(scores, rating_len, num_rows, users,
                                                                train_indptr, train_indices);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

namespace nrc {
// ----------------------------------------------------------------------------------------
// Finalisation of the tensor-core candidate passes (tc_eval.cu).  One warp per user.
// ----------------------------------------------------------------------------------------

// The oracle's score: fp32 FMA chain over k ascending (D % 4 == 0 on this path).
__device__ __forceinline__ float tc_exact_score(const float4* __restrict__ su4, const float* __restrict__ Vtab,
                                                int item, int D) {
    const float4* v = reinterpret_cast<const float4*>(Vtab + (size_t)item * D);
    float acc = 0.0f;
#pragma unroll 4
    for (int q = 0; q < (D >> 2); ++q) {
        const float4 b = __ldg(v + q);
        const float4 a = su4[q];
        acc = __fmaf_rn(a.x, b.x, acc);
        acc = __fmaf_rn(a.y, b.y, acc);
        acc = __fmaf_rn(a.z, b.z, acc);
        acc = __fmaf_rn(a.w, b.w, acc);
    }
    return acc;
}

// Main pass: exact re-scoring of the user's candidate lists (any order) and the same tie-aware
// selection as eval_mf_fast_kernel.  Users with ties inside the top K+1 go to `und_rows` (second,
// heap-replay pass); users with an overflowed list go to `slow_rows` (full-catalogue heap replay).
__global__ void __launch_bounds__(256)
eval_tc_finalize_kernel(const float* __restrict__ Utab, const float* __restrict__ Vtab, int D,
                        const int32_t* __restrict__ users, int num_eval,
                        const int64_t* __restrict__ test_ptr, const int32_t* __restrict__ test_idx,
                        const int32_t* __restrict__ cand, const int32_t* __restrict__ cand_cnt,
                        const float* __restrict__ cand_val, const float* __restrict__ margin, int nslots, int cap,
                        int K, int L, int M, int force_exact, float* __restrict__ results,
                        int32_t* __restrict__ ranks, int32_t* __restrict__ slow_count,
                        int32_t* __restrict__ slow_rows, int32_t* __restrict__ und_count,
                        int32_t* __restrict__ und_rows) {
    extern __shared__ int smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int row = blockIdx.x * (blockDim.x >> 5) + warp;
    if (row >= num_eval) return;
    float* su = reinterpret_cast<float*>(smem) + warp * ((D + 4 * K + 3) & ~3);   // float4 reads
    int* rank = reinterpret_cast<int*>(su + D);
    const int32_t* ccnt = cand_cnt + (size_t)row * nslots;
    bool overflow = false;
    for (int sl = lane; sl < nslots; sl += kWarp) overflow |= ccnt[sl] > cap;
    if (__any_sync(kFull, overflow)) {
        if (lane == 0) slow_rows[atomicAdd(slow_count, 1)] = row;
        return;
    }
    if (force_exact) {
        if (lane == 0) und_rows[atomicAdd(und_count, 1)] = row;
        return;
    }
    const int u = users[row];
    for (int k = lane; k < D; k += kWarp) su[k] = Utab[(size_t)u * D + k];
    __syncwarp();
    const float4* su4 = reinterpret_cast<const float4*>(su);
    // Phase 1 (no gathers): the (K+1)-th best APPROXIMATE score over all candidates.  Every item of
    // the exact top K+1 has an approximate score >= that value - margin (both the item's score and
    // the order statistic move by at most margin/2 between exact and approximate), so only those
    // candidates -- ~1.4 (K+1) of the ~15 (K+1) in the lists -- need an exact re-score.
    float a_cut = -INFINITY;
    {
        float av = -INFINITY, athr = -INFINITY;
        int ai = -1;
        for (int sl = 0; sl < nslots; ++sl) {
            const int cnt = ccnt[sl];
            const float* arow = cand_val + ((size_t)row * nslots + sl) * cap;
            for (int base = 0; base < cnt; base += kWarp) {
                const int idx = base + lane;
                const float s = (idx < cnt) ? arow[idx] : -INFINITY;
                topk_offer(s, idx, idx < cnt, av, ai, athr, K, lane);
            }
        }
        a_cut = athr - margin[row];     // -inf while fewer than K+1 candidates exist
    }
    // Phase 2: exact fp32 re-score (the oracle's FMA chain) of the survivors, tie-aware selection
    float tv = -INFINITY, thr = -INFINITY;
    int ti = -1;
    for (int sl = 0; sl < nslots; ++sl) {
        const int cnt = ccnt[sl];
        const int32_t* crow = cand + ((size_t)row * nslots + sl) * cap;
        const float* arow = cand_val + ((size_t)row * nslots + sl) * cap;
        for (int base = 0; base < cnt; base += kWarp) {
            const int idx = base + lane;
            const bool keep = idx < cnt && !(arow[idx] < a_cut);
            if (!__any_sync(kFull, keep)) continue;
            const int item = keep ? crow[idx] : -1;
            const float s = keep ? tc_exact_score(su4, Vtab, item, D) : -INFINITY;
            topk_offer<false>(s, item, keep, tv, ti, thr, K, lane);
        }
    }
    // A NaN among the L items that seed the reference's heap reorders it (no comparison with a NaN
    // holds), and neither this selection nor the candidate passes see it: such users take the
    // full-catalogue heap replay.  Masked seeds are not excluded here (-inf in the reference), which
    // only sends a few more users to the exact replay.
    bool seed_nan = false;
    for (int j = lane; j < L; j += kWarp) seed_nan |= isnan(tc_exact_score(su4, Vtab, j, D));
    if (__any_sync(kFull, seed_nan)) {
        if (lane == 0) slow_rows[atomicAdd(slow_count, 1)] = row;
        return;
    }
    if (!topk_decided(tv, false, K, lane)) {
        if (lane == 0) und_rows[atomicAdd(und_count, 1)] = row;
        return;
    }
    if (lane < K) rank[lane] = ti;
    user_epilogue(rank, rank + K, K, row, u, test_ptr, test_idx, M, results, ranks, lane);
}

__global__ void tc_gather_users_kernel(const int32_t* __restrict__ users, const int32_t* __restrict__ rows, int n,
                                       int32_t* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = users[rows[i]];
}

// Replay pass, for the users with ties: the reference's heap (evaluate.h:33-47) replayed over the
// only elements that can change it -- the first L items, which seed it, and the replay pass's
// candidates in ascending item order (lists in slot order), a superset of every later element
// that beats the heap root when offered.  One CTA per user: all warps re-score the candidates
// exactly (scores parked in `scratch`), then warp 0 replays the heap.  `urow[i]` is the row of
// the original call.
__global__ void __launch_bounds__(256)
eval_tc_replay_kernel(const float* __restrict__ Utab, const float* __restrict__ Vtab, int D,
                      const int32_t* __restrict__ users2, const int32_t* __restrict__ urow, int n_und,
                      const int64_t* __restrict__ train_ptr, const int32_t* __restrict__ train_idx,
                      const int64_t* __restrict__ test_ptr, const int32_t* __restrict__ test_idx,
                      const int32_t* __restrict__ cand, const int32_t* __restrict__ cand_cnt,
                      float* __restrict__ scratch, int nslots, int cap,
                      int K, int L, int M, float* __restrict__ results, int32_t* __restrict__ ranks,
                      int32_t* __restrict__ slow_count, int32_t* __restrict__ slow_rows) {
    extern __shared__ int smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i = blockIdx.x;
    const int row = urow[i];
    float* su = reinterpret_cast<float*>(smem);
    Heap h;   // [idx L][val L][epilogue scratch 3K] after the user row
    h.idx = reinterpret_cast<int*>(su + ((D + 3) & ~3));
    h.val = reinterpret_cast<float*>(h.idx + L);
    const int32_t* ccnt = cand_cnt + (size_t)i * nslots;
    bool overflow = false;
    for (int sl = threadIdx.x; sl < nslots; sl += blockDim.x) overflow |= ccnt[sl] > cap;
    if (__syncthreads_or(overflow ? 1 : 0)) {
        if (threadIdx.x == 0) slow_rows[atomicAdd(slow_count, 1)] = row;
        return;
    }
    const int u = users2[i];
    for (int k = threadIdx.x; k < D; k += blockDim.x) su[k] = Utab[(size_t)u * D + k];
    __syncthreads();
    const float4* su4 = reinterpret_cast<const float4*>(su);
    for (int sl = 0; sl < nslots; ++sl) {   // exact scores of every candidate, one per thread
        const int cnt = ccnt[sl];
        const size_t base = ((size_t)i * nslots + sl) * cap;
        for (int idx = threadIdx.x; idx < cnt; idx += blockDim.x) {
            const int item = cand[base + idx];
            scratch[base + idx] = (item >= L) ? tc_exact_score(su4, Vtab, item, D) : -INFINITY;
        }
    }
    __syncthreads();
    if (warp != 0) return;
    const int64_t tr0 = train_ptr[u];
    const int64_t trn = train_ptr[u + 1] - tr0;
    float thr = heap_seed(h, L, lane, [&](int j) {
        const float s = tc_exact_score(su4, Vtab, j, D);
        return sorted_contains(train_idx + tr0, trn, j) ? -INFINITY : s;
    });
    for (int sl = 0; sl < nslots; ++sl) {
        const int cnt = ccnt[sl];
        const size_t base = ((size_t)i * nslots + sl) * cap;
        for (int b0 = 0; b0 < cnt; b0 += kWarp) {
            const int idx = b0 + lane;
            const int item = (idx < cnt) ? cand[base + idx] : -1;
            const bool ok = item >= L;
            const float s = ok ? scratch[base + idx] : -INFINITY;
            thr = offer_candidates(h, L, s, item, ok, thr, lane);
        }
    }
    if (lane == 0) heap_sort(h, L);
    user_epilogue(h.idx, h.idx + 2 * L, K, row, u, test_ptr, test_idx, M, results, ranks, lane);
}
}  // namespace nrc

// nrc_eval_mf with the score step on the tensor cores (wgmma), for large catalogues.
//   pass 0: bf16 candidate pass with the (K+1)-th best score as running threshold -> exact fp32
//           re-scoring -> tie-aware selection -> metrics (users without ties: almost all);
//   pass 1: users with ties only: candidate pass with the reference's heap root (2K-th best) as
//           threshold -> libstdc++ heap replayed over the first 2K items + those candidates;
//   users whose candidate list overflowed: full-catalogue heap replay (eval_mf_kernel).
// Same results as nrc_eval_mf, bit for bit.  Synchronises `stream` once (to size pass 1), so it
// cannot be captured into a CUDA graph.  cand_cap: entries per candidate list (0 = 1024; 2048 above 2^20 items).
extern "C" int nrc_eval_mf_tc(const float* user_table, const float* item_table, int32_t dim,
                              int32_t num_items, const int32_t* users, int32_t num_eval_users,
                              const int64_t* train_indptr, const int32_t* train_indices,
                              const int64_t* test_indptr, const int32_t* test_indices,
                              const int32_t* metric_host, int32_t metric_num, int32_t top_k,
                              int32_t cand_cap, float* results, int32_t* ranks, void* stream) {
    NRC_REQUIRE(top_k > 0 && top_k + 1 <= 32, NRC_E_LIMIT, "the tensor-core path needs top_k in [1, 31]");
    NRC_REQUIRE(num_items > top_k, NRC_E_VALUE, "num_items (%d) must be > top_k (%d)", num_items, top_k);
    // shared memory: 2 user tiles + >= 2 item stages + per-user lists (33 words, 65 for the replay
    // pass when 2*top_k > 32) must fit 227 KB -- dim 192 leaves room for the short lists only
    NRC_REQUIRE(dim == 64 || dim == 128 || (dim == 192 && 2 * top_k <= 32), NRC_E_LIMIT,
                "the tensor-core path supports dim 64, 128 (top_k <= 31) and 192 (top_k <= 16); got dim %d top_k %d",
                dim, top_k);
    int rc = check_metrics(metric_host, metric_num);
    if (rc) return rc;
    if (num_eval_users <= 0) return NRC_OK;
    g_last_was_tc = true;
    const int K = top_k, cap = cand_cap > 0 ? cand_cap : (num_items > (1 << 20) ? 2048 : 1024);
    const int L = (2 * K < num_items) ? 2 * K : num_items;   // evaluate.h:38 heap size
    cudaStream_t st = as_stream(stream);
    rc = tc::prepare_items(item_table, dim, num_items, st);
    if (rc) return rc;
    tc::CandLists c0;
    rc = tc::run_pass(0, user_table, users, num_eval_users, train_indptr, train_indices, K + 1, cap, &c0, st);
    if (rc) return rc;
    // g_slow: [count, rows...] full-catalogue replays; g_und: [count, rows..., gathered user ids...]
    rc = grow_list(g_slow, g_slow_cap, num_eval_users, 1);
    if (rc) return rc;
    rc = grow_list(g_und, g_und_cap, num_eval_users, 2);
    if (rc) return rc;
    NRC_CUDA_CHECK(cudaMemsetAsync(g_slow, 0, sizeof(int32_t), st));
    NRC_CUDA_CHECK(cudaMemsetAsync(g_und, 0, sizeof(int32_t), st));
    const int warps = 8;
    {
        const size_t smem = (size_t)warps * ((dim + 4 * K + 3) & ~3) * 4;
        eval_tc_finalize_kernel<<<(num_eval_users + warps - 1) / warps, warps * 32, smem, st>>>(
            user_table, item_table, dim, users, num_eval_users, test_indptr, test_indices, c0.cand, c0.cnt,
            c0.scratch, c0.margin, c0.nslots, c0.cap, K, L, metric_num, g_force_exact ? 1 : 0, results, ranks, g_slow, g_slow + 1, g_und,
            g_und + 1);
        NRC_CUDA_CHECK(cudaGetLastError());
    }
    int32_t n_und = 0;
    NRC_CUDA_CHECK(cudaMemcpyAsync(&n_und, g_und, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    NRC_CUDA_CHECK(cudaStreamSynchronize(st));
    g_last_replays = n_und;
    if (n_und > 0) {
        int32_t* und_rows = g_und + 1;
        int32_t* users2 = g_und + 1 + num_eval_users;
        tc_gather_users_kernel<<<(n_und + 255) / 256, 256, 0, st>>>(users, und_rows, n_und, users2);
        NRC_CUDA_CHECK(cudaGetLastError());
        tc::CandLists c1;
        rc = tc::run_pass(1, user_table, users2, n_und, train_indptr, train_indices, L, cap > 2048 ? cap : 2048,
                          &c1, st);
        if (rc) return rc;
        const size_t smem = (size_t)(((dim + 3) & ~3) + 2 * L + 3 * K) * 4;
        eval_tc_replay_kernel<<<n_und, 256, smem, st>>>(
            user_table, item_table, dim, users2, und_rows, n_und, train_indptr, train_indices, test_indptr,
            test_indices, c1.cand, c1.cnt, c1.scratch, c1.nslots, c1.cap, K, L, metric_num, results, ranks, g_slow,
            g_slow + 1);
        NRC_CUDA_CHECK(cudaGetLastError());
    }
    // full-catalogue heap replay for users whose candidate list overflowed (rare)
    rc = set_smem_limits();
    if (rc) return rc;
    return launch_mf_replay(user_table, item_table, dim, num_items, users, num_eval_users, train_indptr,
                            train_indices, test_indptr, test_indices, K, L, metric_num, results, ranks, g_slow, st);
}

// ----------------------------------------------------------------------------------------
// Item-sharded evaluation (SURVEY 8e: tables that exceed one GPU).  Every rank scores its own item
// shard (nrc_eval_mf on the shard, top_k + 1 ranks only), re-scores those few candidates exactly
// (nrc_mf_score_pairs), the [B, K+1] (score, global id) lists of all ranks are all-gathered and the
// user's home rank merges them (nrc_eval_merge_candidates).  For a user without exact score ties
// inside its global top K+1 the merged ranking IS the reference's (evaluate.h:23-50: the K largest
// scores in descending order -- each of them is among the K+1 best of its own shard); users with
// such ties are counted (*tie_count) and ranked score-descending, id-ascending (SURVEY 7: the
// reference's own order among equal scores is an artefact of its heap).
// ----------------------------------------------------------------------------------------
namespace nrc {

__global__ void mf_score_pairs_kernel(const float* __restrict__ Urows, const float* __restrict__ V, int D,
                                      const int32_t* __restrict__ items, int C, int64_t total,
                                      const int64_t* __restrict__ train_ptr, const int32_t* __restrict__ train_idx,
                                      float* __restrict__ out) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = e / C;
        const int item = items[e];
        float s = -INFINITY;
        if (item >= 0) {
            const int64_t t0 = train_ptr[b];
            if (!sorted_contains(train_idx + t0, train_ptr[b + 1] - t0, item))
                s = tc_exact_score(reinterpret_cast<const float4*>(Urows + (size_t)b * D), V, item, D);
        }
        out[e] = s;
    }
}

// (score desc, id asc) order on pairs
__device__ __forceinline__ bool pair_before(float sa, int ia, float sb, int ib) {
    return sa > sb || (sa == sb && ia < ib);
}

constexpr int kMergePerLane = 16;   // candidates per lane: C <= 512

__global__ void __launch_bounds__(256)
eval_merge_kernel(const int32_t* __restrict__ cand_ids, const float* __restrict__ cand_scores, int C, int num_rows,
                  const int64_t* __restrict__ test_ptr, const int32_t* __restrict__ test_idx, int K, int M,
                  float* __restrict__ results, int32_t* __restrict__ ranks, int32_t* __restrict__ tie_count) {
    extern __shared__ int smem_i[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const int row = blockIdx.x * wpb + warp;
    if (row >= num_rows) return;
    int* rank = smem_i + warp * 4 * K;
    float sc[kMergePerLane];
    int id[kMergePerLane];
    bool has_nan = false;
#pragma unroll
    for (int q = 0; q < kMergePerLane; ++q) {
        const int c = q * 32 + lane;
        const bool ok = c < C;
        sc[q] = ok ? cand_scores[(size_t)row * C + c] : -INFINITY;
        id[q] = ok ? cand_ids[(size_t)row * C + c] : INT32_MAX;
        if (sc[q] == -INFINITY) id[q] = INT32_MAX;        // masked / padding entries never win a tie
        has_nan |= isnan(sc[q]);
    }
    // a NaN candidate is never picked, but the reference's heap may hold it: the order is not decided
    bool tie = __any_sync(kFull, has_nan);
    float prev = NAN;                                     // equals nothing: a lone +inf at rank 0 is no tie
    for (int r = 0; r <= K; ++r) {                        // K picks + one more to see a tie at the cut
        float bs = -INFINITY; int bi = INT32_MAX, bq = -1;
#pragma unroll
        for (int q = 0; q < kMergePerLane; ++q)
            if (pair_before(sc[q], id[q], bs, bi)) { bs = sc[q]; bi = id[q]; bq = q; }
        float ws = bs; int wi = bi;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float os = __shfl_xor_sync(kFull, ws, o);
            const int oi = __shfl_xor_sync(kFull, wi, o);
            if (pair_before(os, oi, ws, wi)) { ws = os; wi = oi; }
        }
        if (ws == prev || ws == -INFINITY) tie = true;    // equal scores inside the top K+1, or too few items
        prev = ws;
        if (r < K) {
            if (lane == 0) rank[r] = (wi == INT32_MAX) ? -1 : wi;
            if (bq >= 0 && bs == ws && bi == wi) {        // the owner retires its entry
#pragma unroll
                for (int q = 0; q < kMergePerLane; ++q)
                    if (q == bq) { sc[q] = -INFINITY; id[q] = INT32_MAX; }
            }
        }
    }
    __syncwarp();
    if (lane == 0 && tie && tie_count) atomicAdd(tie_count, 1);
    user_epilogue(rank, rank + K, K, row, row, test_ptr, test_idx, M, results, ranks, lane);
}

}  // namespace nrc

// Exact fp32 scores (the FMA chain every evaluator kernel uses) of C candidate items per row:
// user_rows f32 [num_rows, dim] (already gathered), items i32 [num_rows, C] ids INTO item_table
// (-1 = none), train CSR indexed by ROW (not by user id) in the same id space as `items`; a masked or
// missing candidate scores -inf.  out f32 [num_rows, C].
extern "C" int nrc_mf_score_pairs(const float* user_rows, const float* item_table, int32_t dim, const int32_t* items,
                                  int32_t num_rows, int32_t C, const int64_t* train_indptr,
                                  const int32_t* train_indices, float* out, void* stream) {
    NRC_REQUIRE(dim > 0 && dim % 4 == 0, NRC_E_LIMIT, "dim %d must be a positive multiple of 4", dim);
    NRC_REQUIRE(num_rows >= 0 && C > 0, NRC_E_VALUE, "bad shape");
    if (num_rows == 0) return NRC_OK;
    const int64_t total = (int64_t)num_rows * C;
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    mf_score_pairs_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(user_rows, item_table, dim, items, C, total,
                                                                           train_indptr, train_indices, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// Merge of per-shard candidate lists + metrics: cand_ids i32 / cand_scores f32 [num_rows, C] (GLOBAL
// item ids; -inf scores are ignored), test CSR indexed by ROW with global item ids.  results f32
// [num_rows, metric_num * top_k] (metric-major, as nrc_eval_score_matrix), ranks i32 [num_rows, top_k]
// (optional), *tie_count += rows whose top K+1 held equal scores or fewer than K+1 items (optional).
extern "C" int nrc_eval_merge_candidates(const int32_t* cand_ids, const float* cand_scores, int32_t C,
                                         int32_t num_rows, const int64_t* test_indptr, const int32_t* test_indices,
                                         const int32_t* metric_host, int32_t metric_num, int32_t top_k,
                                         float* results, int32_t* ranks, int32_t* tie_count, void* stream) {
    NRC_REQUIRE(top_k > 0 && top_k <= kMaxTopK, NRC_E_LIMIT, "top_k %d outside [1, %d]", top_k, kMaxTopK);
    NRC_REQUIRE(C > top_k && C <= 32 * kMergePerLane, NRC_E_LIMIT, "C = %d candidates per row outside (top_k, %d]", C,
                32 * kMergePerLane);
    int rc = check_metrics(metric_host, metric_num);
    if (rc) return rc;
    if (num_rows <= 0) return NRC_OK;
    int warps = 8;
    while (warps > 1 && (size_t)warps * 4 * top_k * 4 > 96 * 1024) warps >>= 1;
    const size_t smem = (size_t)warps * 4 * top_k * 4;   // above 48 KB from top_k 385 on
    NRC_CUDA_CHECK(cudaFuncSetAttribute(eval_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    eval_merge_kernel<<<(num_rows + warps - 1) / warps, warps * 32, smem, as_stream(stream)>>>(
        cand_ids, cand_scores, C, num_rows, test_indptr, test_indices, top_k, metric_num, results, ranks, tie_count);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_mean_rows(const float* results, int64_t num_rows, int32_t num_cols,
                             float* out, void* stream) {
    NRC_REQUIRE(num_cols >= 0 && num_rows >= 0, NRC_E_VALUE, "negative shape");
    if (num_cols == 0) return NRC_OK;
    if (num_cols == 1) {   // one metric at top_k 1: numpy's pairwise order, one thread
        mean_column_kernel<<<1, 1, 0, as_stream(stream)>>>(results, num_rows, out);
        NRC_CUDA_CHECK(cudaGetLastError());
        return NRC_OK;
    }
    mean_rows_kernel<<<(num_cols + 31) / 32, 256, 0, as_stream(stream)>>>(results, num_rows, num_cols, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}
