// Negative sampler: counter-based Philox4x32-10 rejection sampling against sorted CSR rows.
//
// Replaces (reference paths):
//   util/cython/random_choice.pyx:12-62   llrand / randint_choice (rejection on libc rand())
//   util/cython/random_choice.pyx:64-89   batch_randint_choice
//   data/sampler.py:71-90                 _sampling_negative_items
//
// The reference's stream (glibc rand(), 5 calls per candidate, data-dependent rejection) is
// inherently serial, so parity here is contractual: each draw is uniform over
// [0, high) \ exclusion(row), independent of every other draw (replace=True) or distinct
// within its row (replace=False).  The k-th candidate of output element e is
//     Philox4x32-10(counter = (e_lo, e_hi, k / 2, stream_lo), key = (seed_lo, seed_hi ^ stream_hi))
// taken as two 64-bit words (k even -> words 0,1; k odd -> words 2,3), reduced `% high`
// exactly like `llrand() % high` (random_choice.pyx:53).  oracle/neurec_oracle.c restates this
// generator on the CPU; tests require bit-equality.
#include "common.cuh"
#include "extras.cuh"
#include "philox.cuh"

namespace nrc {

__global__ void sample_negatives_kernel(const int64_t* __restrict__ tptr,
                                        const int32_t* __restrict__ tidx,
                                        const int32_t* __restrict__ users, int64_t n, int neg_num,
                                        int num_items, uint64_t seed, uint64_t stream_id,
                                        int64_t first_index, int32_t* __restrict__ out) {
    const int64_t total = n * neg_num;
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total;
         e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = e / neg_num;
        const int u = users[p];
        const int64_t beg = tptr[u];
        const int64_t deg = tptr[u + 1] - beg;
        const uint64_t elem = (uint64_t)(first_index * neg_num + e);
        out[e] = philox_draw_excluding(elem, seed, stream_id, num_items, tidx + beg, deg);
    }
}

// replace=True: one thread per output element.
__global__ void batch_choice_replace_kernel(int high, const int64_t* __restrict__ optr, int n_rows,
                                            int64_t total, const int64_t* __restrict__ eptr,
                                            const int32_t* __restrict__ eidx, uint64_t seed,
                                            uint64_t stream_id, int32_t* __restrict__ out) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total;
         e += (int64_t)gridDim.x * blockDim.x) {
        // row = upper_bound(optr, e) - 1
        int lo = 0, hi = n_rows;
        while (lo < hi) {
            int mid = (lo + hi) >> 1;
            if (optr[mid + 1] <= e) lo = mid + 1; else hi = mid;
        }
        const int64_t beg = eptr ? eptr[lo] : 0;
        const int64_t deg = eptr ? eptr[lo + 1] - beg : 0;
        out[e] = philox_draw_excluding((uint64_t)e, seed, stream_id, high, eidx + beg, deg);
    }
}

// replace=False: one thread per row, sequential inside the row (random_choice.pyx:52-58:
// an accepted value joins the omission set).
__global__ void batch_choice_noreplace_kernel(int high, const int64_t* __restrict__ optr,
                                              int n_rows, const int64_t* __restrict__ eptr,
                                              const int32_t* __restrict__ eidx, uint64_t seed,
                                              uint64_t stream_id, int32_t* __restrict__ out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const int64_t o0 = optr[r], o1 = optr[r + 1];
    const int64_t beg = eptr ? eptr[r] : 0;
    const int64_t deg = eptr ? eptr[r + 1] - beg : 0;
    if (high - deg <= (o1 - o0)) {  // random_choice.pyx:36-37 "not enough integers"
        for (int64_t e = o0; e < o1; ++e) out[e] = -1;
        return;
    }
    for (int64_t e = o0; e < o1; ++e) {
        for (uint32_t k = 0;; ++k) {
            const int32_t a = philox_candidate((uint64_t)e, k, seed, stream_id, high);
            if (deg > 0 && sorted_contains(eidx + beg, deg, a)) continue;
            bool dup = false;
            for (int64_t q = o0; q < e; ++q) dup |= (out[q] == a);
            if (dup) continue;
            out[e] = a;
            break;
        }
    }
}

}  // namespace nrc

using namespace nrc;

extern "C" int nrc_sample_negatives(const int64_t* train_indptr, const int32_t* train_indices,
                                    const int32_t* users, int64_t n, int32_t neg_num,
                                    int32_t num_items, uint64_t seed, uint64_t stream_id,
                                    int64_t first_index, int32_t* out, void* stream) {
    // sampler.py:72-73
    NRC_REQUIRE(neg_num > 0, NRC_E_VALUE, "'neg_num' must be a positive integer.");
    NRC_REQUIRE(num_items > 0 && n >= 0, NRC_E_VALUE, "num_items must be positive, n >= 0");
    if (n == 0) return NRC_OK;
    const int64_t total = n * neg_num;
    const int threads = 256;
    int64_t blocks = (total + threads - 1) / threads;
    const int64_t cap = (int64_t)sm_count() * 16;
    const int capped = blocks > cap ? 1 : 0;
    if (blocks > cap) blocks = cap;
    extras_route(kExSampleNegatives, blocks, capped);
    sample_negatives_kernel<<<(unsigned)blocks, threads, 0, as_stream(stream)>>>(
        train_indptr, train_indices, users, n, neg_num, num_items, seed, stream_id, first_index, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_batch_randint_choice(int32_t high, const int64_t* out_indptr, int32_t n_rows,
                                        int64_t total_out, int32_t replace,
                                        const int64_t* excl_indptr, const int32_t* excl_indices,
                                        uint64_t seed, uint64_t stream_id, int32_t* out,
                                        void* stream) {
    NRC_REQUIRE(high > 0, NRC_E_VALUE, "'high' must be positive");
    NRC_REQUIRE(n_rows >= 0 && total_out >= 0, NRC_E_VALUE, "negative shape");
    if (n_rows == 0 || total_out == 0) return NRC_OK;
    const int threads = 256;
    if (replace) {
        int64_t blocks = (total_out + threads - 1) / threads;
        const int64_t cap = (int64_t)sm_count() * 16;
        const int capped = blocks > cap ? 1 : 0;
        if (blocks > cap) blocks = cap;
        extras_route(kExBatchChoice, blocks, capped, -1, -1, -1, 1);
        batch_choice_replace_kernel<<<(unsigned)blocks, threads, 0, as_stream(stream)>>>(
            high, out_indptr, n_rows, total_out, excl_indptr, excl_indices, seed, stream_id, out);
    } else {
        extras_route(kExBatchChoice, (n_rows + threads - 1) / threads, 0, -1, -1, -1, 0);
        batch_choice_noreplace_kernel<<<(n_rows + threads - 1) / threads, threads, 0,
                                        as_stream(stream)>>>(high, out_indptr, n_rows, excl_indptr,
                                                             excl_indices, seed, stream_id, out);
    }
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}
