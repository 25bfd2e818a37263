// One training epoch as a pure function of (train CSR, seed, epoch): shuffled order + negatives.
//
// Replaces (reference paths):
//   util/data_iterator.py:45-63      RandomSampler: np.random.permutation(n) per epoch
//   util/data_iterator.py:133-155    _DataLoaderIter: per-sample python gather + zip transposition
//   data/sampler.py:121-147,189-206  Pointwise/PairwiseSampler.__iter__ (sample, lay out, iterate)
//
// The reference materialises a uniformly random permutation on the host every epoch and gathers
// python lists through it.  Here the order is a keyed BIJECTION of [0, n) evaluated per element
// on the device (no permutation array, no gather pass, nothing on the host):
//
//   perm(p) = cycle-walk of an alternating unbalanced Feistel network over b = max(2, ceil(log2 n))
//   bits, 8 rounds, round function = Philox-style 32x32->64 multiply + xorshift-multiply finisher,
//   round keys = 2 blocks of Philox4x32-10 keyed by (seed, epoch).
//
// Each round maps (L, R) -> (R, L ^ (F(R, k_r) & mask(|L|))), which is invertible for any F and any
// split, so the network permutes [0, 2^b); walking the cycle until the value drops below n
// restricts it to a permutation of [0, n) (expected < 2 evaluations since 2^b < 2n).  Parity with
// the reference is contractual (every sample exactly once per epoch, a different order every
// epoch, position statistics of a random permutation -- tests/test_epoch.py); the CPU restatement
// oracle/neurec_oracle.c::orc_feistel_* must agree bit for bit.
#pragma once
#include "common.cuh"
#include "philox.cuh"

namespace nrc {

constexpr int kFeistelRounds = 8;

struct Feistel {
    uint32_t key[kFeistelRounds];
    uint64_t n;          // domain size; perm is the identity when shuffle == 0
    int32_t bits_l;      // bits of the left half before round 0 (floor(b/2))
    int32_t bits_r;      // bits of the right half before round 0 (b - bits_l)
    int32_t shuffle;
};

__host__ __device__ __forceinline__ uint32_t feistel_mix(uint32_t r, uint32_t key) {
    const uint32_t v = r ^ key;
    const uint64_t prod = (uint64_t)0xD2511F53u * v;
    uint32_t f = (uint32_t)(prod >> 32) ^ (uint32_t)prod;
    f = (f ^ (f >> 15)) * 0x9E3779B1u;
    return f ^ (f >> 13);
}

__host__ __device__ __forceinline__ uint64_t feistel_once(const Feistel& F, uint64_t x) {
    int bl = F.bits_l, br = F.bits_r;
    uint32_t L = (uint32_t)(x >> br), R = (uint32_t)(x & ((1ull << br) - 1ull));
#pragma unroll
    for (int r = 0; r < kFeistelRounds; ++r) {
        const uint32_t nr = L ^ (feistel_mix(R, F.key[r]) & (uint32_t)((1ull << bl) - 1ull));
        L = R; R = nr;
        const int t = bl; bl = br; br = t;
    }
    return ((uint64_t)L << br) | R;
}

__host__ __device__ __forceinline__ int64_t feistel_perm(const Feistel& F, int64_t p) {
    if (!F.shuffle) return p;
    uint64_t x = (uint64_t)p;
    do { x = feistel_once(F, x); } while (x >= F.n);
    return (int64_t)x;
}

// The network run backwards: round r maps (L, R) back to (R ^ (F(L, k_r) & mask(|R|)), L).  After an even number of
// rounds the halves have their initial widths again, so the output splits as the input did.
static_assert(kFeistelRounds % 2 == 0, "feistel_once_inv assumes the halves end at their initial widths");
__host__ __device__ __forceinline__ uint64_t feistel_once_inv(const Feistel& F, uint64_t x) {
    int bl = F.bits_l, br = F.bits_r;
    uint32_t L = (uint32_t)(x >> br), R = (uint32_t)(x & ((1ull << br) - 1ull));
#pragma unroll
    for (int r = kFeistelRounds - 1; r >= 0; --r) {
        const uint32_t pl = R ^ (feistel_mix(L, F.key[r]) & (uint32_t)((1ull << br) - 1ull));
        R = L; L = pl;
        const int t = bl; bl = br; br = t;
    }
    return ((uint64_t)L << br) | R;
}

// perm^-1: the shuffled position at which unshuffled index q is visited (walks the cycle backwards)
__host__ __device__ __forceinline__ int64_t feistel_perm_inv(const Feistel& F, int64_t q) {
    if (!F.shuffle) return q;
    uint64_t x = (uint64_t)q;
    do { x = feistel_once_inv(F, x); } while (x >= F.n);
    return (int64_t)x;
}

// What an epoch is made of (all device pointers).
struct EpochSpec {
    const int64_t* tptr;    // train CSR row pointers [num_users + 1]
    const int32_t* tidx;    // train CSR items, ascending per row
    const int32_t* users;   // flattened positives: user of positive q    (data/sampler.py:24-39)
    const int32_t* pos;     // flattened positives: item of positive q
    int64_t n_pos;
    int64_t n_samples;      // pairwise: n_pos; pointwise: n_pos * (neg_num + 1)
    int32_t neg_num;
    int32_t num_items;
    int32_t pairwise;
    uint64_t seed, stream_id;   // negative-sampler stream (sampler.cu)
    Feistel perm;
};

// Sample at shuffled position p.
//   pairwise : (user, positive item, k-th negative of that positive)      sampler.py:189-206
//   pointwise: positions [0, n_pos) of the unshuffled layout are the positives (label 1.0), then
//              the k-th negatives of all positives, k-major (sampler.py:139-141 transposes the
//              negative array before flattening), label 0.0                 sampler.py:121-147
__device__ __forceinline__ void epoch_sample(const EpochSpec& E, int64_t p, int k, int32_t& u, int32_t& item,
                                             int32_t& third) {
    const int64_t idx = feistel_perm(E.perm, p);
    if (E.pairwise) {
        u = __ldg(E.users + idx);
        item = __ldg(E.pos + idx);
        const int64_t beg = __ldg(E.tptr + u);
        third = philox_draw_excluding((uint64_t)(idx * E.neg_num + k), E.seed, E.stream_id, E.num_items,
                                      E.tidx + beg, __ldg(E.tptr + u + 1) - beg);
    } else if (idx < E.n_pos) {
        u = __ldg(E.users + idx);
        item = __ldg(E.pos + idx);
        third = __float_as_int(1.0f);
    } else {
        const int64_t t = idx - E.n_pos;
        const int64_t kk = t / E.n_pos, q = t - kk * E.n_pos;
        u = __ldg(E.users + q);
        const int64_t beg = __ldg(E.tptr + u);
        item = philox_draw_excluding((uint64_t)(q * E.neg_num + kk), E.seed, E.stream_id, E.num_items,
                                     E.tidx + beg, __ldg(E.tptr + u + 1) - beg);
        third = __float_as_int(0.0f);
    }
}

// host side (epoch.cu)
int feistel_init(Feistel& F, int64_t n, int shuffle, uint64_t seed, uint64_t epoch);
int epoch_spec_init(EpochSpec& E, const int64_t* tptr, const int32_t* tidx, const int32_t* users, const int32_t* pos,
                    int64_t n_pos, int32_t neg_num, int32_t num_items, int32_t pairwise, int32_t shuffle,
                    uint64_t seed, uint64_t stream_id);

// Grid-wide barrier of a cooperative launch (all CTAs co-resident).  `counter` counts arrivals
// monotonically from 0 at kernel start; the k-th barrier completes when it reaches k * gridDim.x.
// bar.sync orders every thread's earlier writes / REDs before thread 0's release-arrive (fence
// cumulativity); thread 0's acquire-load polling orders them before every later read of the CTA.
__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int& target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        target += gridDim.x;
        unsigned int seen;
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
        } while (seen < target);
    }
    __syncthreads();
}

}  // namespace nrc
