// MF-family training step: fused triplet gather -> score -> loss -> gradient accumulation,
// TensorFlow-1.12-faithful optimizer apply, and the per-epoch driver.
//
// Replaces (reference paths):
//   model/general_recommender/MF.py:54-76    _create_inference / _create_loss / _create_optimizer
//   util/learner.py:2-41                     optimizer / pairwise_loss / pointwise_loss
//   util/tool.py:216-217                     l2_loss
//   model/general_recommender/MF.py:92-108   the per-batch sess.run loop of train_model
// and the third-party arithmetic behind them (tensorflow==1.12.3, not vendored):
// embedding_lookup gradients as IndexedSlices, duplicate indices summed before the update
// (optimizer.py::_deduplicate_indexed_slices), Adam applied densely to the whole variable
// (adam.py::_apply_sparse_shared), other optimizers only to the touched rows.
//
// Two phases per step, as TF does (all reads of the pre-step tables happen before any write):
//   phase 1  one warp per triplet/sample: coalesced row gathers, shuffle-reduced dots,
//            row gradients added with RED.ADD into dense accumulators (duplicates sum)
//   phase 2  element-wise optimizer over every table of the model in ONE launch; zeroes the
//            accumulators for the next step.
#include <stdlib.h>

#include "common.cuh"
#include "epoch.cuh"
#include "learner.cuh"
#include "mf.cuh"
#include "mf_routes.cuh"
#include "optim.cuh"

namespace nrc {

int32_t g_mf_routes[kMfKernels][kMfFields] = {{-1, -1, -1, -1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1, -1},
                                              {-1, -1, -1, -1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1, -1},
                                              {-1, -1, -1, -1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1, -1}};

// Phase 1 of a step: one warp per triplet (PAIRWISE: third = negative items) or sample (third = labels' bits).
// The any-dim form of mf_sample_grad, ordinary loads.
template <bool PAIRWISE>
__global__ void __launch_bounds__(256)
mf_grad_kernel(const float* __restrict__ U, const float* __restrict__ V, int D, const int32_t* __restrict__ users,
               const int32_t* __restrict__ items, const int32_t* __restrict__ third, int64_t batch, int loss_kind,
               float reg, float* __restrict__ gU, float* __restrict__ gV, int32_t* __restrict__ tU,
               int32_t* __restrict__ tV, int32_t stamp, float* __restrict__ loss) {
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const int wpb = blockDim.x >> 5;
    const float inv_b = 1.0f / (float)batch;
    float loss_acc = 0.0f;
    for (int64_t b = (int64_t)blockIdx.x * wpb + wib; b < batch; b += (int64_t)gridDim.x * wpb)
        loss_acc += mf_sample_grad<PAIRWISE, 0, false>(U, V, gU, gV, tU, tV, D, reg, loss_kind, lane, users[b], items[b],
                                                       third[b], inv_b, stamp);
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
}

// ----------------------------------------------------------------------------------------
// Large-table path (BASELINE config 5: tables that leave no room for a dense gradient
// accumulator): BPR + plain SGD in ONE pass.  One warp per triplet, lane owns VEC consecutive
// floats of the row (dim = 32*VEC): three coalesced row gathers, two shuffle-reduced dots,
// g = -sigmoid(-x), then `var -= lr * grad` applied in place with vector RED.ADD (float4 /
// float2 atomics, sm_90+), so duplicate rows still accumulate every contribution.  Algorithmic
// traffic: 3 rows read + 3 rows read-modify-written = 24*dim + 12 B per triplet (SURVEY 8d).
// Deviation from TF, by construction: a triplet may read a row another triplet of the same
// batch has already updated ("hogwild inside a batch"); identical to the two-phase step when
// no row repeats inside the batch.
// ----------------------------------------------------------------------------------------
// A table row-sharded over up to 8 GPUs of one NVLink domain: shard r holds rows
// [r*rows_per_shard, (r+1)*rows_per_shard) at base[r]; base[own rank] is local memory, the others
// are peer mappings (CUDA IPC), read with plain loads and updated with RED over NVLink.
struct RowShards {
    float* base[8];
    int32_t rows_per_shard;   // 0: a single local table at base[0]
    int32_t self;             // this rank's shard (rows of other shards live in peer memory)
    int32_t vec_remote;       // how rows of OTHER ranks are updated: 0 scalar REDs, otherwise vector REDs -- NRC_PEER_VEC_RED (default 1)
    int32_t force_remote;     // debug (NRC_FORCE_REMOTE_PATH=1): take the remote update path for local item rows too
    // Replicated head (n_hot > 0): rows [0, n_hot) -- the loader relabels items by descending train degree, so these
    // are the most popular ones -- are READ from this rank's replica `hot` (L2-resident) and their deltas are
    // accumulated into this rank's `hot_delta`; the caller all-reduces hot_delta between steps and applies it
    // (nrc_mf_hot_apply).  Thousands of triplets per step hit the same few rows: without the replica every one of
    // them is a same-address atomic that crosses NVLink to the owner.
    float* hot;
    float* hot_delta;
    int32_t n_hot;
    // SHARDED is a compile-time switch and the shard base is picked with constant indices only, so
    // the struct stays in the kernel-parameter constant bank (a dynamic index would spill it to
    // local memory and cost the single-GPU kernel ~15 % of its bandwidth).
    // row to READ; `upd` receives the address the row's delta is added to (the same row unless it is replicated)
    template <bool SHARDED>
    __device__ __forceinline__ float* row(int32_t id, int D, bool& remote, float*& upd) const {
        if (id < n_hot) {
            remote = false;
            upd = hot_delta + (size_t)id * D;
            return hot + (size_t)id * D;
        }
        float* p = row<SHARDED>(id, D, remote);
        upd = p;
        return p;
    }
    template <bool SHARDED>
    __device__ __forceinline__ float* row(int32_t id, int D, bool& remote) const {
        if constexpr (!SHARDED) {
            remote = force_remote != 0;
            return base[0] + (size_t)id * D;
        } else {
            const int32_t owner = id / rows_per_shard;
            remote = owner != self || force_remote;
            float* b = base[0];
#pragma unroll
            for (int r = 1; r < 8; ++r) b = (owner == r) ? base[r] : b;
            return b + (size_t)(id - owner * rows_per_shard) * D;
        }
    }
};

// In-place row update.  Local rows take one vector RED; rows in peer memory take scalar REDs
// (32-bit float atomics are the form every NVLink generation forwards to the owner's L2).
template <int VEC>
__device__ __forceinline__ void red_row(float* p, const float (&d)[VEC], bool remote) {
    if (remote) {   // scalar form
#pragma unroll
        for (int t = 0; t < VEC; ++t) atomicAdd(p + t, d[t]);
        return;
    }
    red_vec<VEC>(p, d);
}

template <int VEC, bool SHARDED>
__global__ void __launch_bounds__(256)
mf_bpr_sgd_fused_kernel(const RowShards U, const RowShards V, const int32_t* __restrict__ users,
                        const int32_t* __restrict__ pos, const int32_t* __restrict__ neg, int64_t batch,
                        float lr, float reg, float* __restrict__ loss) {
    constexpr int D = 32 * VEC;
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    float loss_acc = 0.0f;
    for (int64_t b = (int64_t)blockIdx.x * wpb + (threadIdx.x >> 5); b < batch; b += (int64_t)gridDim.x * wpb) {
        bool ru, ri, rj;
        float* pu = U.row<SHARDED>(users[b], D, ru) + lane * VEC;
        float* qi = V.row<SHARDED>(pos[b], D, ri) + lane * VEC;
        float* qj = V.row<SHARDED>(neg[b], D, rj) + lane * VEC;
        float a[VEC], bi[VEC], bj[VEC];
        ld_vec<VEC>(pu, a); ld_vec<VEC>(qi, bi); ld_vec<VEC>(qj, bj);
        float di = 0.f, dj = 0.f, sq = 0.f;
#pragma unroll
        for (int t = 0; t < VEC; ++t) {
            di = fmaf(a[t], bi[t], di);
            dj = fmaf(a[t], bj[t], dj);
            sq += a[t] * a[t] + bi[t] * bi[t] + bj[t] * bj[t];
        }
        di = warp_sum(di); dj = warp_sum(dj);
        const float x = di - dj;
        float l = neg_log_sigmoid(x);
        if (reg != 0.0f) l += reg * 0.5f * warp_sum(sq);
        loss_acc += l;
        const float g = neg_log_sigmoid_grad(x);
        float du[VEC], dvi[VEC], dvj[VEC];
#pragma unroll
        for (int t = 0; t < VEC; ++t) {
            du[t] = -lr * (g * (bi[t] - bj[t]) + reg * a[t]);
            dvi[t] = -lr * (g * a[t] + reg * bi[t]);
            dvj[t] = -lr * (-g * a[t] + reg * bj[t]);
        }
        red_row<VEC>(pu, du, ru && U.vec_remote == 0);
        red_row<VEC>(qi, dvi, ri && V.vec_remote == 0);
        red_row<VEC>(qj, dvj, rj && V.vec_remote == 0);
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
}

static int peer_red_mode() {
    static int vec = -1;
    if (vec < 0) { const char* e = getenv("NRC_PEER_VEC_RED"); vec = e ? atoi(e) : 1; }
    return vec;
}

static int launch_bpr_sgd(const RowShards& SU, const RowShards& SV, int dim, const int32_t* users,
                          const int32_t* pos, const int32_t* neg, int64_t batch, float lr, float reg, float* loss,
                          cudaStream_t st) {
    int64_t blocks = (batch + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 8;   // 8 resident CTAs of 256 threads per SM
    const bool capped = blocks > cap;
    if (blocks > cap) blocks = cap;
    const unsigned gb = (unsigned)blocks;
#define NRC_LAUNCH_SGD(VEC, SH) \
    mf_bpr_sgd_fused_kernel<VEC, SH><<<gb, 256, 0, st>>>(SU, SV, users, pos, neg, batch, lr, reg, loss)
    const bool sharded = SU.rows_per_shard != 0;
    mf_route(kMfSgdIds, dim == 128 ? 4 : dim == 64 ? 2 : 1, sharded, -1, -1, blocks, capped, -1);
    if (dim == 128) { if (sharded) NRC_LAUNCH_SGD(4, true); else NRC_LAUNCH_SGD(4, false); }
    else if (dim == 64) { if (sharded) NRC_LAUNCH_SGD(2, true); else NRC_LAUNCH_SGD(2, false); }
    else { if (sharded) NRC_LAUNCH_SGD(1, true); else NRC_LAUNCH_SGD(1, false); }
#undef NRC_LAUNCH_SGD
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// ----------------------------------------------------------------------------------------
// The same single-pass step fed straight from the train CSR: positions [first, first + count) of
// the shuffled epoch (epoch.cuh) are sampled INSIDE the kernel -- no id arrays in HBM, no sampler
// or shuffle pass in front (data/sampler.py:71-90,189-206 + util/data_iterator.py:59 fused in).
// A persistent grid (one 768-thread CTA per SM) splits [first, first + count) evenly;
// a CTA takes its share 768 consecutive positions at a time:
//   phase a  one THREAD per triplet: bijection -> (user, positive) -> Philox rejection draw against
//            the user's sorted row; ~10 dependent loads, 768 chains in flight per CTA.  When the
//            positives are the CSR itself, also whether any other position of the launch visits one
//            of the user's positives (perm^-1 of each: arithmetic only, no loads);
//   phase b  one WARP per triplet, two triplets in flight per warp: row gathers (float4 per lane),
//            shuffle-reduced dots, in-place vector RED.ADD (the hottest head rows: shared memory, below);
//            a user row no other triplet touches gets a plain store of value + delta instead.
// On one H100 vector REDs were as fast as one bulk reduce-add per row (cp.reduce.async.bulk) and need
// no staging buffer (profiles/r3_sgd_breakdown_n1.json).
// User rows are always local (the train CSR is sharded by user owner, SURVEY 8e); item rows may
// live on any rank (RowShards) and are then read / RED-updated over NVLink by the same kernel.
// ----------------------------------------------------------------------------------------

// Rows [0, T) of the replicated head are held in shared memory for the whole launch, T = 32 KB of rows (64 at
// d = 128).  They are the most popular items: at the benchmark's Zipf(1.05) law the top 64 take ~11 % of all row
// updates of a 2^20-triplet step, row 0 alone ~64 000, and every in-place update of one of them is a same-address
// atomic serialised in one L2 slice.  Each CTA reads them from its own copy and sums its deltas with shared-memory
// atomics, so such a row receives one global reduce-add per CTA instead of one per occurrence.
template <int VEC>
constexpr int kSgdTierRows = 8192 / (32 * VEC);
template <int VEC>
constexpr size_t kSgdTierBytes = (size_t)2 * kSgdTierRows<VEC> * 32 * VEC * sizeof(float);   // values + deltas

// an item row into registers: from the shared-memory tier (id < nt) or from global / peer memory
template <int VEC, bool SHARDED>
__device__ __forceinline__ void load_item(const RowShards& V, int32_t id, int nt, const float* s_val, int lane,
                                          float (&v)[VEC]) {
    if (id < nt) {
        ld_vec<VEC>(s_val + id * (32 * VEC) + lane * VEC, v);
    } else {
        bool remote;
        float* upd;
        ld_vec<VEC>(V.row<SHARDED>(id, 32 * VEC, remote, upd) + lane * VEC, v);
    }
}

// an item row's delta: shared-memory atomics into the tier (element lane*VEC + t of the row at t*32 + lane, so the
// 32 lanes hit 32 banks), else vector REDs in place (scalar REDs for peer rows when vec_remote == 0)
template <int VEC, bool SHARDED>
__device__ __forceinline__ void update_item(const RowShards& V, int32_t id, int nt, float* s_dlt, int lane,
                                            const float (&d)[VEC]) {
    if (id < nt) {
#pragma unroll
        for (int t = 0; t < VEC; ++t) atomicAdd(s_dlt + id * (32 * VEC) + t * 32 + lane, d[t]);
    } else {
        bool remote;
        float* upd;
        V.row<SHARDED>(id, 32 * VEC, remote, upd);
        red_row<VEC>(upd + lane * VEC, d, remote && V.vec_remote == 0);
    }
}

// The add a float RED performs (round to nearest, subnormals flushed): never contracted with the multiply that made d
__device__ __forceinline__ float add_as_red(float x, float d) {
    float r;
    asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(x), "f"(d));
    return r;
}

// Positives of a user at most this long are checked for other visits in the launch (one inverse bijection each);
// longer rows always take the RED.
constexpr int64_t kOnceMaxRow = 32;
constexpr int32_t kUserOnce = INT32_MIN;   // bit 31 of s_u: the user row is touched by this triplet alone

// Pairwise sample at shuffled position p (epoch_sample with k = 0, the same bits).  With `user_once`, u carries
// kUserOnce when no other position of [first, first + count) visits one of the user's positives: the positives are CSR
// positions [beg, end) (pos_users is the row expansion of tptr), and the position visiting q is perm^-1(q).
__device__ __forceinline__ void stream_sample(const EpochSpec& E, int64_t p, int64_t first, int64_t count, bool user_once,
                                              int32_t& u, int32_t& item, int32_t& third) {
    const int64_t idx = feistel_perm(E.perm, p);
    u = __ldg(E.users + idx);
    item = __ldg(E.pos + idx);
    const int64_t beg = __ldg(E.tptr + u), end = __ldg(E.tptr + u + 1);
    third = philox_draw_excluding((uint64_t)(idx * E.neg_num), E.seed, E.stream_id, E.num_items, E.tidx + beg, end - beg);
    if (user_once && end - beg <= kOnceMaxRow) {
        bool alone = true;
#pragma unroll 1
        for (int64_t q = beg; q < end; ++q) {
            if (q == idx) continue;
            const int64_t r = feistel_perm_inv(E.perm, q);
            alone &= (uint64_t)(r - first) >= (uint64_t)count;
        }
        if (alone) u |= kUserOnce;
    }
}

// One CTA of 768 threads per SM: one copy of the tier per SM leaves the rest of the SM's shared memory to L1 and flushes
// one set of tier deltas per SM.  On one H100 it measured 3 % faster than three CTAs of 256 threads (three tier copies)
// and than two of 384 or 512 (profiles/r4_sgd_breakdown_n1.json).
constexpr int kStreamThreads = 768;

template <int VEC, bool SHARDED>
__global__ void __launch_bounds__(kStreamThreads, 1)
mf_bpr_sgd_stream_kernel(float* __restrict__ U_local, const RowShards V, const EpochSpec E, int64_t first,
                         int64_t count, int user_once, float lr, float reg, float* __restrict__ loss) {
    constexpr int D = 32 * VEC, CH = kStreamThreads, T = kSgdTierRows<VEC>;
    constexpr int TPW = 2;                     // triplets in flight per warp (3 and 4 measured slower)
    __shared__ int32_t s_u[CH], s_i[CH], s_j[CH];   // s_u: user id | kUserOnce (stream_sample)
    extern __shared__ __align__(16) float s_tier[];
    float* const s_val = s_tier;               // [T][D] pre-step values of head rows [0, nt)
    float* const s_dlt = s_tier + T * D;       // [T][D] this CTA's summed deltas of those rows
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nt = V.n_hot < T ? V.n_hot : T;
    for (int e = threadIdx.x; e < nt * D / 4; e += blockDim.x) {
        reinterpret_cast<float4*>(s_val)[e] = reinterpret_cast<const float4*>(V.hot)[e];
        reinterpret_cast<float4*>(s_dlt)[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    // an even share of [0, count) per CTA of the persistent grid, sampled kStreamThreads positions at a time
    const int64_t lo = count * blockIdx.x / gridDim.x, hi = count * (blockIdx.x + 1) / gridDim.x;
    float loss_acc = 0.0f;
    for (int64_t c0 = lo; c0 < hi; c0 += CH) {
        const int n = (hi - c0 < CH) ? (int)(hi - c0) : CH;
        if ((int)threadIdx.x < n) {
            int32_t u, i, j;
            stream_sample(E, first + c0 + threadIdx.x, first, count, user_once != 0, u, i, j);
            s_u[threadIdx.x] = u; s_i[threadIdx.x] = i; s_j[threadIdx.x] = j;
        }
        __syncthreads();
        // TPW triplets per warp in flight: all 3 * TPW row loads are issued before the first is used
        for (int t0 = warp * TPW; t0 < n; t0 += (kStreamThreads / 32) * TPW) {
            float a[TPW][VEC], b[TPW][VEC], c[TPW][VEC];
#pragma unroll
            for (int k = 0; k < TPW; ++k) {
                const int t = (t0 + k < n) ? t0 + k : t0;
                ld_vec<VEC>(U_local + (size_t)(s_u[t] & ~kUserOnce) * D + lane * VEC, a[k]);
                load_item<VEC, SHARDED>(V, s_i[t], nt, s_val, lane, b[k]);
                load_item<VEC, SHARDED>(V, s_j[t], nt, s_val, lane, c[k]);
            }
            float di[TPW], dj[TPW], sq[TPW];
#pragma unroll
            for (int k = 0; k < TPW; ++k) {
                di[k] = 0.f; dj[k] = 0.f; sq[k] = 0.f;
#pragma unroll
                for (int t = 0; t < VEC; ++t) {
                    di[k] = fmaf(a[k][t], b[k][t], di[k]); dj[k] = fmaf(a[k][t], c[k][t], dj[k]);
                    sq[k] += a[k][t] * a[k][t] + b[k][t] * b[k][t] + c[k][t] * c[k][t];
                }
                di[k] = warp_sum(di[k]); dj[k] = warp_sum(dj[k]);
            }
#pragma unroll
            for (int k = 0; k < TPW; ++k) {
                if (t0 + k >= n) break;
                const int t = t0 + k;
                const float x = di[k] - dj[k];
                float l = neg_log_sigmoid(x);
                if (reg != 0.0f) l += reg * 0.5f * warp_sum(sq[k]);
                loss_acc += l;
                const float g = neg_log_sigmoid_grad(x);
                float du[VEC], dvi[VEC], dvj[VEC];
#pragma unroll
                for (int q = 0; q < VEC; ++q) {
                    du[q] = -lr * (g * (b[k][q] - c[k][q]) + reg * a[k][q]);
                    dvi[q] = -lr * (g * a[k][q] + reg * b[k][q]);
                    dvj[q] = -lr * (-g * a[k][q] + reg * c[k][q]);
                }
                const int32_t su = s_u[t];
                float* const pu = U_local + (size_t)(su & ~kUserOnce) * D + lane * VEC;
                if (su & kUserOnce) {   // no other triplet of the launch reads or writes the row: a + du is what RED leaves
#pragma unroll
                    for (int q = 0; q < VEC; ++q) du[q] = add_as_red(a[k][q], du[q]);
                    st_vec<VEC>(pu, du);
                } else {
                    red_row<VEC>(pu, du, false);
                }
                update_item<VEC, SHARDED>(V, s_i[t], nt, s_dlt, lane, dvi);
                update_item<VEC, SHARDED>(V, s_j[t], nt, s_dlt, lane, dvj);
            }
        }
        __syncthreads();
    }
    __syncthreads();
    // the tier's deltas: one vector RED per row slice into hot_delta (rows this CTA never touched add nothing)
    for (int e = threadIdx.x; e < nt * 32; e += blockDim.x) {
        const int r = e >> 5, l = e & 31;
        float d[VEC];
        bool any = false;
#pragma unroll
        for (int t = 0; t < VEC; ++t) { d[t] = s_dlt[r * D + t * 32 + l]; any |= d[t] != 0.0f; }
        if (any) red_row<VEC>(V.hot_delta + (size_t)r * D + l * VEC, d, false);
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
}

template <int VEC, bool SH>
static int launch_stream(float* U_local, const RowShards& SV, const EpochSpec& E, int64_t first, int64_t count,
                         int user_once, float lr, float reg, float* loss, cudaStream_t st) {
    constexpr size_t smem = kSgdTierBytes<VEC>;
    static int64_t grid_cap = 0;     // the persistent grid: as many CTAs as fit on the device at once
    if (!grid_cap) {
        NRC_CUDA_CHECK(cudaFuncSetAttribute(mf_bpr_sgd_stream_kernel<VEC, SH>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem));
        int per_sm = 0;
        NRC_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mf_bpr_sgd_stream_kernel<VEC, SH>, kStreamThreads, smem));
        NRC_REQUIRE(per_sm > 0, NRC_E_CUDA, "mf_bpr_sgd_stream_kernel does not fit on an SM");
        grid_cap = (int64_t)per_sm * sm_count();
    }
    int64_t blocks = (count + kStreamThreads - 1) / kStreamThreads;
    const bool capped = blocks > grid_cap;
    if (blocks > grid_cap) blocks = grid_cap;
    mf_route(kMfSgdCsr, VEC, SH, user_once, SV.n_hot < kSgdTierRows<VEC> ? SV.n_hot : kSgdTierRows<VEC>, blocks, capped,
             -1);
    mf_bpr_sgd_stream_kernel<VEC, SH><<<(unsigned)blocks, kStreamThreads, smem, st>>>(U_local, SV, E, first, count,
                                                                                      user_once, lr, reg, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

static int launch_bpr_sgd_stream(float* U_local, const RowShards& SV, int dim, const EpochSpec& E, int64_t first,
                                 int64_t count, float lr, float reg, float* loss, cudaStream_t st) {
    const bool sharded = SV.rows_per_shard != 0;
    // user rows touched once are found from the CSR: only when the positives are the CSR itself
    const int user_once = E.pos == E.tidx ? 1 : 0;
#define NRC_STREAM(VEC) (sharded ? launch_stream<VEC, true>(U_local, SV, E, first, count, user_once, lr, reg, loss, st) \
                                 : launch_stream<VEC, false>(U_local, SV, E, first, count, user_once, lr, reg, loss, st))
    if (dim == 128) return NRC_STREAM(4);
    if (dim == 64) return NRC_STREAM(2);
    return NRC_STREAM(1);
#undef NRC_STREAM
}

// ----------------------------------------------------------------------------------------
// The explicitly-named LAZY-Adam variant for tables too large for TF's dense Adam (SURVEY 8d,
// configs[4] "plus an explicitly-named lazy-Adam run"): tf.contrib.opt.LazyAdamOptimizer semantics
// -- only the rows of the batch move:  m = b1*m + (1-b1)*g;  v = b2*v + (1-b2)*g*g;
// var -= lr_t * m / (sqrt(v) + eps) -- applied per TRIPLET in one pass (no batch-wide de-duplication:
// a row that repeats inside the batch is updated once per occurrence by plain loads / stores, so
// concurrent occurrences may overwrite each other; identical to LazyAdam when no row repeats).
// NOT what the reference's learner=adam does (that is dense, optim.cu); never used for parity claims.
// Algorithmic traffic: rows of (var, m, v) read + written for 3 rows = 72*dim + 12 B per triplet.
// ----------------------------------------------------------------------------------------
// one row of (var, m, v) with the slots already in registers: all nine row loads of a triplet are issued together
template <int VEC>
__device__ __forceinline__ void lazy_adam_row(float* var, float* m, float* v, const float (&x)[VEC], float (&mm)[VEC],
                                              float (&vv)[VEC], const float (&g)[VEC], float lr_t, float b1, float b2,
                                              float eps) {
    float out[VEC];
#pragma unroll
    for (int t = 0; t < VEC; ++t) {
        mm[t] = b1 * mm[t] + (1.0f - b1) * g[t];
        vv[t] = b2 * vv[t] + (1.0f - b2) * g[t] * g[t];
        out[t] = x[t] - lr_t * mm[t] / (sqrtf(vv[t]) + eps);
    }
    st_vec<VEC>(m, mm); st_vec<VEC>(v, vv); st_vec<VEC>(var, out);
}

template <int VEC>
__global__ void __launch_bounds__(256, 3)
mf_bpr_lazy_adam_stream_kernel(float* __restrict__ U, float* __restrict__ mU, float* __restrict__ vU, float* __restrict__ V,
                               float* __restrict__ mV, float* __restrict__ vV, const EpochSpec E, int64_t first, int64_t count,
                               float lr_t, float b1, float b2, float eps, float reg, float* __restrict__ loss) {
    constexpr int D = 32 * VEC;
    constexpr int CH = 256;
    __shared__ int32_t s_u[CH], s_i[CH], s_j[CH];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float loss_acc = 0.0f;
    for (int64_t c0 = (int64_t)blockIdx.x * CH; c0 < count; c0 += (int64_t)gridDim.x * CH) {
        const int n = (count - c0 < CH) ? (int)(count - c0) : CH;
        if ((int)threadIdx.x < n) {
            int32_t u, i, j;
            epoch_sample(E, first + c0 + threadIdx.x, 0, u, i, j);
            s_u[threadIdx.x] = u; s_i[threadIdx.x] = i; s_j[threadIdx.x] = j;
        }
        __syncthreads();
        for (int t = warp; t < n; t += 8) {
            const size_t ou = (size_t)s_u[t] * D + lane * VEC, oi = (size_t)s_i[t] * D + lane * VEC,
                         oj = (size_t)s_j[t] * D + lane * VEC;
            // nine independent row loads in flight per triplet (rows of var, m, v of the three ids)
            float a[VEC], bi[VEC], bj[VEC], mu[VEC], vu[VEC], mi[VEC], vi[VEC], mj[VEC], vj[VEC];
            ld_vec<VEC>(U + ou, a); ld_vec<VEC>(V + oi, bi); ld_vec<VEC>(V + oj, bj);
            ld_vec<VEC>(mU + ou, mu); ld_vec<VEC>(vU + ou, vu);
            ld_vec<VEC>(mV + oi, mi); ld_vec<VEC>(vV + oi, vi);
            ld_vec<VEC>(mV + oj, mj); ld_vec<VEC>(vV + oj, vj);
            float di = 0.f, dj = 0.f, sq = 0.f;
#pragma unroll
            for (int c = 0; c < VEC; ++c) {
                di = fmaf(a[c], bi[c], di); dj = fmaf(a[c], bj[c], dj);
                sq += a[c] * a[c] + bi[c] * bi[c] + bj[c] * bj[c];
            }
            di = warp_sum(di); dj = warp_sum(dj);
            const float x = di - dj;
            float l = neg_log_sigmoid(x);
            if (reg != 0.0f) l += reg * 0.5f * warp_sum(sq);
            loss_acc += l;
            const float g = neg_log_sigmoid_grad(x);
            float gu[VEC], gi[VEC], gj[VEC];
#pragma unroll
            for (int c = 0; c < VEC; ++c) {
                gu[c] = g * (bi[c] - bj[c]) + reg * a[c];
                gi[c] = g * a[c] + reg * bi[c];
                gj[c] = -g * a[c] + reg * bj[c];
            }
            lazy_adam_row<VEC>(U + ou, mU + ou, vU + ou, a, mu, vu, gu, lr_t, b1, b2, eps);
            lazy_adam_row<VEC>(V + oi, mV + oi, vV + oi, bi, mi, vi, gi, lr_t, b1, b2, eps);
            lazy_adam_row<VEC>(V + oj, mV + oj, vV + oj, bj, mj, vj, gj, lr_t, b1, b2, eps);
        }
        __syncthreads();
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
}

static int grad_grid(int64_t batch) {
    const int wpb = 8;
    int64_t blocks = (batch + wpb - 1) / wpb;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

}  // namespace nrc

using namespace nrc;

extern "C" int nrc_mf_pairwise_grad(const float* user_table, const float* item_table, int32_t dim,
                                    const int32_t* users, const int32_t* pos_items,
                                    const int32_t* neg_items, int64_t batch, int32_t loss_kind,
                                    float reg, float* grad_user, float* grad_item,
                                    int32_t* touched_user, int32_t* touched_item, int32_t stamp,
                                    float* loss, void* stream) {
    // learner.py:27-28 raises for an unknown loss
    NRC_REQUIRE(loss_kind == NRC_LOSS_BPR || loss_kind == NRC_LOSS_HINGE ||
                    loss_kind == NRC_LOSS_SQUARE,
                NRC_E_VALUE, "please choose a suitable loss function");
    NRC_REQUIRE(dim > 0 && batch >= 0, NRC_E_VALUE, "dim must be positive, batch >= 0");
    if (batch == 0) return NRC_OK;
    mf_route(kMfGrad, 0, 0, -1, -1, grad_grid(batch), (batch + 7) / 8 > (int64_t)sm_count() * 8, -1);
    mf_grad_kernel<true><<<grad_grid(batch), 256, 0, as_stream(stream)>>>(
        user_table, item_table, dim, users, pos_items, neg_items, batch, loss_kind, reg, grad_user,
        grad_item, touched_user, touched_item, stamp, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_mf_pointwise_grad(const float* user_table, const float* item_table, int32_t dim,
                                     const int32_t* users, const int32_t* items,
                                     const float* labels, int64_t batch, int32_t loss_kind,
                                     float reg, float* grad_user, float* grad_item,
                                     int32_t* touched_user, int32_t* touched_item, int32_t stamp,
                                     float* loss, void* stream) {
    // learner.py:39-40
    NRC_REQUIRE(loss_kind == NRC_LOSS_CROSS_ENTROPY || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                "please choose a suitable loss function");
    NRC_REQUIRE(dim > 0 && batch >= 0, NRC_E_VALUE, "dim must be positive, batch >= 0");
    if (batch == 0) return NRC_OK;
    mf_route(kMfGrad, 0, 0, -1, -1, grad_grid(batch), (batch + 7) / 8 > (int64_t)sm_count() * 8, -1);
    mf_grad_kernel<false><<<grad_grid(batch), 256, 0, as_stream(stream)>>>(
        user_table, item_table, dim, users, items, reinterpret_cast<const int32_t*>(labels), batch, loss_kind, reg,
        grad_user, grad_item, touched_user, touched_item, stamp, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_mf_bpr_sgd_fused(float* user_table, float* item_table, int32_t dim,
                                    const int32_t* users, const int32_t* pos_items,
                                    const int32_t* neg_items, int64_t batch, float lr, float reg,
                                    float* loss, void* stream) {
    NRC_REQUIRE(dim == 32 || dim == 64 || dim == 128, NRC_E_LIMIT,
                "the fused single-pass step supports dim 32, 64 or 128 (got %d)", dim);
    NRC_REQUIRE(batch >= 0, NRC_E_VALUE, "batch must be >= 0");
    if (batch == 0) return NRC_OK;
    RowShards SU{}, SV{};
    SU.base[0] = user_table; SV.base[0] = item_table;
    return launch_bpr_sgd(SU, SV, dim, users, pos_items, neg_items, batch, lr, reg, loss, as_stream(stream));
}

// The same single-pass step on ROW-SHARDED tables (BASELINE config 5): every rank runs it on its
// own triplets (users it owns, items anywhere); rows of other ranks are read and updated in place
// through peer memory over NVLink -- gather, score, loss, gradient and the exchange are ONE kernel,
// there is no all-to-all of ids, rows or gradients.
extern "C" int nrc_mf_bpr_sgd_sharded(float* const* user_shards, float* const* item_shards, int32_t world,
                                      int32_t self_rank, int64_t users_per_shard, int64_t items_per_shard, int32_t dim,
                                      const int32_t* users, const int32_t* pos_items, const int32_t* neg_items,
                                      int64_t batch, float lr, float reg, float* loss, void* stream) {
    NRC_REQUIRE(world >= 1 && world <= 8, NRC_E_LIMIT, "world %d outside [1, 8]", world);
    NRC_REQUIRE(self_rank >= 0 && self_rank < world, NRC_E_VALUE, "self_rank %d outside [0, %d)", self_rank, world);
    NRC_REQUIRE(user_shards != nullptr && item_shards != nullptr, NRC_E_VALUE, "shard pointer arrays are NULL");
    NRC_REQUIRE(users_per_shard > 0 && items_per_shard > 0 && users_per_shard < (1ll << 31) &&
                    items_per_shard < (1ll << 31) && users_per_shard * world < (1ll << 31) &&
                    items_per_shard * world < (1ll << 31),
                NRC_E_LIMIT, "global row ids must fit int32");
    NRC_REQUIRE(dim == 32 || dim == 64 || dim == 128, NRC_E_LIMIT, "fused SGD supports dim 32, 64, 128 (got %d)", dim);
    if (batch <= 0) return NRC_OK;
    RowShards SU{}, SV{};
    for (int r = 0; r < world; ++r) {
        NRC_REQUIRE(user_shards[r] != nullptr && item_shards[r] != nullptr, NRC_E_VALUE, "shard %d is NULL", r);
        SU.base[r] = user_shards[r];
        SV.base[r] = item_shards[r];
    }
    SU.rows_per_shard = (int32_t)users_per_shard;
    SV.rows_per_shard = (int32_t)items_per_shard;
    SU.self = SV.self = self_rank;
    SU.vec_remote = SV.vec_remote = peer_red_mode();
    return launch_bpr_sgd(SU, SV, dim, users, pos_items, neg_items, batch, lr, reg, loss, as_stream(stream));
}

// Steps of a BPR + SGD epoch straight from the train CSR: positions [first, first + count) of the
// shuffled epoch `epoch` are sampled, scored and applied by ONE kernel (nrc_epoch_build +
// nrc_mf_bpr_sgd_fused / _sharded without the id arrays in between).  user_table is THIS rank's
// row block (pos_users are local row ids: the train CSR is partitioned by user owner); items are
// global ids, item_shards[r] the row block of rank r (world = 1: the whole table).
extern "C" int nrc_mf_bpr_sgd_epoch_hot(float* user_table, float* const* item_shards, int32_t world, int32_t self_rank,
                                    int64_t items_per_shard, int32_t dim, const int64_t* train_indptr,
                                    const int32_t* train_indices, const int32_t* pos_users, const int32_t* pos_items,
                                    int64_t n_pos, int32_t num_items, int32_t shuffle, uint64_t seed, uint64_t epoch,
                                    int64_t first, int64_t count, float lr, float reg, float* loss, float* hot, float* hot_delta,
                                    int32_t n_hot, void* stream) {
    NRC_REQUIRE(world >= 1 && world <= 8, NRC_E_LIMIT, "world %d outside [1, 8]", world);
    NRC_REQUIRE(self_rank >= 0 && self_rank < world, NRC_E_VALUE, "self_rank %d outside [0, %d)", self_rank, world);
    NRC_REQUIRE(user_table != nullptr && item_shards != nullptr, NRC_E_VALUE, "table pointers are NULL");
    NRC_REQUIRE(dim == 32 || dim == 64 || dim == 128, NRC_E_LIMIT, "fused SGD supports dim 32, 64, 128 (got %d)", dim);
    NRC_REQUIRE(world == 1 || (items_per_shard > 0 && items_per_shard * world < (1ll << 31) &&
                               items_per_shard * world >= num_items),
                NRC_E_VALUE, "items_per_shard %lld x world %d must cover num_items %d and fit int32",
                (long long)items_per_shard, world, num_items);
    EpochSpec E;
    int rc = epoch_spec_init(E, train_indptr, train_indices, pos_users, pos_items, n_pos, 1, num_items, 1, shuffle, seed,
                             epoch);
    if (rc) return rc;
    NRC_REQUIRE(first >= 0 && count >= 0 && first + count <= n_pos, NRC_E_VALUE,
                "[first, first + count) = [%lld, %lld) outside the epoch's %lld triplets", (long long)first,
                (long long)(first + count), (long long)n_pos);
    if (count == 0) return NRC_OK;
    RowShards SV{};
    for (int r = 0; r < world; ++r) {
        NRC_REQUIRE(item_shards[r] != nullptr, NRC_E_VALUE, "item shard %d is NULL", r);
        SV.base[r] = item_shards[r];
    }
    SV.rows_per_shard = world > 1 ? (int32_t)items_per_shard : 0;
    SV.self = self_rank;
    NRC_REQUIRE(n_hot >= 0 && n_hot <= num_items && (n_hot == 0 || (hot != nullptr && hot_delta != nullptr)), NRC_E_VALUE,
                "n_hot %d needs 0 <= n_hot <= num_items and the replica / delta buffers", n_hot);
    SV.hot = hot; SV.hot_delta = hot_delta; SV.n_hot = n_hot;
    {
        static int vec = -1, force = -1;
        if (vec < 0) vec = peer_red_mode();
        if (force < 0) { const char* e = getenv("NRC_FORCE_REMOTE_PATH"); force = e ? atoi(e) : 0; }
        SV.vec_remote = vec;
        SV.force_remote = force;
    }
    return launch_bpr_sgd_stream(user_table, SV, dim, E, first, count, lr, reg, loss, as_stream(stream));
}

extern "C" int nrc_mf_bpr_sgd_epoch(float* user_table, float* const* item_shards, int32_t world, int32_t self_rank,
                                    int64_t items_per_shard, int32_t dim, const int64_t* train_indptr,
                                    const int32_t* train_indices, const int32_t* pos_users, const int32_t* pos_items,
                                    int64_t n_pos, int32_t num_items, int32_t shuffle, uint64_t seed, uint64_t epoch,
                                    int64_t first, int64_t count, float lr, float reg, float* loss, void* stream) {
    return nrc_mf_bpr_sgd_epoch_hot(user_table, item_shards, world, self_rank, items_per_shard, dim, train_indptr,
                                    train_indices, pos_users, pos_items, n_pos, num_items, shuffle, seed, epoch, first,
                                    count, lr, reg, loss, nullptr, nullptr, 0, stream);
}

namespace nrc {
__global__ void __launch_bounds__(256) hot_apply_kernel(float4* __restrict__ hot, float4* __restrict__ delta, int64_t n4) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n4; e += (int64_t)gridDim.x * blockDim.x) {
        float4 h = hot[e];
        const float4 d = delta[e];
        h.x += d.x; h.y += d.y; h.z += d.z; h.w += d.w;
        hot[e] = h;
        delta[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}
}  // namespace nrc

extern "C" int nrc_mf_hot_apply(float* hot, float* hot_delta, int64_t n_floats, void* stream) {
    NRC_REQUIRE(n_floats >= 0 && (n_floats & 3) == 0, NRC_E_VALUE, "n_floats %lld must be a multiple of 4", (long long)n_floats);
    if (n_floats == 0) return NRC_OK;
    NRC_REQUIRE(hot && hot_delta, NRC_E_VALUE, "replica / delta pointers are NULL");
    int64_t blocks = (n_floats / 4 + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    hot_apply_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(reinterpret_cast<float4*>(hot),
                                                                      reinterpret_cast<float4*>(hot_delta), n_floats / 4);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// BPR with LAZY Adam straight from the train CSR (single GPU): the explicitly-named lazy variant of
// nrc_mf_bpr_sgd_epoch for tables where TF's dense Adam pass is out of reach.  lr_t = Adam's
// lr * sqrt(1 - b2^t) / (1 - b1^t) of this step (one value per call = per batch).
extern "C" int nrc_mf_bpr_lazy_adam_epoch(float* user_table, float* user_m, float* user_v, float* item_table, float* item_m,
                                          float* item_v, int32_t dim, const int64_t* train_indptr,
                                          const int32_t* train_indices, const int32_t* pos_users, const int32_t* pos_items,
                                          int64_t n_pos, int32_t num_items, int32_t shuffle, uint64_t seed, uint64_t epoch,
                                          int64_t first, int64_t count, float lr_t, float beta1, float beta2, float eps,
                                          float reg, float* loss, void* stream) {
    NRC_REQUIRE(dim == 32 || dim == 64 || dim == 128, NRC_E_LIMIT, "lazy Adam supports dim 32, 64, 128 (got %d)", dim);
    NRC_REQUIRE(user_table && user_m && user_v && item_table && item_m && item_v, NRC_E_VALUE, "table / slot pointers are NULL");
    EpochSpec E;
    int rc = epoch_spec_init(E, train_indptr, train_indices, pos_users, pos_items, n_pos, 1, num_items, 1, shuffle, seed,
                             epoch);
    if (rc) return rc;
    NRC_REQUIRE(first >= 0 && count >= 0 && first + count <= n_pos, NRC_E_VALUE,
                "[first, first + count) = [%lld, %lld) outside the epoch's %lld triplets", (long long)first,
                (long long)(first + count), (long long)n_pos);
    if (count == 0) return NRC_OK;
    int64_t blocks = (count + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    const bool capped = blocks > cap;
    if (blocks > cap) blocks = cap;
    mf_route(kMfLazyAdam, dim / 32, 0, -1, -1, blocks, capped, -1);
    cudaStream_t st = as_stream(stream);
#define NRC_LAZY(VEC) mf_bpr_lazy_adam_stream_kernel<VEC><<<(unsigned)blocks, 256, 0, st>>>( \
        user_table, user_m, user_v, item_table, item_m, item_v, E, first, count, lr_t, beta1, beta2, eps, reg, loss)
    if (dim == 128) NRC_LAZY(4); else if (dim == 64) NRC_LAZY(2); else NRC_LAZY(1);
#undef NRC_LAZY
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// Host bookkeeping of the routes the most recent MF training launches took (see the header); no device work.
extern "C" int nrc_mf_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "out is NULL");
    for (int k = 0; k < kMfKernels; ++k)
        for (int f = 0; f < kMfFields; ++f) out[k * kMfFields + f] = g_mf_routes[k][f];
    return NRC_OK;
}

// Peer mappings are only usable by kernels of this device after peer access is enabled.
extern "C" int nrc_enable_peer_access(int32_t peer_device) {
    int cur = 0;
    NRC_CUDA_CHECK(cudaGetDevice(&cur));
    if (cur == peer_device) return NRC_OK;
    int can = 0;
    NRC_CUDA_CHECK(cudaDeviceCanAccessPeer(&can, cur, peer_device));
    NRC_REQUIRE(can, NRC_E_CUDA, "device %d cannot access device %d", cur, peer_device);
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return NRC_OK; }
    NRC_CUDA_CHECK(e);
    return NRC_OK;
}

extern "C" int nrc_opt_apply_rows(int32_t opt_kind, float* var, float* grad, float* slot0,
                                  float* slot1, const int32_t* touched, int32_t stamp, int64_t rows,
                                  int32_t dim, const float* hyper_host, void* stream) {
    OptLaunch L;
    int rc = opt_launch_init(L, opt_kind, hyper_host);
    if (rc) return rc;
    rc = opt_launch_add(L, var, grad, slot0, slot1, touched, rows, dim, /*dense_var=*/0);
    if (rc) return rc;
    return opt_launch_run(L, stamp, as_stream(stream));
}

extern "C" int nrc_opt_apply_multi(int32_t opt_kind, int32_t n_vars, float* const* var,
                                   float* const* grad, float* const* slot0, float* const* slot1,
                                   const int32_t* const* touched, const int64_t* rows,
                                   const int32_t* dims, const int32_t* dense_var, int32_t stamp,
                                   const float* hyper_host, void* stream) {
    OptLaunch L;
    int rc = opt_launch_init(L, opt_kind, hyper_host);
    if (rc) return rc;
    for (int i = 0; i < n_vars; ++i) {
        rc = opt_launch_add(L, var[i], grad[i], slot0 ? slot0[i] : nullptr,
                            slot1 ? slot1[i] : nullptr, touched ? touched[i] : nullptr, rows[i],
                            dims[i], dense_var ? dense_var[i] : 0);
        if (rc) return rc;
    }
    return opt_launch_run(L, stamp, as_stream(stream));
}

extern "C" int nrc_mf_train_epoch(float* user_table, float* item_table, int32_t num_users,
                                  int32_t num_items, int32_t dim, const int32_t* users,
                                  const int32_t* items, const void* third, int64_t n,
                                  int32_t batch_size, int32_t pairwise, int32_t loss_kind, float reg,
                                  int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                                  float* grad_user, float* grad_item, int32_t* touched_user,
                                  int32_t* touched_item, float* slot0_user, float* slot1_user,
                                  float* slot0_item, float* slot1_item, int32_t first_stamp,
                                  float* step_loss, void* stream) {
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    NRC_REQUIRE(n >= 0 && dim > 0, NRC_E_VALUE, "n >= 0 and dim > 0 required");
    cudaStream_t st = as_stream(stream);
    const int64_t steps = (n + batch_size - 1) / batch_size;  // sampler.py:208-213
    if (steps == 0) return NRC_OK;
    NRC_CUDA_CHECK(cudaMemsetAsync(step_loss, 0, (size_t)steps * sizeof(float), st));
    float hyper[4] = {hyper_host[0], hyper_host[1], hyper_host[2], hyper_host[3]};
    for (int64_t s = 0; s < steps; ++s) {
        const int64_t off = s * batch_size;
        const int64_t bs = (n - off < batch_size) ? (n - off) : batch_size;
        const int32_t stamp = first_stamp + (int32_t)s;
        int rc;
        if (pairwise)
            rc = nrc_mf_pairwise_grad(user_table, item_table, dim, users + off, items + off,
                                      reinterpret_cast<const int32_t*>(third) + off, bs, loss_kind,
                                      reg, grad_user, grad_item, touched_user, touched_item, stamp,
                                      step_loss + s, stream);
        else
            rc = nrc_mf_pointwise_grad(user_table, item_table, dim, users + off, items + off,
                                       reinterpret_cast<const float*>(third) + off, bs, loss_kind,
                                       reg, grad_user, grad_item, touched_user, touched_item, stamp,
                                       step_loss + s, stream);
        if (rc) return rc;
        if (opt_kind == NRC_OPT_ADAM) hyper[0] = lr_t_host[s];
        OptLaunch L;
        rc = opt_launch_init(L, opt_kind, hyper);
        if (rc) return rc;
        opt_launch_add(L, user_table, grad_user, slot0_user, slot1_user, touched_user, num_users, dim, 0);
        opt_launch_add(L, item_table, grad_item, slot0_item, slot1_item, touched_item, num_items, dim, 0);
        rc = opt_launch_run(L, stamp, st);
        if (rc) return rc;
    }
    return NRC_OK;
}

extern "C" int nrc_mf_train_step_host(float* user_table, float* item_table, int32_t num_users,
                                      int32_t num_items, int32_t dim, const int32_t* users_host,
                                      const int32_t* items_host, const void* third_host,
                                      int64_t batch, int32_t pairwise, int32_t loss_kind, float reg,
                                      int32_t opt_kind, const float* hyper_host, float* grad_user,
                                      float* grad_item, int32_t* touched_user,
                                      int32_t* touched_item, float* slot0_user, float* slot1_user,
                                      float* slot0_item, float* slot1_item, int32_t stamp,
                                      void* staging, float* loss_host, void* stream) {
    NRC_REQUIRE(batch > 0 && dim > 0, NRC_E_VALUE, "batch and dim must be positive");
    cudaStream_t st = as_stream(stream);
    int32_t* d_users = reinterpret_cast<int32_t*>(staging);
    int32_t* d_items = d_users + batch;
    int32_t* d_third = d_items + batch;
    float* d_loss = reinterpret_cast<float*>(d_third + batch);
    const size_t nb = (size_t)batch * sizeof(int32_t);
    NRC_CUDA_CHECK(cudaMemcpyAsync(d_users, users_host, nb, cudaMemcpyHostToDevice, st));
    NRC_CUDA_CHECK(cudaMemcpyAsync(d_items, items_host, nb, cudaMemcpyHostToDevice, st));
    NRC_CUDA_CHECK(cudaMemcpyAsync(d_third, third_host, nb, cudaMemcpyHostToDevice, st));
    NRC_CUDA_CHECK(cudaMemsetAsync(d_loss, 0, sizeof(float), st));
    int rc;
    if (pairwise)
        rc = nrc_mf_pairwise_grad(user_table, item_table, dim, d_users, d_items, d_third, batch,
                                  loss_kind, reg, grad_user, grad_item, touched_user, touched_item,
                                  stamp, d_loss, stream);
    else
        rc = nrc_mf_pointwise_grad(user_table, item_table, dim, d_users, d_items,
                                   reinterpret_cast<const float*>(d_third), batch, loss_kind, reg,
                                   grad_user, grad_item, touched_user, touched_item, stamp, d_loss,
                                   stream);
    if (rc) return rc;
    OptLaunch L;
    rc = opt_launch_init(L, opt_kind, hyper_host);
    if (rc) return rc;
    opt_launch_add(L, user_table, grad_user, slot0_user, slot1_user, touched_user, num_users, dim, 0);
    opt_launch_add(L, item_table, grad_item, slot0_item, slot1_item, touched_item, num_items, dim, 0);
    rc = opt_launch_run(L, stamp, st);
    if (rc) return rc;
    NRC_CUDA_CHECK(cudaMemcpyAsync(loss_host, d_loss, sizeof(float), cudaMemcpyDeviceToHost, st));
    NRC_CUDA_CHECK(cudaStreamSynchronize(st));
    return NRC_OK;
}
