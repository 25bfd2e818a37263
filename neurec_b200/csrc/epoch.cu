// The device-resident training epoch: shuffle + negative sampling + every step of the epoch in
// ONE launch (MF family), and the stand-alone epoch builder the other models chain in front of
// their step kernels.
//
// Replaces (reference paths):
//   util/data_iterator.py:45-63,133-155   np.random.permutation + per-sample python batching
//   data/sampler.py:71-90,121-147,189-206 per-epoch negative sampling and batch layout
//   model/general_recommender/MF.py:92-108 the `for batch: sess.run((loss, optimizer))` loop
//
// nrc_mf_epoch_fused is a persistent cooperative kernel (one 512-thread CTA per SM, all
// co-resident): phase A materialises the epoch's (user, item, third) arrays through the keyed
// bijection of epoch.cuh with the Philox rejection sampler fused in; then, per step,
//   phase 1  warp per triplet: row gathers (lane owns dim/32 consecutive floats), shuffle-reduced
//            dots, loss, gradients added into the dense accumulators with vector RED.ADD,
//   grid barrier,
//   phase 2  TensorFlow-1.12 optimizer over BOTH tables (float4 per thread; Adam is dense, TF's
//            _apply_sparse_shared), accumulators zeroed,
//   grid barrier.
// Two barriers per step keep TF's semantics with each phase a plain pass over its data: every
// gradient read sees the pre-step tables, and Adam moves every row every step.  The tables (0.7 MB for ml-100k) stay in
// L2; a step costs two barrier round trips plus ~1 us of latency-bound work instead of two
// kernel launches and their gaps.
#include "epoch.cuh"
#include "mf.cuh"
#include "mf_routes.cuh"
#include "optim.cuh"

#include <cooperative_groups.h>

namespace nrc {

// ------------------------------------------------------------------------------ host side
static void philox4x32_10_host(uint32_t c[4], uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)M0 * c[0], p1 = (uint64_t)M1 * c[2];
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0, n1 = (uint32_t)p1;
        const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1, n3 = (uint32_t)p0;
        c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
        k0 += W0; k1 += W1;
    }
}

int feistel_init(Feistel& F, int64_t n, int shuffle, uint64_t seed, uint64_t epoch) {
    NRC_REQUIRE(n >= 0 && n < (1ll << 62), NRC_E_LIMIT, "shuffle domain %lld outside [0, 2^62)", (long long)n);
    int b = 2;
    while (b < 62 && (1ull << b) < (uint64_t)n) ++b;
    F.n = (uint64_t)n;
    F.bits_l = b / 2;
    F.bits_r = b - b / 2;
    F.shuffle = (shuffle && n > 1) ? 1 : 0;
    for (uint32_t blk = 0; blk < kFeistelRounds / 4; ++blk) {
        uint32_t c[4] = {(uint32_t)epoch, (uint32_t)(epoch >> 32), 0x5348464Cu /* 'SHFL' */, blk};
        philox4x32_10_host(c, (uint32_t)seed, (uint32_t)(seed >> 32));
        for (int j = 0; j < 4; ++j) F.key[blk * 4 + j] = c[j];
    }
    return NRC_OK;
}

int epoch_spec_init(EpochSpec& E, const int64_t* tptr, const int32_t* tidx, const int32_t* users, const int32_t* pos,
                    int64_t n_pos, int32_t neg_num, int32_t num_items, int32_t pairwise, int32_t shuffle,
                    uint64_t seed, uint64_t stream_id) {
    // sampler.py:117-118,185-186
    NRC_REQUIRE(neg_num > 0, NRC_E_VALUE, "'neg_num' must be a positive integer.");
    NRC_REQUIRE(num_items > 0 && n_pos >= 0, NRC_E_VALUE, "num_items must be positive, n_pos >= 0");
    E.tptr = tptr; E.tidx = tidx; E.users = users; E.pos = pos;
    E.n_pos = n_pos;
    E.n_samples = pairwise ? n_pos : n_pos * (int64_t)(neg_num + 1);
    E.neg_num = neg_num; E.num_items = num_items; E.pairwise = pairwise ? 1 : 0;
    E.seed = seed; E.stream_id = stream_id;
    return feistel_init(E.perm, E.n_samples, shuffle, seed, stream_id);
}

// ------------------------------------------------------------------------------ kernels
__global__ void shuffle_perm_kernel(const Feistel F, int64_t n, int64_t* __restrict__ out) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
        out[p] = feistel_perm(F, p);
}

// third: pairwise -> int32 [n_out, neg_num] negatives; pointwise -> f32 [n_out] labels
__global__ void epoch_build_kernel(const EpochSpec E, int64_t first, int64_t n_out, int32_t* __restrict__ out_users,
                                   int32_t* __restrict__ out_items, int32_t* __restrict__ out_third) {
    const int kn = E.pairwise ? E.neg_num : 1;
    const int64_t total = n_out * kn;
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = e / kn;
        const int k = (int)(e - p * kn);
        int32_t u, it, th;
        epoch_sample(E, first + p, k, u, it, th);
        if (k == 0) { out_users[p] = u; out_items[p] = it; }
        out_third[e] = th;
    }
}

struct MfEpochParams {
    EpochSpec E;
    float* U; float* V;
    float* gU; float* gV;
    int32_t* tU; int32_t* tV;
    float* s0U; float* s1U; float* s0V; float* s1V;
    int32_t* ws_u; int32_t* ws_i; int32_t* ws_t;
    float* step_loss;
    float* adam_pows;           // device [2]: beta1^t, beta2^t of the NEXT step (fp32, TF's beta-power variables)
    unsigned int* barrier;
    int64_t n_used;             // samples consumed per epoch (drop_last trims the tail)
    int64_t first_step, num_steps, steps_total;
    int32_t num_users, num_items, D, batch_size;
    int32_t loss_kind, opt_kind, first_stamp, build;
    float reg, h0, h1, h2, h3;
};

template <bool PAIRWISE, int VEC>
__global__ void __launch_bounds__(512, 1) mf_epoch_kernel(const MfEpochParams P) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_g = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nthr = (int64_t)gridDim.x * blockDim.x;
    unsigned int target = 0;

    if (P.build) {   // phase A: this epoch's shuffled samples with their negatives
        for (int64_t p = tid; p < P.n_used; p += nthr) {
            int32_t u, it, th;
            epoch_sample(P.E, p, 0, u, it, th);
            P.ws_u[p] = u; P.ws_i[p] = it; P.ws_t[p] = th;
        }
        for (int64_t s = tid; s < P.steps_total; s += nthr) P.step_loss[s] = 0.0f;
        grid_barrier(P.barrier, target);
    }

    // TF keeps beta1^t / beta2^t as fp32 variables multiplied once per step (adam.py::_finish)
    const bool adam = P.opt_kind == NRC_OPT_ADAM;
    float p1 = 0.0f, p2 = 0.0f;
    if (adam) { p1 = __ldcg(P.adam_pows); p2 = __ldcg(P.adam_pows + 1); }
    const bool has0 = P.opt_kind != NRC_OPT_GD;
    const bool has1 = adam || P.opt_kind == NRC_OPT_RMSPROP;
    const int D = P.D;
    const int64_t eU = (int64_t)P.num_users * D, eAll = eU + (int64_t)P.num_items * D;

    for (int64_t s = P.first_step; s < P.first_step + P.num_steps; ++s) {
        const int64_t off = s * P.batch_size;
        const int64_t cnt = (P.n_used - off < P.batch_size) ? (P.n_used - off) : P.batch_size;
        const int32_t stamp = P.first_stamp + (int32_t)(s - P.first_step);
        // ---- phase 1: gradients of the batch
        const float inv_b = 1.0f / (float)cnt;
        float loss_acc = 0.0f;
        for (int64_t b = warp_g; b < cnt; b += warps) {
            const int32_t u = __ldcg(P.ws_u + off + b), i = __ldcg(P.ws_i + off + b), t = __ldcg(P.ws_t + off + b);
            loss_acc += mf_sample_grad<PAIRWISE, VEC, true>(P.U, P.V, P.gU, P.gV, P.tU, P.tV, D, P.reg, P.loss_kind, lane,
                                                            u, i, t, inv_b, stamp);
        }
        if (lane == 0 && warp_g < cnt) atomicAdd(P.step_loss + s, loss_acc);
        grid_barrier(P.barrier, target);
        // ---- phase 2: optimizer over both tables
        float h0 = P.h0;
        if (adam) {   // lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t), fp32 (adam.py::_prepare)
            h0 = __fdiv_rn(__fmul_rn(P.h0, __fsqrt_rn(__fsub_rn(1.0f, p2))), __fsub_rn(1.0f, p1));
            p1 = __fmul_rn(p1, P.h1);
            p2 = __fmul_rn(p2, P.h2);
        }
        if ((D & 3) == 0) {
            for (int64_t e = tid * 4; e < eAll; e += nthr * 4) {
                const bool isU = e < eU;
                const int64_t i = isU ? e : e - eU;
                float* var = (isU ? P.U : P.V) + i;
                float* grd = (isU ? P.gU : P.gV) + i;
                float* s0p = (isU ? P.s0U : P.s0V) + i;
                float* s1p = (isU ? P.s1U : P.s1V) + i;
                const int32_t* tch = isU ? P.tU : P.tV;
                const float4 g = __ldcg(reinterpret_cast<const float4*>(grd));
                float4 v = __ldcg(reinterpret_cast<const float4*>(var));
                float4 a = has0 ? __ldcg(reinterpret_cast<const float4*>(s0p)) : make_float4(0.f, 0.f, 0.f, 0.f);
                float4 c = has1 ? __ldcg(reinterpret_cast<const float4*>(s1p)) : make_float4(0.f, 0.f, 0.f, 0.f);
                const bool touched = (adam || P.opt_kind == NRC_OPT_GD) ? true : (__ldcg(tch + i / D) == stamp);
                opt_update(P.opt_kind, 0, touched, h0, P.h1, P.h2, P.h3, v.x, g.x, a.x, c.x);
                opt_update(P.opt_kind, 0, touched, h0, P.h1, P.h2, P.h3, v.y, g.y, a.y, c.y);
                opt_update(P.opt_kind, 0, touched, h0, P.h1, P.h2, P.h3, v.z, g.z, a.z, c.z);
                opt_update(P.opt_kind, 0, touched, h0, P.h1, P.h2, P.h3, v.w, g.w, a.w, c.w);
                *reinterpret_cast<float4*>(var) = v;
                if (has0) *reinterpret_cast<float4*>(s0p) = a;
                if (has1) *reinterpret_cast<float4*>(s1p) = c;
                *reinterpret_cast<float4*>(grd) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        } else {
            for (int64_t e = tid; e < eAll; e += nthr) {
                const bool isU = e < eU;
                const int64_t i = isU ? e : e - eU;
                float* var = (isU ? P.U : P.V) + i;
                float* grd = (isU ? P.gU : P.gV) + i;
                const float g = __ldcg(grd);
                float v = __ldcg(var);
                float a = has0 ? __ldcg((isU ? P.s0U : P.s0V) + i) : 0.0f;
                float c = has1 ? __ldcg((isU ? P.s1U : P.s1V) + i) : 0.0f;
                const bool touched = __ldcg((isU ? P.tU : P.tV) + i / D) == stamp;
                opt_update(P.opt_kind, 0, touched, h0, P.h1, P.h2, P.h3, v, g, a, c);
                *var = v;
                if (has0) (isU ? P.s0U : P.s0V)[i] = a;
                if (has1) (isU ? P.s1U : P.s1V)[i] = c;
                *grd = 0.0f;
            }
        }
        grid_barrier(P.barrier, target);
    }
    if (adam && tid == 0) { P.adam_pows[0] = p1; P.adam_pows[1] = p2; }
}

// per-device barrier word of the persistent kernels
static unsigned int* g_barrier[16] = {nullptr};
int epoch_barrier_word(unsigned int** out) {
    int dev = 0;
    NRC_CUDA_CHECK(cudaGetDevice(&dev));
    NRC_REQUIRE(dev >= 0 && dev < 16, NRC_E_LIMIT, "device ordinal %d outside [0, 16)", dev);
    if (!g_barrier[dev]) NRC_CUDA_CHECK(cudaMalloc(&g_barrier[dev], 256));
    *out = g_barrier[dev];
    return NRC_OK;
}

static int build_grid(int64_t total) {
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    return blocks < 1 ? 1 : (int)blocks;
}

}  // namespace nrc

using namespace nrc;

// out[p] = position of the unshuffled sample that lands at shuffled position p, p in [0, n):
// the permutation RandomSampler would hand to BatchSampler (util/data_iterator.py:45-63).
extern "C" int nrc_shuffle_perm(int64_t n, int32_t shuffle, uint64_t seed, uint64_t epoch, int64_t* out,
                                void* stream) {
    Feistel F;
    int rc = feistel_init(F, n, shuffle, seed, epoch);
    if (rc) return rc;
    if (n == 0) return NRC_OK;
    shuffle_perm_kernel<<<build_grid(n), 256, 0, as_stream(stream)>>>(F, n, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// One epoch of a Pairwise / PointwiseSampler (data/sampler.py:189-206 / 121-147) as device arrays:
// positions [first, first + n_out) of the shuffled epoch.
extern "C" int nrc_epoch_build(const int64_t* train_indptr, const int32_t* train_indices, const int32_t* pos_users,
                               const int32_t* pos_items, int64_t n_pos, int32_t neg_num, int32_t num_items,
                               int32_t pairwise, int32_t shuffle, uint64_t seed, uint64_t epoch, int64_t first,
                               int64_t n_out, int32_t* out_users, int32_t* out_items, void* out_third,
                               void* stream) {
    EpochSpec E;
    int rc = epoch_spec_init(E, train_indptr, train_indices, pos_users, pos_items, n_pos, neg_num, num_items,
                             pairwise, shuffle, seed, epoch);
    if (rc) return rc;
    NRC_REQUIRE(first >= 0 && n_out >= 0 && first + n_out <= E.n_samples, NRC_E_VALUE,
                "[first, first + n_out) = [%lld, %lld) outside the epoch's %lld samples", (long long)first,
                (long long)(first + n_out), (long long)E.n_samples);
    if (n_out == 0) return NRC_OK;
    epoch_build_kernel<<<build_grid(n_out * (pairwise ? neg_num : 1)), 256, 0, as_stream(stream)>>>(
        E, first, n_out, out_users, out_items, reinterpret_cast<int32_t*>(out_third));
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_mf_epoch_fused(float* user_table, float* item_table, int32_t num_users, int32_t num_items,
                                  int32_t dim, const int64_t* train_indptr, const int32_t* train_indices,
                                  const int32_t* pos_users, const int32_t* pos_items, int64_t n_pos, int32_t neg_num,
                                  int32_t pairwise, int32_t shuffle, int32_t drop_last, uint64_t seed, uint64_t epoch,
                                  int32_t batch_size, int64_t first_step, int64_t num_steps, int32_t loss_kind,
                                  float reg, int32_t opt_kind, const float* hyper_host, float* adam_pows,
                                  float* grad_user, float* grad_item, int32_t* touched_user, int32_t* touched_item,
                                  float* slot0_user, float* slot1_user, float* slot0_item, float* slot1_item,
                                  int32_t first_stamp, int32_t* ws_users, int32_t* ws_items, void* ws_third,
                                  float* step_loss, void* stream) {
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    NRC_REQUIRE(dim > 0, NRC_E_VALUE, "dim must be positive");
    NRC_REQUIRE(opt_kind >= NRC_OPT_GD && opt_kind <= NRC_OPT_MOMENTUM, NRC_E_VALUE, "please select a suitable optimizer");
    if (pairwise) {
        NRC_REQUIRE(loss_kind == NRC_LOSS_BPR || loss_kind == NRC_LOSS_HINGE || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                    "please choose a suitable loss function");
        NRC_REQUIRE(neg_num == 1, NRC_E_VALUE, "MF trains on one negative per positive (MF.py:88)");
    } else {
        NRC_REQUIRE(loss_kind == NRC_LOSS_CROSS_ENTROPY || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                    "please choose a suitable loss function");
    }
    NRC_REQUIRE(opt_kind != NRC_OPT_ADAM || adam_pows != nullptr, NRC_E_VALUE, "adam needs the beta-power state");
    MfEpochParams P;
    int rc = epoch_spec_init(P.E, train_indptr, train_indices, pos_users, pos_items, n_pos, neg_num, num_items, pairwise,
                             shuffle, seed, epoch);
    if (rc) return rc;
    const int64_t n = P.E.n_samples;
    P.n_used = drop_last ? (n / batch_size) * batch_size : n;
    P.steps_total = (P.n_used + batch_size - 1) / batch_size;      // sampler.py:150-155,208-213
    NRC_REQUIRE(first_step >= 0 && num_steps >= 0 && first_step + num_steps <= P.steps_total, NRC_E_VALUE,
                "steps [%lld, %lld) outside the epoch's %lld steps", (long long)first_step,
                (long long)(first_step + num_steps), (long long)P.steps_total);
    if (num_steps == 0) return NRC_OK;
    P.U = user_table; P.V = item_table; P.gU = grad_user; P.gV = grad_item;
    P.tU = touched_user; P.tV = touched_item;
    P.s0U = slot0_user; P.s1U = slot1_user; P.s0V = slot0_item; P.s1V = slot1_item;
    P.ws_u = ws_users; P.ws_i = ws_items; P.ws_t = reinterpret_cast<int32_t*>(ws_third);
    P.step_loss = step_loss; P.adam_pows = adam_pows;
    P.first_step = first_step; P.num_steps = num_steps;
    P.num_users = num_users; P.num_items = num_items; P.D = dim; P.batch_size = batch_size;
    P.loss_kind = loss_kind; P.opt_kind = opt_kind; P.first_stamp = first_stamp;
    P.build = first_step == 0 ? 1 : 0;
    P.reg = reg;
    P.h0 = hyper_host ? hyper_host[0] : 0.0f; P.h1 = hyper_host ? hyper_host[1] : 0.0f;
    P.h2 = hyper_host ? hyper_host[2] : 0.0f; P.h3 = hyper_host ? hyper_host[3] : 0.0f;
    rc = epoch_barrier_word(&P.barrier);
    if (rc) return rc;
    cudaStream_t st = as_stream(stream);
    NRC_CUDA_CHECK(cudaMemsetAsync(P.barrier, 0, sizeof(unsigned int), st));
    const void* fn;
#define NRC_PICK(PW) \
    fn = dim == 128 ? (const void*)mf_epoch_kernel<PW, 4> : dim == 64 ? (const void*)mf_epoch_kernel<PW, 2> \
       : dim == 32 ? (const void*)mf_epoch_kernel<PW, 1> : (const void*)mf_epoch_kernel<PW, 0>
    if (pairwise) { NRC_PICK(true); } else { NRC_PICK(false); }
#undef NRC_PICK
    int per_sm = 0;
    NRC_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 512, 0));
    NRC_REQUIRE(per_sm >= 1, NRC_E_CUDA, "the persistent epoch kernel does not fit an SM");
    // capped: the largest batch of the launch has more samples than the grid has warps (phase 1 loops)
    const int64_t rest = P.n_used - first_step * batch_size, most = rest < batch_size ? rest : batch_size;
    mf_route(kMfEpoch, dim == 128 ? 4 : dim == 64 ? 2 : dim == 32 ? 1 : 0, 0, -1, -1, sm_count(),
             most > (int64_t)sm_count() * (512 / 32), (dim & 3) == 0 ? 1 : 0);
    void* args[] = {&P};
    NRC_CUDA_CHECK(cudaLaunchCooperativeKernel(fn, dim3(sm_count()), dim3(512), args, 0, st));
    return NRC_OK;
}
