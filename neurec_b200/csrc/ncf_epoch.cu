// NeuMF / MLP: the device-resident epoch -- shuffle + negative sampling + every step of the epoch
// in ONE persistent cooperative launch (the NCF counterpart of nrc_mf_epoch_fused).
//
// Replaces (reference paths):
//   model/general_recommender/NeuMF.py:126-151, MLP.py:100-120   the per-batch sess.run loop
//   data/sampler.py:71-90,121-147,189-206, util/data_iterator.py:45-63,133-155   sampler + batching
//
// One 256-thread CTA per SM, all co-resident.  Per step:
//   phase 1  every CTA copies the tower weights (27 KB per tower, padded row stride out+1) into
//            shared memory once, then its two 128-thread groups each take samples of the batch:
//            gather the four embedding rows, tower forward and backward out of shared memory
//            (k-ranges split over thread groups, partial sums combined in fixed order), embedding
//            gradients added into the dense accumulators with RED (duplicates sum, TF's
//            IndexedSlices de-duplication), activations / deltas of every layer to an L2-resident
//            scratch buffer;
//   grid barrier
//   phase 2  (a) dense weights: thread quartet per weight entry, dW = sum_s a[s][k] * delta[s][j]
//            over four batch slices + shuffle reduction (fixed order, no atomics), then the
//            TensorFlow-1.12 dense-gradient optimizer formula on that entry in place;
//            (b) the four embedding tables: the IndexedSlices optimizer (Adam dense over every row),
//            accumulators zeroed;
//   grid barrier.
// Arithmetic identical to nrc_ncf_train_epoch except for the summation order of dW (fixed slices
// instead of atomics) -- tests compare both with oracle/tf_math.NCFTrainer.
#include "epoch.cuh"
#include "learner.cuh"
#include "ncf.cuh"
#include "optim.cuh"

namespace nrc {

constexpr int kEpThreads = 256;
constexpr int kGroups = kEpThreads / kNcfThreads;   // sample groups per CTA
constexpr int kWSlices = 4;                         // batch slices per weight entry (adjacent lanes)

struct NcfSeg {            // one embedding table for the optimizer phase
    float* var; float* grad; float* s0; float* s1; const int32_t* touched;
    int64_t elems; int dim;
};

struct NcfEpochParams {
    EpochSpec E;
    NcfDev S;
    NcfPtrs P;
    float* dense;                 // writable alias of P.dense
    float* d_s0; float* d_s1;     // optimizer slots of the packed dense parameters
    NcfSeg seg[4];
    int32_t* ws_u; int32_t* ws_i; int32_t* ws_t;
    float* scratch;               // [batch][2 * passes * act_size]
    float* step_loss;
    float* adam_pows;
    unsigned int* barrier;
    int64_t n_used, first_step, num_steps, steps_total;
    int32_t batch_size, pairwise, loss_kind, opt_kind, first_stamp, build;
    int64_t seg_end[4];                    // running float4-group counts of seg[0..3] (tables_vec4)
    int32_t tables_vec4;                   // every table width a multiple of 4 (and 16-byte aligned rows)
    int32_t sw_floats;                     // shared-memory floats of the weight copy (towers, rounded up to 4)
    int32_t wblocked, wblocks, sred_off;   // blocked weight-gradient path: 4 x 4 blocks per tower; smem offset (floats) of its reduction slots
    float reg_mf, reg_mlp, h0, h1, h2, h3;
};

__device__ __forceinline__ void group_sync(int grp) {
    asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(kNcfThreads) : "memory");
}

__device__ __forceinline__ float group_sum(float v, float* red, int tid, int grp) {
    v = warp_sum(v);
    if ((tid & 31) == 0) red[tid >> 5] = v;
    group_sync(grp);
    const float r = red[0] + red[1] + red[2] + red[3];
    group_sync(grp);
    return r;
}

// a_out = relu(a_in . W + b); W in shared memory exactly as in global memory (row stride out)
__device__ __forceinline__ void fwd_layer(const float* __restrict__ W, const float* __restrict__ B, int in, int out,
                                          const float* a_in, float* a_out, float* part, int tid, int grp) {
    if (NCF_FWD_SPLIT(in, out)) {
        const int G = kNcfThreads / out, kpg = in / G, j = tid % out, g = tid / out;
        float acc = 0.0f;
#pragma unroll 8
        for (int kk = 0; kk < kpg; ++kk) acc = fmaf(a_in[g * kpg + kk], W[(g * kpg + kk) * out + j], acc);
        part[tid] = acc;
        group_sync(grp);
        if (tid < out) {
            float s = B[tid];
            for (int q = 0; q < G; ++q) s += part[q * out + tid];
            a_out[tid] = fmaxf(s, 0.0f);              // tf.nn.relu
        }
    } else {
        for (int j = tid; j < out; j += kNcfThreads) {
            float acc = B[j];
            for (int k = 0; k < in; ++k) acc = fmaf(a_in[k], W[k * out + j], acc);
            a_out[j] = fmaxf(acc, 0.0f);
        }
    }
    group_sync(grp);
}

// d_in[k] = (mask ? a_in[k] > 0 : 1) * sum_j W[k][j] d_out[j].  Threads (k, jq) walk their jpt columns
// starting at a k-dependent rotation so that the lanes of a warp (16 or 8 different k) hit different
// banks of the unpadded row-major W.
__device__ __forceinline__ void bwd_layer(const float* __restrict__ W, int in, int out, const float* d_out,
                                          const float* a_in, float* d_in, bool mask, int tid, int grp) {
    if (NCF_BWD_SPLIT(in, out)) {
        const int tpr = kNcfThreads / in, jpt = out / tpr, k = tid / tpr, jq = tid % tpr;
        float s = 0.0f;
        int jj = k % jpt;
#pragma unroll 8
        for (int c = 0; c < jpt; ++c) {
            s = fmaf(W[k * out + jq * jpt + jj], d_out[jq * jpt + jj], s);
            jj = (jj + 1 == jpt) ? 0 : jj + 1;
        }
        for (int o = tpr >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(kFull, s, o);
        if (jq == 0) d_in[k] = mask ? ((a_in[k] > 0.0f) ? s : 0.0f) : s;
    } else {
        const int lane = tid & 31, wrp = tid >> 5;
        for (int k = wrp; k < in; k += kNcfThreads / 32) {
            float s = 0.0f;
            for (int j = lane; j < out; j += kWarp) s = fmaf(W[k * out + j], d_out[j], s);
            s = warp_sum(s);
            if (lane == 0) d_in[k] = mask ? ((a_in[k] > 0.0f) ? s : 0.0f) : s;
        }
    }
    group_sync(grp);
}

__device__ __forceinline__ void ncf_sample(const NcfEpochParams& Q, const float* sW, float* sAct, float* sDel, float* part,
                                           float* red, int tid, int grp, int64_t b, int64_t cnt, int32_t u, int32_t it0,
                                           int32_t third, int32_t stamp, float& loss_out) {
    const NcfDev& S = Q.S;
    const NcfPtrs& P = Q.P;
    const int passes = Q.pairwise ? 2 : 1;
    const int it[2] = {it0, Q.pairwise ? third : 0};
    const int MD = S.mlp_dim, L = S.n_layers;
    float yhat[2] = {0.0f, 0.0f};
    for (int p = 0; p < passes; ++p) {
        float* act = sAct + p * S.act_size;
        float mf = 0.0f;
        for (int k = tid; k < S.mf_dim; k += kNcfThreads)
            mf = fmaf(__ldcg(P.mf_user + (size_t)u * S.mf_dim + k), __ldcg(P.mf_item + (size_t)it[p] * S.mf_dim + k), mf);
        for (int k = tid; k < 2 * MD; k += kNcfThreads)
            act[k] = (k < MD) ? __ldcg(P.mlp_user + (size_t)u * MD + k) : __ldcg(P.mlp_item + (size_t)it[p] * MD + (k - MD));
        group_sync(grp);
        const float* tw = sW + (size_t)((p == 1 && S.n_towers == 2) ? 1 : 0) * S.tower_size;
        for (int l = 0; l < L; ++l)
            fwd_layer(tw + S.w_off[l], tw + S.b_off[l], S.in_dim[l], S.out_dim[l], act + S.a_off[l], act + S.a_off[l + 1],
                      part, tid, grp);
        float s = 0.0f;
        if (L > 0)
            for (int j = tid; j < S.out_dim[L - 1]; j += kNcfThreads) s += act[S.a_off[L] + j];
        yhat[p] = group_sum(mf + s, red, tid, grp);      // NeuMF.py:85 reduce_sum(concat(mf, mlp))
    }
    float l, g;
    if (Q.pairwise) pairwise_loss_grad(Q.loss_kind, yhat[0] - yhat[1], l, g);   // NeuMF.py:92
    else pointwise_loss_grad(Q.loss_kind, yhat[0], __int_as_float(third), 1.0f / (float)cnt, l, g);
    float sq_mf = 0.f, sq_mlp = 0.f;
    for (int p = 0; p < passes; ++p) {
        const float gp = (p == 0) ? g : -g;
        const float* tw = sW + (size_t)((p == 1 && S.n_towers == 2) ? 1 : 0) * S.tower_size;
        float* act = sAct + p * S.act_size;
        float* del = sDel + p * S.act_size;
        if (L > 0) {
            for (int j = tid; j < S.out_dim[L - 1]; j += kNcfThreads)
                del[S.a_off[L] + j] = (act[S.a_off[L] + j] > 0.0f) ? gp : 0.0f;     // ReluGrad on the last layer
            group_sync(grp);
            for (int l2 = L - 1; l2 >= 0; --l2)
                bwd_layer(tw + S.w_off[l2], S.in_dim[l2], S.out_dim[l2], del + S.a_off[l2 + 1], act + S.a_off[l2],
                          del + S.a_off[l2], l2 > 0, tid, grp);
        }
        for (int k = tid; k < S.mf_dim; k += kNcfThreads) {
            const float pu = __ldcg(P.mf_user + (size_t)u * S.mf_dim + k);
            const float qi = __ldcg(P.mf_item + (size_t)it[p] * S.mf_dim + k);
            atomicAdd(P.g_mf_user + (size_t)u * S.mf_dim + k, gp * qi + (p == 0 ? Q.reg_mf * pu : 0.f));
            atomicAdd(P.g_mf_item + (size_t)it[p] * S.mf_dim + k, gp * pu + Q.reg_mf * qi);
            sq_mf += qi * qi + (p == 0 ? pu * pu : 0.f);
        }
        for (int k = tid; k < 2 * MD; k += kNcfThreads) {
            const float a = act[k];
            if (k < MD) {
                atomicAdd(P.g_mlp_user + (size_t)u * MD + k, del[k] + (p == 0 ? Q.reg_mlp * a : 0.f));
                if (p == 0) sq_mlp += a * a;
            } else {
                atomicAdd(P.g_mlp_item + (size_t)it[p] * MD + (k - MD), del[k] + Q.reg_mlp * a);
                sq_mlp += a * a;
            }
        }
        if (tid == 0) P.t_item[it[p]] = stamp;
    }
    if (tid == 0) P.t_user[u] = stamp;
    if (Q.reg_mf != 0.f || Q.reg_mlp != 0.f)             // NeuMF.py:94-100
        l += group_sum(Q.reg_mf * 0.5f * sq_mf + Q.reg_mlp * 0.5f * sq_mlp, red, tid, grp);
    loss_out = l;
    float* out_s = Q.scratch + (size_t)b * (2 * passes * S.act_size);
    for (int e = tid; e < passes * S.act_size; e += kNcfThreads) {
        out_s[e] = sAct[e];
        out_s[passes * S.act_size + e] = sDel[e];
    }
    group_sync(grp);
}

__global__ void __launch_bounds__(kEpThreads, 1) ncf_epoch_kernel(const NcfEpochParams Q) {
    extern __shared__ __align__(16) float sm[];
    const NcfDev& S = Q.S;
    const int tid_cta = threadIdx.x, grp = tid_cta / kNcfThreads, tid = tid_cta % kNcfThreads;
    const int passes = Q.pairwise ? 2 : 1;
    float* sW = sm;                                                     // n_towers padded towers
    float* gbase = sW + (size_t)Q.sw_floats + (size_t)grp * (2 * passes * S.act_size + kNcfThreads + 8);
    float* sAct = gbase;
    float* sDel = sAct + passes * S.act_size;
    float* part = sDel + passes * S.act_size;
    float* red = part + kNcfThreads;
    const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nthr = (int64_t)gridDim.x * blockDim.x;
    unsigned int target = 0;

    if (Q.build) {
        for (int64_t p = gtid; p < Q.n_used; p += nthr) {
            int32_t u, it, th;
            epoch_sample(Q.E, p, 0, u, it, th);
            Q.ws_u[p] = u; Q.ws_i[p] = it; Q.ws_t[p] = th;
        }
        for (int64_t s = gtid; s < Q.steps_total; s += nthr) Q.step_loss[s] = 0.0f;
        grid_barrier(Q.barrier, target);
    }
    const bool adam = Q.opt_kind == NRC_OPT_ADAM;
    float p1 = 0.0f, p2 = 0.0f;
    if (adam) { p1 = __ldcg(Q.adam_pows); p2 = __ldcg(Q.adam_pows + 1); }
    const bool has0 = Q.opt_kind != NRC_OPT_GD;
    const bool has1 = adam || Q.opt_kind == NRC_OPT_RMSPROP;
    const int dense_total = S.tower_size * S.n_towers;
    const int stride = 2 * passes * S.act_size;

    for (int64_t s = Q.first_step; s < Q.first_step + Q.num_steps; ++s) {
        const int64_t off = s * Q.batch_size;
        const int64_t cnt = (Q.n_used - off < Q.batch_size) ? (Q.n_used - off) : Q.batch_size;
        const int32_t stamp = Q.first_stamp + (int32_t)(s - Q.first_step);
        // ---- phase 1: this step's weights -> shared memory (padded rows), then the samples
        {   // straight float4 copy (the packed dense buffer is 16-byte aligned and sw_floats is a multiple of 4):
            // every thread's loads are independent -> one L2 round trip
            const int n4 = Q.sw_floats >> 2, total = S.tower_size * S.n_towers;
            const float4* src4 = reinterpret_cast<const float4*>(Q.dense);
            float4* dst4 = reinterpret_cast<float4*>(sW);
            float4 v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int e = tid_cta + i * kEpThreads;
                if (e < n4) {
                    if (e * 4 + 3 < total) v[i] = __ldcg(src4 + e);
                    else {      // the tail of a buffer whose length is not a multiple of 4
                        float t4[4] = {0.f, 0.f, 0.f, 0.f};
                        for (int c = 0; c < 4; ++c) if (e * 4 + c < total) t4[c] = __ldcg(Q.dense + e * 4 + c);
                        v[i] = make_float4(t4[0], t4[1], t4[2], t4[3]);
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int e = tid_cta + i * kEpThreads;
                if (e < n4) dst4[e] = v[i];
            }
            for (int e = tid_cta + 8 * kEpThreads; e < n4; e += kEpThreads) {    // towers beyond 8192 floats
                if (e * 4 + 3 < total) dst4[e] = __ldcg(src4 + e);
                else for (int c = 0; c < 4; ++c) sW[e * 4 + c] = (e * 4 + c < total) ? __ldcg(Q.dense + e * 4 + c) : 0.0f;
            }
        }
        __syncthreads();
        float loss_acc = 0.0f;
        for (int64_t b = (int64_t)blockIdx.x * kGroups + grp; b < cnt; b += (int64_t)gridDim.x * kGroups) {
            float l = 0.0f;
            ncf_sample(Q, sW, sAct, sDel, part, red, tid, grp, b, cnt, __ldcg(Q.ws_u + off + b), __ldcg(Q.ws_i + off + b),
                       __ldcg(Q.ws_t + off + b), stamp, l);
            loss_acc += l;
        }
        if (tid == 0 && loss_acc != 0.0f) atomicAdd(Q.step_loss + s, loss_acc);
        grid_barrier(Q.barrier, target);
        // ---- phase 2
        float h0 = Q.h0;
        if (adam) {
            h0 = __fdiv_rn(__fmul_rn(Q.h0, __fsqrt_rn(__fsub_rn(1.0f, p2))), __fsub_rn(1.0f, p1));
            p1 = __fmul_rn(p1, Q.h1);
            p2 = __fmul_rn(p2, Q.h2);
        }
        // (a) dense weights.  Blocked path (every layer width a multiple of 4): a 64-thread group owns a 4 x 4
        // block of one layer's weight matrix (or 4 bias entries); each thread takes the samples s = lane64,
        // lane64 + 64, ... with ONE float4 of activations and ONE float4 of deltas per sample (all loads of a
        // thread are independent: one L2 round trip), 16 FMAs per sample; the 64 partial blocks are summed by
        // warp shuffles + one shared-memory hop in fixed order; 16 lanes apply the dense optimizer formula.
        if (Q.wblocked) {
            const int grp64 = tid_cta >> 6, l64 = tid_cta & 63, wl = tid_cta & 31;
            float* sred = sm + Q.sred_off + grp64 * 16;
            for (int bi = blockIdx.x * (kEpThreads / 64) + grp64; bi < Q.wblocks * S.n_towers; bi += gridDim.x * (kEpThreads / 64)) {
                const int tower = bi / Q.wblocks;
                int bb = bi - tower * Q.wblocks, l = 0;
                bool is_bias = false;
                for (;; ++l) {
                    const int nw = (S.in_dim[l] >> 2) * (S.out_dim[l] >> 2), nb = S.out_dim[l] >> 2;
                    if (bb < nw) break;
                    bb -= nw;
                    if (bb < nb) { is_bias = true; break; }
                    bb -= nb;
                }
                const int ob = S.out_dim[l] >> 2;
                const int k0 = is_bias ? 0 : (bb / ob) * 4, j0 = (is_bias ? bb : bb % ob) * 4;
                float acc[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) acc[i] = 0.0f;
                for (int p = 0; p < passes; ++p) {
                    if (S.n_towers == 2 && p != tower) continue;     // shared tower (MLP.py:53-54): both passes feed dW
                    const float* ap = Q.scratch + p * S.act_size + S.a_off[l] + k0;
                    const float* dp = Q.scratch + (passes + p) * S.act_size + S.a_off[l + 1] + j0;
#pragma unroll 4
                    for (int64_t ss = l64; ss < cnt; ss += 64) {
                        const float4 d4 = __ldcg(reinterpret_cast<const float4*>(dp + ss * stride));
                        const float4 a4 = is_bias ? make_float4(1.f, 0.f, 0.f, 0.f)
                                                  : __ldcg(reinterpret_cast<const float4*>(ap + ss * stride));
                        const float av[4] = {a4.x, a4.y, a4.z, a4.w}, dv[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
                        for (int r = 0; r < 4; ++r)
#pragma unroll
                            for (int c = 0; c < 4; ++c) acc[r * 4 + c] = fmaf(av[r], dv[c], acc[r * 4 + c]);
                    }
                }
#pragma unroll
                for (int i = 0; i < 16; ++i) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) acc[i] += __shfl_xor_sync(kFull, acc[i], o);
                }
                float mine = 0.0f;                                   // lane i keeps entry i of the block
#pragma unroll
                for (int i = 0; i < 16; ++i) mine = (wl == i) ? acc[i] : mine;
                if ((l64 >> 5) == 1 && wl < 16) sred[wl] = mine;     // second warp of the group -> shared memory
                asm volatile("bar.sync %0, 64;" ::"r"(3 + grp64) : "memory");
                if ((l64 >> 5) == 0 && wl < 16) {
                    const float g = mine + sred[wl];
                    const int r = wl >> 2, c = wl & 3;
                    if (!is_bias || r == 0) {
                        const int e = is_bias ? (S.b_off[l] + j0 + c) : (S.w_off[l] + (k0 + r) * S.out_dim[l] + j0 + c);
                        const int e_all = tower * S.tower_size + e;
                        float var = __ldcg(Q.dense + e_all);
                        float a0 = has0 ? __ldcg(Q.d_s0 + e_all) : 0.0f;
                        float a1 = has1 ? __ldcg(Q.d_s1 + e_all) : 0.0f;
                        opt_update(Q.opt_kind, 1, true, h0, Q.h1, Q.h2, Q.h3, var, g, a0, a1);
                        Q.dense[e_all] = var;
                        if (has0) Q.d_s0[e_all] = a0;
                        if (has1) Q.d_s1[e_all] = a1;
                    }
                }
                asm volatile("bar.sync %0, 64;" ::"r"(3 + grp64) : "memory");
            }
        } else {
        // generic path: lane quartet per entry, batch in kWSlices fixed slices
        const int64_t quartets = (int64_t)dense_total * kWSlices;
        for (int64_t q0 = gtid; q0 < ((quartets + 31) & ~(int64_t)31); q0 += nthr) {   // warp-uniform trip count
            const bool live = q0 < quartets;
            const int e_all = live ? (int)(q0 / kWSlices) : 0, slice = (int)(q0 % kWSlices);
            const int tower = e_all / S.tower_size, e = e_all - tower * S.tower_size;
            int l = 0;
            while (l + 1 < S.n_layers && e >= S.w_off[l + 1]) ++l;
            const bool is_bias = e >= S.b_off[l];
            const int out = S.out_dim[l];
            const int k = is_bias ? 0 : (e - S.w_off[l]) / out;
            const int j = is_bias ? (e - S.b_off[l]) : (e - S.w_off[l]) % out;
            const int64_t s0 = (cnt * slice) / kWSlices, s1 = (cnt * (slice + 1)) / kWSlices;
            float acc = 0.0f;
            for (int p = 0; p < passes && live; ++p) {
                // tower t collects pass t (two towers) or both passes (shared weights, MLP.py:53-54)
                if (S.n_towers == 2 && p != tower) continue;
                const float* a = Q.scratch + p * S.act_size + S.a_off[l] + k;
                const float* d = Q.scratch + (passes + p) * S.act_size + S.a_off[l + 1] + j;
#pragma unroll 4
                for (int64_t ss = s0; ss < s1; ++ss) {
                    const float dj = __ldcg(d + ss * stride);
                    const float av = is_bias ? 1.0f : __ldcg(a + ss * stride);
                    acc = fmaf(av, dj, acc);
                }
            }
            acc += __shfl_xor_sync(kFull, acc, 1);
            acc += __shfl_xor_sync(kFull, acc, 2);
            if (live && slice == 0) {
                float var = __ldcg(Q.dense + e_all);
                float a0 = has0 ? __ldcg(Q.d_s0 + e_all) : 0.0f;
                float a1 = has1 ? __ldcg(Q.d_s1 + e_all) : 0.0f;
                opt_update(Q.opt_kind, 1, true, h0, Q.h1, Q.h2, Q.h3, var, acc, a0, a1);
                Q.dense[e_all] = var;
                if (has0) Q.d_s0[e_all] = a0;
                if (has1) Q.d_s1[e_all] = a1;
            }
        }
        }
        // (b) embedding tables.  All four tables form ONE flat space of float4 groups (a grid of one 256-thread
        // CTA per SM covers ml-100k's 26k groups in a single trip: one latency chain instead of four).
        if (Q.tables_vec4) {
            const bool stamped = !(adam || Q.opt_kind == NRC_OPT_GD);
            const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int64_t gi = gtid; gi < Q.seg_end[3]; gi += nthr) {
                const int t = (gi >= Q.seg_end[0]) + (gi >= Q.seg_end[1]) + (gi >= Q.seg_end[2]);
                const NcfSeg& G = Q.seg[t];
                const int64_t e = (gi - (t ? Q.seg_end[t - 1] : 0)) * 4;
                const float4 g = __ldcg(reinterpret_cast<const float4*>(G.grad + e));
                float4 v = __ldcg(reinterpret_cast<const float4*>(G.var + e));
                float4 a = has0 ? __ldcg(reinterpret_cast<const float4*>(G.s0 + e)) : z4;
                float4 c = has1 ? __ldcg(reinterpret_cast<const float4*>(G.s1 + e)) : z4;
                const bool t1 = stamped ? (__ldcg(G.touched + e / G.dim) == stamp) : true;
                opt_update(Q.opt_kind, 0, t1, h0, Q.h1, Q.h2, Q.h3, v.x, g.x, a.x, c.x);
                opt_update(Q.opt_kind, 0, t1, h0, Q.h1, Q.h2, Q.h3, v.y, g.y, a.y, c.y);
                opt_update(Q.opt_kind, 0, t1, h0, Q.h1, Q.h2, Q.h3, v.z, g.z, a.z, c.z);
                opt_update(Q.opt_kind, 0, t1, h0, Q.h1, Q.h2, Q.h3, v.w, g.w, a.w, c.w);
                *reinterpret_cast<float4*>(G.var + e) = v;
                if (has0) *reinterpret_cast<float4*>(G.s0 + e) = a;
                if (has1) *reinterpret_cast<float4*>(G.s1 + e) = c;
                *reinterpret_cast<float4*>(G.grad + e) = z4;
            }
        } else {
#pragma unroll 1
            for (int t = 0; t < 4; ++t) {
                const NcfSeg& G = Q.seg[t];
                for (int64_t e = gtid; e < G.elems; e += nthr) {
                    const float g = __ldcg(G.grad + e);
                    float v = __ldcg(G.var + e);
                    float a = has0 ? __ldcg(G.s0 + e) : 0.0f, c = has1 ? __ldcg(G.s1 + e) : 0.0f;
                    const bool touched = __ldcg(G.touched + e / G.dim) == stamp;
                    opt_update(Q.opt_kind, 0, touched, h0, Q.h1, Q.h2, Q.h3, v, g, a, c);
                    G.var[e] = v;
                    if (has0) G.s0[e] = a;
                    if (has1) G.s1[e] = c;
                    G.grad[e] = 0.0f;
                }
            }
        }
        grid_barrier(Q.barrier, target);
    }
    if (adam && gtid == 0) { Q.adam_pows[0] = p1; Q.adam_pows[1] = p2; }
}

int epoch_barrier_word(unsigned int** out);   // epoch.cu

static float* g_ep_scratch = nullptr;
static size_t g_ep_scratch_floats = 0;

}  // namespace nrc

using namespace nrc;

extern "C" int nrc_ncf_epoch_fused(const nrc_ncf_shape* shape, float* mf_user, float* mf_item, float* mlp_user,
                                   float* mlp_item, float* dense, const int64_t* train_indptr,
                                   const int32_t* train_indices, const int32_t* pos_users, const int32_t* pos_items,
                                   int64_t n_pos, int32_t neg_num, int32_t pairwise, int32_t shuffle, int32_t drop_last,
                                   uint64_t seed, uint64_t epoch, int32_t batch_size, int64_t first_step,
                                   int64_t num_steps, int32_t loss_kind, float reg_mf, float reg_mlp, int32_t opt_kind,
                                   const float* hyper_host, float* adam_pows, float* const* grads, float* const* slot0,
                                   float* const* slot1, int32_t* touched_user, int32_t* touched_item,
                                   int32_t first_stamp, int32_t* ws_users, int32_t* ws_items, void* ws_third,
                                   float* step_loss, void* stream) {
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    NRC_REQUIRE(opt_kind >= NRC_OPT_GD && opt_kind <= NRC_OPT_MOMENTUM, NRC_E_VALUE, "please select a suitable optimizer");
    NRC_REQUIRE(grads != nullptr, NRC_E_VALUE, "gradient accumulators are NULL");
    NcfEpochParams Q;
    int rc = ncf_make(Q.S, shape);
    if (rc) return rc;
    if (pairwise) {
        NRC_REQUIRE(loss_kind == NRC_LOSS_BPR || loss_kind == NRC_LOSS_HINGE || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                    "please choose a suitable loss function");
        NRC_REQUIRE(neg_num == 1, NRC_E_VALUE, "pairwise NCF trains on one negative per positive (NeuMF.py:126)");
    } else {
        NRC_REQUIRE(loss_kind == NRC_LOSS_CROSS_ENTROPY || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                    "please choose a suitable loss function");
    }
    NRC_REQUIRE(opt_kind != NRC_OPT_ADAM || adam_pows != nullptr, NRC_E_VALUE, "adam needs the beta-power state");
    rc = epoch_spec_init(Q.E, train_indptr, train_indices, pos_users, pos_items, n_pos, neg_num, shape->num_items, pairwise,
                         shuffle, seed, epoch);
    if (rc) return rc;
    const int64_t n = Q.E.n_samples;
    Q.n_used = drop_last ? (n / batch_size) * batch_size : n;
    Q.steps_total = (Q.n_used + batch_size - 1) / batch_size;
    NRC_REQUIRE(first_step >= 0 && num_steps >= 0 && first_step + num_steps <= Q.steps_total, NRC_E_VALUE,
                "steps [%lld, %lld) outside the epoch's %lld steps", (long long)first_step,
                (long long)(first_step + num_steps), (long long)Q.steps_total);
    if (num_steps == 0) return NRC_OK;
    const NcfDev& S = Q.S;
    const int passes = pairwise ? 2 : 1;
    Q.sw_floats = (S.n_towers * S.tower_size + 3) & ~3;
    const size_t smem_floats = (size_t)Q.sw_floats + (size_t)kGroups * (2 * passes * S.act_size + kNcfThreads + 8);
    const size_t smem = (smem_floats + (kEpThreads / 64) * 16) * 4;
    Q.sred_off = (int32_t)smem_floats;
    Q.wblocked = 1; Q.wblocks = 0;
    for (int l = 0; l < S.n_layers; ++l) {
        if ((S.in_dim[l] & 3) || (S.out_dim[l] & 3)) Q.wblocked = 0;
        Q.wblocks += (S.in_dim[l] >> 2) * (S.out_dim[l] >> 2) + (S.out_dim[l] >> 2);
    }
    if ((S.act_size & 3) || S.n_layers == 0) Q.wblocked = 0;
    NRC_REQUIRE(smem <= 200 * 1024, NRC_E_LIMIT, "NCF tower needs %zu B of shared memory", smem);
    const size_t need = (size_t)2 * passes * S.act_size * (size_t)batch_size;
    if (need > g_ep_scratch_floats) {
        if (g_ep_scratch) NRC_CUDA_CHECK(cudaFree(g_ep_scratch));
        g_ep_scratch = nullptr; g_ep_scratch_floats = 0;
        NRC_CUDA_CHECK(cudaMalloc(&g_ep_scratch, (need + 1024) * sizeof(float)));
        g_ep_scratch_floats = need + 1024;
    }
    Q.P = NcfPtrs{mf_user, mf_item, mlp_user, mlp_item, dense, grads[0], grads[1], grads[2], grads[3], nullptr,
                  touched_user, touched_item};
    Q.dense = dense;
    Q.d_s0 = slot0 ? slot0[4] : nullptr;
    Q.d_s1 = slot1 ? slot1[4] : nullptr;
    float* vars[4] = {mf_user, mf_item, mlp_user, mlp_item};
    const int64_t rows[4] = {shape->num_users, shape->num_items, shape->num_users, shape->num_items};
    const int dims[4] = {S.mf_dim, S.mf_dim, S.mlp_dim, S.mlp_dim};
    const int32_t* tch[4] = {touched_user, touched_item, touched_user, touched_item};
    for (int t = 0; t < 4; ++t)
        Q.seg[t] = NcfSeg{vars[t], grads[t], slot0 ? slot0[t] : nullptr, slot1 ? slot1[t] : nullptr, tch[t],
                          rows[t] * dims[t], dims[t] > 0 ? dims[t] : 1};
    Q.tables_vec4 = 1;
    for (int t = 0; t < 4; ++t) {
        const NcfSeg& G = Q.seg[t];
        const auto misaligned = [](const void* q) { return q && (reinterpret_cast<uintptr_t>(q) & 15) != 0; };
        if (G.elems && ((G.dim & 3) || misaligned(G.var) || misaligned(G.grad) || misaligned(G.s0) || misaligned(G.s1)))
            Q.tables_vec4 = 0;
        Q.seg_end[t] = (t ? Q.seg_end[t - 1] : 0) + G.elems / 4;
    }
    Q.ws_u = ws_users; Q.ws_i = ws_items; Q.ws_t = reinterpret_cast<int32_t*>(ws_third);
    Q.scratch = g_ep_scratch; Q.step_loss = step_loss; Q.adam_pows = adam_pows;
    Q.first_step = first_step; Q.num_steps = num_steps;
    Q.batch_size = batch_size; Q.pairwise = pairwise ? 1 : 0; Q.loss_kind = loss_kind; Q.opt_kind = opt_kind;
    Q.first_stamp = first_stamp; Q.build = first_step == 0 ? 1 : 0;
    Q.reg_mf = reg_mf; Q.reg_mlp = reg_mlp;
    Q.h0 = hyper_host ? hyper_host[0] : 0.0f; Q.h1 = hyper_host ? hyper_host[1] : 0.0f;
    Q.h2 = hyper_host ? hyper_host[2] : 0.0f; Q.h3 = hyper_host ? hyper_host[3] : 0.0f;
    rc = epoch_barrier_word(&Q.barrier);
    if (rc) return rc;
    cudaStream_t st = as_stream(stream);
    NRC_CUDA_CHECK(cudaMemsetAsync(Q.barrier, 0, sizeof(unsigned int), st));
    static bool attr_done = false;
    if (!attr_done) {
        NRC_CUDA_CHECK(cudaFuncSetAttribute(ncf_epoch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_done = true;
    }
    int per_sm = 0;
    NRC_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ncf_epoch_kernel, kEpThreads, smem));
    NRC_REQUIRE(per_sm >= 1, NRC_E_CUDA, "the persistent NCF epoch kernel does not fit an SM");
    ncf_routes_reset();
    g_ncf_routes[kRouteEpochDwBlocked] = Q.wblocked;
    g_ncf_routes[kRouteEpochTablesVec4] = Q.tables_vec4;
    g_ncf_routes[kRouteFwdSplit] = g_ncf_routes[kRouteBwdSplit] = 0;
    for (int l = 0; l < S.n_layers; ++l) {
        if (NCF_FWD_SPLIT(S.in_dim[l], S.out_dim[l])) g_ncf_routes[kRouteFwdSplit] |= 1 << l;
        if (NCF_BWD_SPLIT(S.in_dim[l], S.out_dim[l])) g_ncf_routes[kRouteBwdSplit] |= 1 << l;
    }
    void* args[] = {&Q};
    NRC_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)ncf_epoch_kernel, dim3(sm_count()), dim3(kEpThreads), args, smem, st));
    return NRC_OK;
}
