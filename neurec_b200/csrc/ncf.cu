// NCF family (MLP, NeuMF = GMF + MLP): fused gather -> MLP tower forward -> loss -> backward ->
// gradient accumulation, and the score-all-items predict.
//
// Replaces (reference paths):
//   model/general_recommender/NeuMF.py:69-104   _create_inference / _create_loss
//   model/general_recommender/MLP.py:57-87      same for the MLP-only model
//   model/general_recommender/NeuMF.py:158-168  predict: one forward over ALL items per user
//   util/learner.py:18-41                       pairwise / pointwise losses
// Third-party arithmetic restated (tensorflow==1.12.3, not vendored): tf.layers.dense =
// relu(x . kernel + bias) with kernel [in, out]; ReluGrad passes dy where the OUTPUT is > 0;
// prediction = reduce_sum(concat(mf_vector, mlp_vector)) -- there is no output layer
// (NeuMF.py:85).  In pairwise NeuMF tf.layers.dense is re-instantiated for the negative tower,
// so the two towers have DIFFERENT weights (NeuMF.py:81-82, 90-92; n_towers = 2); MLP.py shares
// its Dense objects (n_towers = 1).
//
// Two kernels per step (the batch is tiny -- 256 samples x 6.7 k MACs -- so the design goal is
// latency, i.e. as many SMs as possible and no serial tail):
//   ncf_sample_kernel  one CTA (4 warps) per sample: gathers the embedding rows, runs the
//                      tower(s) forward and backward with the dense weights read through L1
//                      (27 KB, shared by every CTA on the SM), adds the embedding-row gradients
//                      to the dense accumulators (duplicates sum) and leaves activations and
//                      deltas of every layer in a scratch buffer;
//   ncf_wgrad_kernel   dW_l = A_l^T . Delta_l and db_l = colsum(Delta_l) over the batch: one
//                      thread per weight entry and batch slice, coalesced over the output
//                      column, one RED.ADD per entry and slice.
#include <stdlib.h>

#include "common.cuh"
#include "learner.cuh"
#include "ncf.cuh"
#include "optim.cuh"

namespace nrc {

int32_t g_ncf_routes[kNcfRoutes] = {-1, -1, -1, -1, -1, -1, -1};

void ncf_routes_reset() {
    for (int r = 0; r < kNcfRoutes; ++r) g_ncf_routes[r] = -1;
}

int ncf_make(NcfDev& S, const nrc_ncf_shape* sh) {
    NRC_REQUIRE(sh != nullptr, NRC_E_VALUE, "shape is NULL");
    NRC_REQUIRE(sh->n_layers >= 0 && sh->n_layers <= kNcfMaxLayers, NRC_E_LIMIT,
                "n_layers %d outside [0, %d]", sh->n_layers, kNcfMaxLayers);
    NRC_REQUIRE(sh->n_towers == 1 || sh->n_towers == 2, NRC_E_VALUE, "n_towers must be 1 or 2");
    NRC_REQUIRE(sh->mf_dim >= 0 && sh->mlp_dim >= 0 && (sh->mf_dim > 0 || sh->n_layers > 0),
                NRC_E_VALUE, "model has neither an MF nor an MLP part");
    NRC_REQUIRE(sh->n_layers == 0 || sh->mlp_dim > 0, NRC_E_VALUE, "mlp_dim must be > 0");
    NRC_REQUIRE(sh->mlp_dim <= 256 && sh->mf_dim <= 1024, NRC_E_LIMIT, "embedding width too large");
    S.mf_dim = sh->mf_dim; S.mlp_dim = sh->n_layers ? sh->mlp_dim : 0;
    S.n_layers = sh->n_layers; S.n_towers = sh->n_towers;
    int in = 2 * S.mlp_dim, off = 0, soff = 0, aoff = 0;
    S.a_off[0] = 0; aoff = in;
    for (int l = 0; l < kNcfMaxLayers; ++l) {
        if (l >= S.n_layers) {
            S.in_dim[l] = S.out_dim[l] = 0;
            S.w_off[l] = S.b_off[l] = S.sw_off[l] = S.sb_off[l] = 0;
            S.a_off[l + 1] = aoff;
            continue;
        }
        const int out = sh->layers[l];
        NRC_REQUIRE(out > 0 && out <= 512, NRC_E_LIMIT, "layer width %d outside [1, 512]", out);
        S.in_dim[l] = in; S.out_dim[l] = out;
        S.w_off[l] = off; off += in * out; S.b_off[l] = off; off += out;
        S.sw_off[l] = soff; soff += in * (out + 1); S.sb_off[l] = soff; soff += out;
        S.a_off[l + 1] = aoff; aoff += out;
        in = out;
    }
    S.tower_size = off; S.s_tower_size = soff; S.act_size = aoff;
    return NRC_OK;
}

__device__ __forceinline__ float block_sum_128(float v, float* red, int tid) {
    v = warp_sum(v);
    if ((tid & 31) == 0) red[tid >> 5] = v;
    __syncthreads();
    const float r = red[0] + red[1] + red[2] + red[3];
    __syncthreads();
    return r;
}

// ----------------------------------------------------------------------------------------
// per-sample forward + backward.  scratch layout per sample: [pass][act_size] activations then
// [pass][act_size] deltas (delta of a_{l+1} = gradient w.r.t. layer l's pre-activation).
// ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kNcfThreads)
ncf_sample_kernel(const NcfDev S, const NcfPtrs P, const int32_t* __restrict__ users,
                  const int32_t* __restrict__ items, const void* __restrict__ third, int64_t batch,
                  int pairwise, int loss_kind, float reg_mf, float reg_mlp, int32_t stamp,
                  float* __restrict__ scratch, float* __restrict__ loss) {
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x;
    const int passes = pairwise ? 2 : 1;
    float* sAct = sm;                                // [passes][act_size]
    float* sDel = sAct + passes * S.act_size;        // [passes][act_size]
    float* red = sDel + passes * S.act_size;         // [8]
    const int64_t b = blockIdx.x;
    const int u = users[b];
    const int it[2] = {items[b], pairwise ? reinterpret_cast<const int32_t*>(third)[b] : 0};

    float yhat[2] = {0.0f, 0.0f};
    for (int p = 0; p < passes; ++p) {
        float* act = sAct + p * S.act_size;
        float mf = 0.0f;
        for (int k = tid; k < S.mf_dim; k += kNcfThreads)
            mf = fmaf(P.mf_user[(size_t)u * S.mf_dim + k], P.mf_item[(size_t)it[p] * S.mf_dim + k], mf);
        for (int k = tid; k < S.mlp_dim; k += kNcfThreads) {
            act[k] = P.mlp_user[(size_t)u * S.mlp_dim + k];
            act[S.mlp_dim + k] = P.mlp_item[(size_t)it[p] * S.mlp_dim + k];
        }
        __syncthreads();
        const float* tw = P.dense + (size_t)((p == 1 && S.n_towers == 2) ? 1 : 0) * S.tower_size;
        for (int l = 0; l < S.n_layers; ++l) {
            const int in = S.in_dim[l], out = S.out_dim[l];
            const float* __restrict__ W = tw + S.w_off[l];
            const float* a = act + S.a_off[l];
            float* o = act + S.a_off[l + 1];
            for (int j = tid; j < out; j += kNcfThreads) {
                float acc = __ldg(tw + S.b_off[l] + j);
#pragma unroll 8
                for (int k = 0; k < in; ++k) acc = fmaf(a[k], __ldg(W + k * out + j), acc);
                o[j] = fmaxf(acc, 0.0f);  // tf.nn.relu
            }
            __syncthreads();
        }
        float s = 0.0f;
        if (S.n_layers > 0)
            for (int j = tid; j < S.out_dim[S.n_layers - 1]; j += kNcfThreads) s += act[S.a_off[S.n_layers] + j];
        yhat[p] = block_sum_128(mf + s, red, tid);   // NeuMF.py:85 reduce_sum(concat(mf, mlp))
    }

    float l, g;
    if (pairwise)   // NeuMF.py:92 result = output - output_neg
        pairwise_loss_grad(loss_kind, yhat[0] - yhat[1], l, g);
    else
        pointwise_loss_grad(loss_kind, yhat[0], reinterpret_cast<const float*>(third)[b], 1.0f / (float)batch, l, g);

    float sq_mf = 0.f, sq_mlp = 0.f;
    for (int p = 0; p < passes; ++p) {
        const float gp = (p == 0) ? g : -g;
        const float* tw = P.dense + (size_t)((p == 1 && S.n_towers == 2) ? 1 : 0) * S.tower_size;
        float* act = sAct + p * S.act_size;
        float* del = sDel + p * S.act_size;
        if (S.n_layers > 0) {
            const int L = S.n_layers;
            for (int j = tid; j < S.out_dim[L - 1]; j += kNcfThreads)
                del[S.a_off[L] + j] = (act[S.a_off[L] + j] > 0.0f) ? gp : 0.0f;
            __syncthreads();
            for (int l2 = L - 1; l2 >= 0; --l2) {
                const int in = S.in_dim[l2], out = S.out_dim[l2];
                const float* __restrict__ W = tw + S.w_off[l2];
                const float* d = del + S.a_off[l2 + 1];
                const float* a = act + S.a_off[l2];
                float* dp = del + S.a_off[l2];
                // one warp per input row k: lanes stride over the (contiguous) row => coalesced
                // weight reads, then a shuffle reduction
                const int lane = tid & 31, wrp = tid >> 5;
                for (int k = wrp; k < in; k += kNcfThreads / 32) {
                    const float* wr = W + (size_t)k * out;
                    float s = 0.0f;
                    for (int j = lane; j < out; j += kWarp) s = fmaf(__ldg(wr + j), d[j], s);
                    s = warp_sum(s);
                    if (lane == 0) dp[k] = (l2 > 0) ? ((a[k] > 0.0f) ? s : 0.0f) : s;
                }
                __syncthreads();
            }
        }
        // embedding-row gradients (IndexedSlices; duplicates sum) + regulariser terms
        for (int k = tid; k < S.mf_dim; k += kNcfThreads) {
            const float pu = P.mf_user[(size_t)u * S.mf_dim + k];
            const float qi = P.mf_item[(size_t)it[p] * S.mf_dim + k];
            atomicAdd(P.g_mf_user + (size_t)u * S.mf_dim + k, gp * qi + (p == 0 ? reg_mf * pu : 0.f));
            atomicAdd(P.g_mf_item + (size_t)it[p] * S.mf_dim + k, gp * pu + reg_mf * qi);
            sq_mf += qi * qi + (p == 0 ? pu * pu : 0.f);
        }
        for (int k = tid; k < S.mlp_dim; k += kNcfThreads) {
            const float mu = act[k], mi = act[S.mlp_dim + k];
            atomicAdd(P.g_mlp_user + (size_t)u * S.mlp_dim + k, del[k] + (p == 0 ? reg_mlp * mu : 0.f));
            atomicAdd(P.g_mlp_item + (size_t)it[p] * S.mlp_dim + k, del[S.mlp_dim + k] + reg_mlp * mi);
            sq_mlp += mi * mi + (p == 0 ? mu * mu : 0.f);
        }
        if (tid == 0) P.t_item[it[p]] = stamp;
    }
    if (tid == 0) P.t_user[u] = stamp;
    if (reg_mf != 0.f || reg_mlp != 0.f) {   // NeuMF.py:94-100
        const float r = block_sum_128(reg_mf * 0.5f * sq_mf + reg_mlp * 0.5f * sq_mlp, red, tid);
        l += r;
    }
    if (tid == 0 && loss) atomicAdd(loss, l);
    // activations and deltas for the weight-gradient kernel
    float* out_s = scratch + (size_t)b * (2 * passes * S.act_size);
    for (int e = tid; e < 2 * passes * S.act_size; e += kNcfThreads) out_s[e] = sm[e];
}

// ----------------------------------------------------------------------------------------
// Fast path for the reference's default tower (conf/NeuMF.properties, conf/MLP.properties:
// layers=[64,32,16], so IN0 = 64): every dimension is a compile-time constant, all 128 threads
// work in every layer (the k-range of a layer is split over thread groups and the partial sums
// are combined in a fixed order), weight rows are read fully coalesced in both directions.
// ----------------------------------------------------------------------------------------
// Weights are pre-loaded into registers (one batch of independent loads at the start of a pass),
// so the dependent chain layer -> layer never waits on global memory.
template <int IN, int OUT>
struct FwdW {
    static constexpr int G = kNcfThreads / OUT, KPG = IN / G;
    float w[KPG];
    float bias;
    __device__ __forceinline__ void load(const float* __restrict__ W, const float* __restrict__ B, int tid) {
        const int j = tid % OUT, g = tid / OUT;
#pragma unroll
        for (int kk = 0; kk < KPG; ++kk) w[kk] = __ldg(W + (g * KPG + kk) * OUT + j);
        bias = (tid < OUT) ? __ldg(B + tid) : 0.0f;
    }
    __device__ __forceinline__ void run(const float* a_in, float* a_out, float* part, int tid) const {
        const int g = tid / OUT;
        float acc = 0.0f;
#pragma unroll
        for (int kk = 0; kk < KPG; ++kk) acc = fmaf(a_in[g * KPG + kk], w[kk], acc);
        part[tid] = acc;
        __syncthreads();
        if (tid < OUT) {
            float s = bias;
#pragma unroll
            for (int q = 0; q < G; ++q) s += part[q * OUT + tid];
            a_out[tid] = fmaxf(s, 0.0f);  // tf.nn.relu
        }
        __syncthreads();
    }
};

template <int IN, int OUT, bool MASK>
struct BwdW {
    static constexpr int TPR = kNcfThreads / IN, JPT = OUT / TPR;   // threads per input row
    float w[JPT];
    __device__ __forceinline__ void load(const float* __restrict__ W, int tid) {
        const int k = tid / TPR, jq = tid % TPR;
#pragma unroll
        for (int jj = 0; jj < JPT; ++jj) w[jj] = __ldg(W + k * OUT + jq * JPT + jj);
    }
    __device__ __forceinline__ void run(const float* d_out, const float* a_in, float* d_in, int tid) const {
        const int k = tid / TPR, jq = tid % TPR;
        float s = 0.0f;
#pragma unroll
        for (int jj = 0; jj < JPT; ++jj) s = fmaf(w[jj], d_out[jq * JPT + jj], s);
#pragma unroll
        for (int o = TPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(kFull, s, o);
        if (jq == 0) d_in[k] = MASK ? ((a_in[k] > 0.0f) ? s : 0.0f) : s;
        __syncthreads();
    }
};

template <int IN0, int O0, int O1, int O2>
__global__ void __launch_bounds__(kNcfThreads)
ncf_sample_fast_kernel(const NcfDev S, const NcfPtrs P, const int32_t* __restrict__ users,
                       const int32_t* __restrict__ items, const void* __restrict__ third,
                       int64_t batch, int pairwise, int loss_kind, float reg_mf, float reg_mlp,
                       int32_t stamp, float* __restrict__ scratch, float* __restrict__ loss) {
    constexpr int ACT = IN0 + O0 + O1 + O2, A1 = IN0, A2 = IN0 + O0, A3 = IN0 + O0 + O1, MD = IN0 / 2;
    constexpr int W0 = 0, B0 = IN0 * O0, W1 = B0 + O0, B1 = W1 + O0 * O1, W2 = B1 + O1, B2 = W2 + O1 * O2;
    __shared__ __align__(16) float sm[4 * ACT + kNcfThreads + 8];
    const int tid = threadIdx.x;
    const int passes = pairwise ? 2 : 1;
    float* sAct = sm;
    float* sDel = sAct + passes * ACT;
    float* part = sm + 4 * ACT;
    float* red = part + kNcfThreads;
    const int64_t b = blockIdx.x;
    const int u = users[b];
    const int it[2] = {items[b], pairwise ? reinterpret_cast<const int32_t*>(third)[b] : 0};

    FwdW<IN0, O0> f0; FwdW<O0, O1> f1; FwdW<O1, O2> f2;
    BwdW<O1, O2, true> g2, h2; BwdW<O0, O1, true> g1, h1; BwdW<IN0, O0, false> g0, h0;   // pass 0 / pass 1
    float yhat[2] = {0.0f, 0.0f};
    for (int p = 0; p < passes; ++p) {
        float* act = sAct + p * ACT;
        float mf = 0.0f;
        for (int k = tid; k < S.mf_dim; k += kNcfThreads)
            mf = fmaf(P.mf_user[(size_t)u * S.mf_dim + k], P.mf_item[(size_t)it[p] * S.mf_dim + k], mf);
        if (tid < MD) act[tid] = P.mlp_user[(size_t)u * MD + tid];
        else if (tid < IN0) act[tid] = P.mlp_item[(size_t)it[p] * MD + (tid - MD)];
        __syncthreads();
        if (p == 0 || S.n_towers == 2) {   // (re)load this pass' tower into registers
            const float* tw = P.dense + (size_t)((p == 1) ? 1 : 0) * S.tower_size;
            f0.load(tw + W0, tw + B0, tid); f1.load(tw + W1, tw + B1, tid); f2.load(tw + W2, tw + B2, tid);
            if (p == 0) { g2.load(tw + W2, tid); g1.load(tw + W1, tid); g0.load(tw + W0, tid); }
            else { h2.load(tw + W2, tid); h1.load(tw + W1, tid); h0.load(tw + W0, tid); }
        }
        f0.run(act, act + A1, part, tid);
        f1.run(act + A1, act + A2, part, tid);
        f2.run(act + A2, act + A3, part, tid);
        const float s = (tid < O2) ? act[A3 + tid] : 0.0f;
        yhat[p] = block_sum_128(mf + s, red, tid);
    }

    float l, g;
    if (pairwise) pairwise_loss_grad(loss_kind, yhat[0] - yhat[1], l, g);
    else pointwise_loss_grad(loss_kind, yhat[0], reinterpret_cast<const float*>(third)[b], 1.0f / (float)batch, l, g);

    float sq_mf = 0.f, sq_mlp = 0.f;
    for (int p = 0; p < passes; ++p) {
        const float gp = (p == 0) ? g : -g;
        float* act = sAct + p * ACT;
        float* del = sDel + p * ACT;
        if (tid < O2) del[A3 + tid] = (act[A3 + tid] > 0.0f) ? gp : 0.0f;
        __syncthreads();
        if (p == 0 || S.n_towers == 1) {
            g2.run(del + A3, act + A2, del + A2, tid);
            g1.run(del + A2, act + A1, del + A1, tid);
            g0.run(del + A1, act, del, tid);
        } else {
            h2.run(del + A3, act + A2, del + A2, tid);
            h1.run(del + A2, act + A1, del + A1, tid);
            h0.run(del + A1, act, del, tid);
        }
        for (int k = tid; k < S.mf_dim; k += kNcfThreads) {
            const float pu = P.mf_user[(size_t)u * S.mf_dim + k];
            const float qi = P.mf_item[(size_t)it[p] * S.mf_dim + k];
            atomicAdd(P.g_mf_user + (size_t)u * S.mf_dim + k, gp * qi + (p == 0 ? reg_mf * pu : 0.f));
            atomicAdd(P.g_mf_item + (size_t)it[p] * S.mf_dim + k, gp * pu + reg_mf * qi);
            sq_mf += qi * qi + (p == 0 ? pu * pu : 0.f);
        }
        if (tid < MD) {
            const float mu = act[tid];
            atomicAdd(P.g_mlp_user + (size_t)u * MD + tid, del[tid] + (p == 0 ? reg_mlp * mu : 0.f));
            if (p == 0) sq_mlp += mu * mu;
        } else if (tid < IN0) {
            const float mi = act[tid];
            atomicAdd(P.g_mlp_item + (size_t)it[p] * MD + (tid - MD), del[tid] + reg_mlp * mi);
            sq_mlp += mi * mi;
        }
        if (tid == 0) P.t_item[it[p]] = stamp;
    }
    if (tid == 0) P.t_user[u] = stamp;
    if (reg_mf != 0.f || reg_mlp != 0.f)
        l += block_sum_128(reg_mf * 0.5f * sq_mf + reg_mlp * 0.5f * sq_mlp, red, tid);
    if (tid == 0 && loss) atomicAdd(loss, l);
    float* out_s = scratch + (size_t)b * (2 * passes * ACT);
    for (int e = tid; e < 2 * passes * ACT; e += kNcfThreads) out_s[e] = sm[e];
}

// dW_l[k][j] += sum_s a_l[s][k] * delta_l[s][j];  db_l[j] += sum_s delta_l[s][j]
// grid = (ceil(max_out/32), ceil((max_in+1)/8), n_layers * slices); block = (32, 8): thread
// (tx, ty) owns entry (k = tile_y*8 + ty, j = tile_x*32 + tx) of layer z / slices, row k == in
// being the bias; no integer division anywhere, delta reads coalesced over j.
__global__ void __launch_bounds__(256)
ncf_wgrad_kernel(const NcfDev S, float* __restrict__ g_dense, const float* __restrict__ scratch,
                 int64_t batch, int passes, int slices) {
    const int l = blockIdx.z / slices, slice = blockIdx.z - l * slices;
    const int in = S.in_dim[l], out = S.out_dim[l];
    const int j = blockIdx.x * 32 + threadIdx.x, k = blockIdx.y * 8 + threadIdx.y;
    if (j >= out || k > in) return;
    const bool is_bias = (k == in);
    const int64_t s0 = (batch * slice) / slices, s1 = (batch * (slice + 1)) / slices;
    const int stride = 2 * passes * S.act_size;
    const int e = is_bias ? (S.b_off[l] + j) : (S.w_off[l] + k * out + j);
    for (int p = 0; p < passes; ++p) {
        const int tower = (p == 1 && S.n_towers == 2) ? 1 : 0;
        const float* a = scratch + p * S.act_size + S.a_off[l] + (is_bias ? 0 : k);
        const float* d = scratch + (passes + p) * S.act_size + S.a_off[l + 1] + j;
        float acc = 0.0f;
#pragma unroll 8
        for (int64_t s = s0; s < s1; ++s) {
            const float dj = __ldg(d + s * stride);
            const float av = is_bias ? 1.0f : __ldg(a + s * stride);
            acc = fmaf(av, dj, acc);
        }
        if (acc != 0.0f) atomicAdd(g_dense + (size_t)tower * S.tower_size + e, acc);
    }
}

// predict for ALL items (NeuMF.py:163-168 / MLP.py:136-140): scores[b, i] = tower-0 forward.
// One warp per (user, item); weights staged in shared memory with row stride out+1.
__global__ void __launch_bounds__(kNcfWarps * 32)
ncf_scores_kernel(const NcfDev S, const NcfPtrs P, const int32_t* __restrict__ users, int n_users,
                  int num_items, float* __restrict__ scores) {
    extern __shared__ __align__(16) float sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* sW = sm;
    float* sAct = sW + S.s_tower_size;
    for (int l = 0; l < S.n_layers; ++l) {
        const int in = S.in_dim[l], out = S.out_dim[l];
#pragma unroll 4
        for (int k = warp; k < in; k += kNcfWarps)
            for (int j = lane; j < out; j += kWarp)
                sW[S.sw_off[l] + k * (out + 1) + j] = __ldg(P.dense + S.w_off[l] + k * out + j);
        for (int e = threadIdx.x; e < out; e += blockDim.x) sW[S.sb_off[l] + e] = P.dense[S.b_off[l] + e];
    }
    __syncthreads();
    float* act = sAct + warp * S.act_size;
    const int64_t total = (int64_t)n_users * num_items;
    for (int64_t e = (int64_t)blockIdx.x * kNcfWarps + warp; e < total; e += (int64_t)gridDim.x * kNcfWarps) {
        const int b = (int)(e / num_items), i = (int)(e - (int64_t)b * num_items);
        const int u = users[b];
        float mf = 0.0f;
        for (int k = lane; k < S.mf_dim; k += kWarp)
            mf = fmaf(P.mf_user[(size_t)u * S.mf_dim + k], P.mf_item[(size_t)i * S.mf_dim + k], mf);
        for (int k = lane; k < S.mlp_dim; k += kWarp) {
            act[k] = P.mlp_user[(size_t)u * S.mlp_dim + k];
            act[S.mlp_dim + k] = P.mlp_item[(size_t)i * S.mlp_dim + k];
        }
        __syncwarp();
        for (int l = 0; l < S.n_layers; ++l) {
            const int in = S.in_dim[l], out = S.out_dim[l];
            const float* W = sW + S.sw_off[l];
            const float* a = act + S.a_off[l];
            float* o = act + S.a_off[l + 1];
            for (int j = lane; j < out; j += kWarp) {
                float acc = sW[S.sb_off[l] + j];
#pragma unroll 8
                for (int k = 0; k < in; ++k) acc = fmaf(a[k], W[k * (out + 1) + j], acc);
                o[j] = fmaxf(acc, 0.0f);
            }
            __syncwarp();
        }
        float s = mf;
        if (S.n_layers > 0)
            for (int j = lane; j < S.out_dim[S.n_layers - 1]; j += kWarp) s += act[S.a_off[S.n_layers] + j];
        s = warp_sum(s);
        if (lane == 0) scores[e] = s;
        __syncwarp();
    }
}

// ----------------------------------------------------------------------------------------
// Fast predict for the reference's default tower (layers [64, 32, 16], mlp_dim 32; NeuMF.py:163-168 /
// MLP.py:136-140 score every item for every test user).  The first layer factorises over the concat:
//   relu([mu, mi] W0 + b0) = relu(A_u + B_i),  A_u = mu W0[:32] + b0 (per user),  B_i = mi W0[32:] (per item)
// so the 64x64 layer costs 64 adds per (user, item) pair once B is tabulated (ncf_item_part_kernel, stored
// TRANSPOSED [64][ldb] so that an item tile is 64 contiguous runs).  Layers 2 and 3 are
// [pairs, 64] x [64, 32] x [32, 16] products done as register-blocked SIMT GEMMs by a 256-thread CTA on
// tiles of 128 items:
//   work unit = (group of 4 users, item tile); the tile of B^T is staged in shared memory ONCE per unit and
//   reused by the 4 users, two at a time (one per 128-thread half of the CTA);
//   layer 2: thread (ti, tj) owns a 4-item x 8-column block: per k one float4 of h1^T (conflict-free) and two
//   float4 of W1 (warp-uniform -> broadcast) feed 32 FMAs.  (The first warp-per-32-pairs kernel fed 4 FMAs per
//   shared-memory load and ran at 1/6 of the fp32 peak; a 4 x 4 block sits exactly on the 128 B/clk
//   shared-memory limit.)
//   layer 3: thread = item with all 16 columns: 16 FMAs per 5 loads; relu, the 16 outputs and the GMF dot are
//   summed (NeuMF.py:85 reduce_sum(concat(mf, mlp))).
// fp32 FMA throughout: same values as the generic kernel up to the association of the sums.
// ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ncf_item_part_kernel(const float* __restrict__ mlp_item, const float* __restrict__ dense, int num_items, int ldb,
                     float* __restrict__ Bt) {
    // Bt[j][i] = sum_k mlp_item[i][k] * W0[32 + k][j];  thread = (j, item) with the item fastest
    __shared__ float sW[32 * 64];
    for (int e = threadIdx.x; e < 32 * 64; e += blockDim.x) sW[e] = dense[32 * 64 + e];
    __syncthreads();
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (int64_t)ldb * 64; t += (int64_t)gridDim.x * blockDim.x) {
        const int j = (int)(t / ldb), i = (int)(t - (int64_t)j * ldb);
        float acc = 0.0f;
        if (i < num_items) {
#pragma unroll 8
            for (int k = 0; k < 32; ++k) acc = fmaf(__ldg(mlp_item + (size_t)i * 32 + k), sW[k * 64 + j], acc);
        }
        Bt[t] = acc;
    }
}

// A[r][j] = b0[j] + sum_k mlp_user[users[r]][k] * W0[k][j] for the evaluated users (one thread per entry, j fastest)
__global__ void __launch_bounds__(256)
ncf_user_part_kernel(const float* __restrict__ mlp_user, const float* __restrict__ dense, const int32_t* __restrict__ users,
                     int n_users, float* __restrict__ A) {
    __shared__ float sW[32 * 64];
    for (int e = threadIdx.x; e < 32 * 64; e += blockDim.x) sW[e] = dense[e];
    __syncthreads();
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (int64_t)n_users * 64; t += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(t >> 6), j = (int)(t & 63);
        const int u = __ldg(users + r);
        float acc = __ldg(dense + 64 * 64 + j);
#pragma unroll 8
        for (int k = 0; k < 32; ++k) acc = fmaf(__ldg(mlp_user + (size_t)u * 32 + k), sW[k * 64 + j], acc);
        A[t] = acc;
    }
}

constexpr int kTileItems = 128, kTileUsers = 4;
constexpr int kTS = kTileItems + 4;       // row stride (floats) of the [k][item] tiles: rows stay 16-byte aligned

// 256 threads = two halves of 128; a half works on ONE user of the current pair: thread (ti, tj) of a half owns
// items 4ti..4ti+3 and columns 8tj..8tj+7 of layer 2 (32 accumulators; per k one float4 of h1^T and two
// warp-uniform float4 of W1 feed 32 FMAs: 6 shared-memory wavefronts per 32 FMA instructions, under the
// 128 B/clk shared-memory limit that a 4 x 4 block sits on), then item `t` with all 16 columns of layer 3.
__global__ void __launch_bounds__(256, 1)
ncf_scores_tile_kernel(const float* __restrict__ mf_user, const float* __restrict__ mf_item, int mf_dim,
                       const float* __restrict__ Au, const float* __restrict__ dense,
                       const float* __restrict__ Bt, int ldb, const int32_t* __restrict__ users, int n_users,
                       int num_items, float* __restrict__ scores) {
    extern __shared__ __align__(16) float sm[];
    constexpr int B0o = 64 * 64, W1o = B0o + 64, B1o = W1o + 64 * 32, W2o = B1o + 32, B2o = W2o + 32 * 16;
    float* sW1 = sm;                                  // [64][32]
    float* sW2 = sW1 + 64 * 32;                       // [32][16]
    float* sb1 = sW2 + 32 * 16;                       // [32]
    float* sb2 = sb1 + 32;                            // [16]
    float* sA = sb2 + 16;                             // [4][64]   A_u of the unit's users
    float* sBt = sA + kTileUsers * 64;                // [64][kTS] B^T tile
    float* h1t = sBt + 64 * kTS;                      // [2][64][kTS] relu(A_u + B_i), transposed, per half
    float* h2t = h1t + 2 * 64 * kTS;                  // [2][32][kTS]
    float* sMfU = h2t + 2 * 32 * kTS;                 // [4][mf_dim]
    const int tid = threadIdx.x;
    for (int e = tid; e < 64 * 32; e += 256) sW1[e] = __ldg(dense + W1o + e);
    for (int e = tid; e < 32 * 16; e += 256) sW2[e] = __ldg(dense + W2o + e);
    if (tid < 32) sb1[tid] = __ldg(dense + B1o + tid);
    if (tid < 16) sb2[tid] = __ldg(dense + B2o + tid);
    const int n_tiles = (num_items + kTileItems - 1) / kTileItems;
    const int n_groups = (n_users + kTileUsers - 1) / kTileUsers;
    const int half = tid >> 7, t = tid & 127;
    const int ti = t & 31, tj = t >> 5;               // layer 2: items 4ti.., columns 8tj..
    float* h1 = h1t + half * 64 * kTS;
    float* h2 = h2t + half * 32 * kTS;
    for (int unit = blockIdx.x; unit < n_groups * n_tiles; unit += gridDim.x) {
        const int ug = unit / n_tiles, tile = unit - ug * n_tiles;
        const int i0 = tile * kTileItems, u0 = ug * kTileUsers;
        __syncthreads();                              // the previous unit's last reads of sMfU, sBt, sA
        // ---- stage the unit: B^T tile, A_u and GMF rows of the 4 users
        for (int e = tid; e < 64 * (kTileItems / 4); e += 256) {
            const int k = e / (kTileItems / 4), c4 = (e % (kTileItems / 4)) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i0 + c4 < ldb) v = __ldg(reinterpret_cast<const float4*>(Bt + (size_t)k * ldb + i0 + c4));   // ldb % 4 == 0, zero padded
            *reinterpret_cast<float4*>(sBt + k * kTS + c4) = v;
        }
        {
            const int uu = tid >> 6, k = tid & 63;
            const bool live = u0 + uu < n_users;
            const int u = live ? __ldg(users + u0 + uu) : 0;
            sA[uu * 64 + k] = live ? __ldg(Au + (size_t)(u0 + uu) * 64 + k) : 0.0f;
            for (int m = k; m < mf_dim; m += 64) sMfU[uu * mf_dim + m] = live ? __ldg(mf_user + (size_t)u * mf_dim + m) : 0.0f;
        }
        __syncthreads();
        for (int pass = 0; pass < kTileUsers / 2 && u0 + 2 * pass < n_users; ++pass) {
            const int uu = 2 * pass + half;           // this half's user slot (may be past the end: computed, not stored)
            // h1^T = relu(A_u + B^T), this half's user
            for (int e = t; e < 64 * (kTileItems / 4); e += 128) {
                const int k = e / (kTileItems / 4), c4 = (e % (kTileItems / 4)) * 4;
                const float a = sA[uu * 64 + k];
                float4 v = *reinterpret_cast<const float4*>(sBt + k * kTS + c4);
                v.x = fmaxf(v.x + a, 0.f); v.y = fmaxf(v.y + a, 0.f); v.z = fmaxf(v.z + a, 0.f); v.w = fmaxf(v.w + a, 0.f);
                *reinterpret_cast<float4*>(h1 + k * kTS + c4) = v;
            }
            __syncthreads();
            // layer 2: acc[i][c] = sum_k h1[4ti + i][k] * W1[k][8tj + c]
            float acc[4][8];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int c = 0; c < 8; ++c) acc[i][c] = 0.0f;
#pragma unroll 4
            for (int k = 0; k < 64; ++k) {
                const float4 a = *reinterpret_cast<const float4*>(h1 + k * kTS + 4 * ti);
                const float4 w0 = *reinterpret_cast<const float4*>(sW1 + k * 32 + 8 * tj);
                const float4 w1 = *reinterpret_cast<const float4*>(sW1 + k * 32 + 8 * tj + 4);
                const float av[4] = {a.x, a.y, a.z, a.w};
                const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int c = 0; c < 8; ++c) acc[i][c] = fmaf(av[i], wv[c], acc[i][c]);
            }
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const float b = sb1[8 * tj + c];
                *reinterpret_cast<float4*>(h2 + (8 * tj + c) * kTS + 4 * ti) =
                    make_float4(fmaxf(acc[0][c] + b, 0.f), fmaxf(acc[1][c] + b, 0.f), fmaxf(acc[2][c] + b, 0.f), fmaxf(acc[3][c] + b, 0.f));
            }
            __syncthreads();
            // layer 3 (item t, all 16 columns) + relu + sum + GMF dot
            float o[16];
#pragma unroll
            for (int c = 0; c < 16; ++c) o[c] = sb2[c];
#pragma unroll 4
            for (int k = 0; k < 32; ++k) {
                const float a = h2[k * kTS + t];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float4 w = *reinterpret_cast<const float4*>(sW2 + k * 16 + 4 * q);
                    o[4 * q + 0] = fmaf(a, w.x, o[4 * q + 0]); o[4 * q + 1] = fmaf(a, w.y, o[4 * q + 1]);
                    o[4 * q + 2] = fmaf(a, w.z, o[4 * q + 2]); o[4 * q + 3] = fmaf(a, w.w, o[4 * q + 3]);
                }
            }
            float sacc = 0.0f;
#pragma unroll
            for (int c = 0; c < 16; ++c) sacc += fmaxf(o[c], 0.0f);
            if (u0 + uu < n_users && i0 + t < num_items) {
                float mf = 0.0f;                              // GMF dot: the item row is one or two L1-resident lines
                const float* q = mf_item + (size_t)(i0 + t) * mf_dim;
#pragma unroll 4
                for (int k = 0; k < mf_dim; ++k) mf = fmaf(sMfU[uu * mf_dim + k], __ldg(q + k), mf);
                scores[(size_t)(u0 + uu) * num_items + i0 + t] = mf + sacc;
            }
        }
    }
}

static float* g_user_part = nullptr;
static size_t g_user_part_floats = 0;
static float* g_item_part = nullptr;
static size_t g_item_part_floats = 0;

// library-owned scratch for activations / deltas, grown on demand (never inside a capture:
// callers warm up once before capturing a step graph)
static float* g_scratch = nullptr;
static size_t g_scratch_floats = 0;

static int ncf_launch_grad(const nrc_ncf_shape* shape, const NcfPtrs& P, const int32_t* users,
                           const int32_t* items, const void* third, int64_t batch, int pairwise,
                           int loss_kind, float reg_mf, float reg_mlp, int32_t stamp, float* loss,
                           cudaStream_t st) {
    NcfDev S;
    int rc = ncf_make(S, shape);
    if (rc) return rc;
    if (pairwise)
        NRC_REQUIRE(loss_kind == NRC_LOSS_BPR || loss_kind == NRC_LOSS_HINGE || loss_kind == NRC_LOSS_SQUARE,
                    NRC_E_VALUE, "please choose a suitable loss function");
    else
        NRC_REQUIRE(loss_kind == NRC_LOSS_CROSS_ENTROPY || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                    "please choose a suitable loss function");
    if (batch <= 0) return NRC_OK;
    const int passes = pairwise ? 2 : 1;
    const size_t per_sample = (size_t)2 * passes * S.act_size;
    const size_t need = per_sample * (size_t)batch;
    if (need > g_scratch_floats) {
        if (g_scratch) NRC_CUDA_CHECK(cudaFree(g_scratch));
        g_scratch = nullptr; g_scratch_floats = 0;
        const size_t cap = need + need / 2 + 1024;
        NRC_CUDA_CHECK(cudaMalloc(&g_scratch, cap * sizeof(float)));
        g_scratch_floats = cap;
    }
    const size_t smem = (per_sample + 8) * sizeof(float);
    NRC_REQUIRE(smem <= 48 * 1024, NRC_E_LIMIT, "NCF tower too wide: %zu B of shared memory", smem);
    const bool fast = S.n_layers == 3 && S.in_dim[0] == 64 && S.out_dim[0] == 64 &&
                      S.out_dim[1] == 32 && S.out_dim[2] == 16;
    const int slices = (batch >= 64) ? kWgradSlices : 1;
    ncf_routes_reset();
    g_ncf_routes[kRouteSampleFast] = fast ? 1 : 0;
    g_ncf_routes[kRouteWgradSlices] = S.n_layers > 0 ? slices : 0;
    if (fast)
        ncf_sample_fast_kernel<64, 64, 32, 16><<<(unsigned)batch, kNcfThreads, 0, st>>>(
            S, P, users, items, third, batch, pairwise, loss_kind, reg_mf, reg_mlp, stamp, g_scratch, loss);
    else
        ncf_sample_kernel<<<(unsigned)batch, kNcfThreads, smem, st>>>(S, P, users, items, third, batch,
                                                                      pairwise, loss_kind, reg_mf, reg_mlp,
                                                                      stamp, g_scratch, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    if (S.n_layers > 0) {
        int max_in = 0, max_out = 0;
        for (int l = 0; l < S.n_layers; ++l) {
            max_in = S.in_dim[l] > max_in ? S.in_dim[l] : max_in;
            max_out = S.out_dim[l] > max_out ? S.out_dim[l] : max_out;
        }
        dim3 grid((max_out + 31) / 32, (max_in + 1 + 7) / 8, S.n_layers * slices);
        ncf_wgrad_kernel<<<grid, dim3(32, 8), 0, st>>>(S, P.g_dense, g_scratch, batch, passes, slices);
        NRC_CUDA_CHECK(cudaGetLastError());
    }
    return NRC_OK;
}

}  // namespace nrc

using namespace nrc;

extern "C" int nrc_ncf_dense_size(const nrc_ncf_shape* shape) {
    NcfDev S;
    if (ncf_make(S, shape)) return NRC_E_VALUE;
    return S.tower_size * S.n_towers;
}

// Host bookkeeping of the code paths the most recent NCF call launched (see the header); no device work.
extern "C" int nrc_ncf_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "NULL output");
    for (int r = 0; r < kNcfRoutes; ++r) out[r] = g_ncf_routes[r];
    return NRC_OK;
}

extern "C" int nrc_ncf_grad(const nrc_ncf_shape* shape, const float* mf_user, const float* mf_item,
                            const float* mlp_user, const float* mlp_item, const float* dense,
                            const int32_t* users, const int32_t* items, const void* third,
                            int64_t batch, int32_t pairwise, int32_t loss_kind, float reg_mf,
                            float reg_mlp, float* g_mf_user, float* g_mf_item, float* g_mlp_user,
                            float* g_mlp_item, float* g_dense, int32_t* touched_user,
                            int32_t* touched_item, int32_t stamp, float* loss, void* stream) {
    NcfPtrs P{mf_user, mf_item, mlp_user, mlp_item, dense, g_mf_user, g_mf_item, g_mlp_user,
              g_mlp_item, g_dense, touched_user, touched_item};
    return ncf_launch_grad(shape, P, users, items, third, batch, pairwise, loss_kind, reg_mf,
                           reg_mlp, stamp, loss, as_stream(stream));
}

extern "C" int nrc_ncf_scores(const nrc_ncf_shape* shape, const float* mf_user, const float* mf_item,
                              const float* mlp_user, const float* mlp_item, const float* dense,
                              const int32_t* users, int32_t n_users, int32_t num_items,
                              float* scores, void* stream) {
    NcfDev S;
    int rc = ncf_make(S, shape);
    if (rc) return rc;
    if (n_users <= 0) return NRC_OK;
    S.n_towers = 1;
    NcfPtrs P{mf_user, mf_item, mlp_user, mlp_item, dense, nullptr, nullptr, nullptr, nullptr,
              nullptr, nullptr, nullptr};
    const bool fast = S.n_layers == 3 && S.mlp_dim == 32 && S.out_dim[0] == 64 && S.out_dim[1] == 32 && S.out_dim[2] == 16 &&
                      S.mf_dim <= 64 && !getenv("NRC_NCF_SCORES_GENERIC");
    if (fast) {
        const int ldb = (num_items + 3) & ~3;
        const size_t need = (size_t)ldb * 64;
        if (need > g_item_part_floats) {
            if (g_item_part) NRC_CUDA_CHECK(cudaFree(g_item_part));
            g_item_part = nullptr; g_item_part_floats = 0;
            NRC_CUDA_CHECK(cudaMalloc(&g_item_part, need * sizeof(float)));
            g_item_part_floats = need;
        }
        cudaStream_t st = as_stream(stream);
        int64_t pb = ((int64_t)ldb * 64 + 255) / 256;
        if (pb > (int64_t)sm_count() * 8) pb = (int64_t)sm_count() * 8;
        ncf_item_part_kernel<<<(unsigned)pb, 256, 0, st>>>(mlp_item, dense, num_items, ldb, g_item_part);
        NRC_CUDA_CHECK(cudaGetLastError());
        const size_t fsmem = ((size_t)64 * 32 + 32 * 16 + 32 + 16 + kTileUsers * 64 + 64 * kTS + 2 * 64 * kTS + 2 * 32 * kTS +
                              (size_t)kTileUsers * S.mf_dim) * 4;
        static bool fattr = false;
        if (!fattr) {
            NRC_CUDA_CHECK(cudaFuncSetAttribute(ncf_scores_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
            fattr = true;
        }
        ncf_routes_reset();
        g_ncf_routes[kRouteScoresTile] = 1;
        const int64_t units = (int64_t)((n_users + kTileUsers - 1) / kTileUsers) * ((num_items + kTileItems - 1) / kTileItems);
        int64_t grid = (int64_t)sm_count();
        if (grid > units) grid = units;
        const size_t need_u = (size_t)n_users * 64;
        if (need_u > g_user_part_floats) {
            if (g_user_part) NRC_CUDA_CHECK(cudaFree(g_user_part));
            g_user_part = nullptr; g_user_part_floats = 0;
            NRC_CUDA_CHECK(cudaMalloc(&g_user_part, need_u * sizeof(float)));
            g_user_part_floats = need_u;
        }
        int64_t ub = ((int64_t)n_users * 64 + 255) / 256;
        if (ub > (int64_t)sm_count() * 8) ub = (int64_t)sm_count() * 8;
        ncf_user_part_kernel<<<(unsigned)ub, 256, 0, st>>>(mlp_user, dense, users, n_users, g_user_part);
        NRC_CUDA_CHECK(cudaGetLastError());
        ncf_scores_tile_kernel<<<(unsigned)grid, 256, fsmem, st>>>(mf_user, mf_item, S.mf_dim, g_user_part, dense, g_item_part, ldb,
                                                                   users, n_users, num_items, scores);
        NRC_CUDA_CHECK(cudaGetLastError());
        return NRC_OK;
    }
    const size_t smem = ((size_t)S.s_tower_size + (size_t)kNcfWarps * S.act_size) * 4;
    NRC_REQUIRE(smem <= 200 * 1024, NRC_E_LIMIT, "NCF tower needs %zu B of shared memory", smem);
    static bool attr_done = false;
    if (!attr_done) {
        NRC_CUDA_CHECK(cudaFuncSetAttribute(ncf_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_done = true;
    }
    ncf_routes_reset();
    g_ncf_routes[kRouteScoresTile] = 0;
    const int64_t total = (int64_t)n_users * num_items;
    int64_t blocks = (total + kNcfWarps - 1) / kNcfWarps;
    const int64_t cap = (int64_t)sm_count() * 4;
    if (blocks > cap) blocks = cap;
    ncf_scores_kernel<<<(unsigned)blocks, kNcfWarps * 32, smem, as_stream(stream)>>>(S, P, users, n_users,
                                                                                    num_items, scores);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_ncf_train_epoch(const nrc_ncf_shape* shape, float* mf_user, float* mf_item,
                                   float* mlp_user, float* mlp_item, float* dense,
                                   const int32_t* users, const int32_t* items, const void* third,
                                   int64_t n, int32_t batch_size, int32_t pairwise, int32_t loss_kind,
                                   float reg_mf, float reg_mlp, int32_t opt_kind,
                                   const float* lr_t_host, const float* hyper_host,
                                   float* const* grads, float* const* slot0, float* const* slot1,
                                   int32_t* touched_user, int32_t* touched_item, int32_t first_stamp,
                                   float* step_loss, void* stream) {
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    NcfDev S;
    int rc = ncf_make(S, shape);
    if (rc) return rc;
    cudaStream_t st = as_stream(stream);
    const int64_t steps = (n + batch_size - 1) / batch_size;
    if (steps == 0) return NRC_OK;
    NRC_CUDA_CHECK(cudaMemsetAsync(step_loss, 0, (size_t)steps * sizeof(float), st));
    float hyper[4] = {hyper_host[0], hyper_host[1], hyper_host[2], hyper_host[3]};
    float* vars[5] = {mf_user, mf_item, mlp_user, mlp_item, dense};
    const int64_t rows[5] = {shape->num_users, shape->num_items, shape->num_users, shape->num_items, 1};
    const int dims[5] = {S.mf_dim, S.mf_dim, S.mlp_dim, S.mlp_dim, S.tower_size * S.n_towers};
    const int32_t* tch[5] = {touched_user, touched_item, touched_user, touched_item, nullptr};
    NcfPtrs P{mf_user, mf_item, mlp_user, mlp_item, dense, grads[0], grads[1], grads[2], grads[3],
              grads[4], touched_user, touched_item};
    for (int64_t s = 0; s < steps; ++s) {
        const int64_t off = s * batch_size;
        const int64_t bs = (n - off < batch_size) ? (n - off) : batch_size;
        const int32_t stamp = first_stamp + (int32_t)s;
        const void* th = pairwise ? (const void*)(reinterpret_cast<const int32_t*>(third) + off)
                                  : (const void*)(reinterpret_cast<const float*>(third) + off);
        rc = ncf_launch_grad(shape, P, users + off, items + off, th, bs, pairwise, loss_kind, reg_mf,
                             reg_mlp, stamp, step_loss + s, st);
        if (rc) return rc;
        if (opt_kind == NRC_OPT_ADAM) hyper[0] = lr_t_host[s];
        OptLaunch L;
        rc = opt_launch_init(L, opt_kind, hyper);
        if (rc) return rc;
        for (int v = 0; v < 5; ++v) {
            if (dims[v] == 0) continue;
            rc = opt_launch_add(L, vars[v], grads[v], slot0 ? slot0[v] : nullptr,
                                slot1 ? slot1[v] : nullptr, tch[v], rows[v], dims[v], v == 4);
            if (rc) return rc;
        }
        rc = opt_launch_run(L, stamp, st);
        if (rc) return rc;
    }
    return NRC_OK;
}
