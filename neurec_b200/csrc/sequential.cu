// The sequential recommenders that score with embedding tables, fed by the time-ordered samplers: FPMC and TransRec
// at high_order = 1 (one recent item per sample), HRM and NPE over a window of the L most recent items, FPMCplus with
// attention over that window conditioned on the candidate item.
//
// Replaces (reference paths):
//   model/sequential_recommender/FPMC.py:61-84       _create_inference / _create_loss (four tables, pairwise / pointwise)
//   model/sequential_recommender/FPMC.py:97-134      train_model's batch loop (sess.run((loss, optimizer)) per batch)
//   model/sequential_recommender/FPMC.py:140-165     predict
//   model/sequential_recommender/TransRec.py:66-91   _create_inference / _create_loss (squared translation distance)
//   model/sequential_recommender/TransRec.py:110-147 train_model's batch loop
//   model/sequential_recommender/TransRec.py:102-107,153-166  prediction graph (Euclidean distance, not squared)
//   model/sequential_recommender/HRM.py:54-91,104-129  pooled window, pooled user, loss; train_model's batch loop
//   model/sequential_recommender/NPE.py:54-71,84-108   summed window, relu products, loss; train_model's batch loop
//   model/sequential_recommender/HRM.py:135-163, NPE.py:114-142  predict (query rows here, scores by nrc_mf_scores)
//   model/sequential_recommender/FPMCplus.py:73-119,141-171  attention MLP, loss, train_model's batch loop
//   model/sequential_recommender/FPMCplus.py:177-205  predict (a per-(user, item) kernel: the attention depends on the item)
//
// None of the training scores is the inner product of one user row and one item row, so none goes through the MF
// kernels:
//   FPMC       x(u, l, i) = <UI_u, IU_i> + <IL_i, LI_l>
//   TransRec   x(u, l, i) = b_i - |(P_u + g) + Q_l - Q_i|^2          (training)
//              s(u, l, j) = b_j - |(P_u + g) + Q_l - Q_j|             (prediction)
//   HRM        x(u, w, i) = <pool_P(P_u, pool_S(E[w_0..L-1])), E_i>
//   NPE        x(u, w, i) = <relu(UI_u), relu(IU_i)> + <relu(IU_i), relu(sum_l IL[w_l])>
// Every gradient kernel runs one warp per sample and adds row gradients into dense accumulators with atomics
// (duplicate ids sum, as TF's IndexedSlices de-duplication does).  TransRec's global vector g enters every sample; its
// gradient is summed per warp, then per CTA in warp order, then across CTAs in CTA order by the last CTA to finish --
// a fixed order for a given batch size, and no atomics onto the same d floats.
#include "common.cuh"
#include "learner.cuh"
#include "optim.cuh"
#include "seq_epoch.cuh"

namespace nrc {

constexpr int kSeqMaxDim = 256;
constexpr int kSeqPerLane = kSeqMaxDim / kWarp;   // row elements one lane holds at the widest dim
constexpr int kSeqWarps = 8;                      // warps of a 256-thread CTA
constexpr int kTransRecCtas = 128;                // TransRec gradient grid cap: work holds one partial g per CTA
constexpr int kScoreRows = 8;                     // score kernels: (user, recent) rows per CTA
constexpr int kSeqMaxWindow = 64;                 // HRM / NPE: recent items per sample

static unsigned seq_grad_grid(int64_t batch, int64_t cap) {
    int64_t blocks = (batch + kSeqWarps - 1) / kSeqWarps;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

// Host record of what the most recent launch of each kernel group decided, for nrc_seq_last_routes (see the header);
// -1 = no such launch yet, or a field the group does not decide.  Written just before the launch, so a call that fails
// its checks or launches nothing leaves it as it was.
enum SeqKernel { kSeqFpmcGrad, kSeqTransRecGrad, kSeqHrmGrad, kSeqNpeGrad, kSeqFpmcScores, kSeqTransRecScores,
                 kSeqHrmQuery, kSeqNpeQuery, kSeqNpeRelu, kSeqKernels };
enum SeqRouteField { kSeqPairwise, kSeqSessionMax, kSeqPreMax, kSeqGridX, kSeqGridY, kSeqCapped, kSeqWindow,
                     kSeqFields };
static struct SeqRoutes {
    int32_t r[kSeqKernels][kSeqFields];
    SeqRoutes() { for (auto& k : r) for (auto& f : k) f = -1; }
} g_seq_routes;

static void seq_route(int kernel, int pairwise, int session_max, int pre_max, int64_t grid_x, int64_t grid_y,
                      int capped, int window) {
    int32_t* r = g_seq_routes.r[kernel];
    r[kSeqPairwise] = pairwise; r[kSeqSessionMax] = session_max; r[kSeqPreMax] = pre_max;
    r[kSeqGridX] = (int32_t)grid_x; r[kSeqGridY] = (int32_t)grid_y; r[kSeqCapped] = capped; r[kSeqWindow] = window;
}

// 1 when seq_grad_grid capped the grid, so a warp takes more than one sample
static int seq_grad_capped(int64_t batch, int64_t cap) { return (batch + kSeqWarps - 1) / kSeqWarps > cap ? 1 : 0; }

// ---------------------------------------------------------------------------------------------
// FPMC (FPMC.py:61-84).  c = dl/dx;
//   pairwise   x = x_i - x_j, reg * l2_loss(UI_u, IU_i, IL_i, LI_l, IU_j, IL_j)
//   pointwise  x = x_i,       reg * l2_loss(UI_u, IU_i, IL_i, LI_l)
// ---------------------------------------------------------------------------------------------
template <bool PAIRWISE>
__global__ void __launch_bounds__(256)
fpmc_grad_kernel(const float* __restrict__ UI, const float* __restrict__ IU, const float* __restrict__ IL,
                 const float* __restrict__ LI, int D, const int32_t* __restrict__ users, const int32_t* __restrict__ recent,
                 const int32_t* __restrict__ items, const void* __restrict__ third, int64_t batch, int loss_kind, float reg,
                 float inv_b, float* __restrict__ gUI, float* __restrict__ gIU, float* __restrict__ gIL,
                 float* __restrict__ gLI, int32_t* __restrict__ tU, int32_t* __restrict__ tI, int32_t* __restrict__ tL,
                 int32_t stamp, float* __restrict__ loss) {
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    float loss_acc = 0.0f;
    for (int64_t b = blockIdx.x * wpb + (threadIdx.x >> 5); b < batch; b += (int64_t)gridDim.x * wpb) {
        const int u = users[b], l = recent[b], i = items[b];
        const int j = PAIRWISE ? static_cast<const int32_t*>(third)[b] : 0;
        const size_t ou = (size_t)u * D, ol = (size_t)l * D, oi = (size_t)i * D, oj = (size_t)j * D;
        float xi = 0.f, xj = 0.f, sq = 0.f;
        for (int t = lane; t < D; t += kWarp) {
            const float a = UI[ou + t], ui = IU[oi + t], li = IL[oi + t], r = LI[ol + t];
            xi = fmaf(a, ui, xi); xi = fmaf(li, r, xi);
            sq += a * a + ui * ui + li * li + r * r;
            if (PAIRWISE) {
                const float uj = IU[oj + t], lj = IL[oj + t];
                xj = fmaf(a, uj, xj); xj = fmaf(lj, r, xj);
                sq += uj * uj + lj * lj;
            }
        }
        xi = warp_sum(xi);
        float lo, c;
        if (PAIRWISE) pairwise_loss_grad(loss_kind, xi - warp_sum(xj), lo, c);
        else pointwise_loss_grad(loss_kind, xi, static_cast<const float*>(third)[b], inv_b, lo, c);
        if (reg != 0.0f) lo += reg * 0.5f * warp_sum(sq);
        loss_acc += lo;
        for (int t = lane; t < D; t += kWarp) {
            const float a = UI[ou + t], ui = IU[oi + t], li = IL[oi + t], r = LI[ol + t];
            if (PAIRWISE) {
                const float uj = IU[oj + t], lj = IL[oj + t];
                atomicAdd(gUI + ou + t, c * (ui - uj) + reg * a);
                atomicAdd(gIU + oi + t, c * a + reg * ui);
                atomicAdd(gIU + oj + t, -c * a + reg * uj);
                atomicAdd(gIL + oi + t, c * r + reg * li);
                atomicAdd(gIL + oj + t, -c * r + reg * lj);
                atomicAdd(gLI + ol + t, c * (li - lj) + reg * r);
            } else {
                atomicAdd(gUI + ou + t, c * ui + reg * a);
                atomicAdd(gIU + oi + t, c * a + reg * ui);
                atomicAdd(gIL + oi + t, c * r + reg * li);
                atomicAdd(gLI + ol + t, c * li + reg * r);
            }
        }
        if (lane == 0) {
            tU[u] = stamp; tI[i] = stamp; tL[l] = stamp;
            if (PAIRWISE) tI[j] = stamp;
        }
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
}

// ---------------------------------------------------------------------------------------------
// TransRec (TransRec.py:66-91).  v_* = ((p + g) + r) - q_*, x_* = b_* - |v_*|^2, c = dl/dx;
//   dx/d{p, g, r} = -2 v,  dx/dq = 2 v,  dx/db = 1
//   pairwise   x = x_i - x_j, reg * l2_loss(p, r, q_j, q_i, b_i, b_j, g)
//   pointwise  x = x_i,       reg * l2_loss(p, r, q_i, b_i, g)
// g is one [1, d] variable, so its reg term enters once per batch.  work: gridDim.x partial sums of g's gradient
// ([gridDim.x, D]) and, after kTransRecCtas * D floats, the CTA completion counter (0 on entry, 0 on exit).
// ---------------------------------------------------------------------------------------------
template <bool PAIRWISE>
__global__ void __launch_bounds__(256)
transrec_grad_kernel(const float* __restrict__ P, const float* __restrict__ Q, const float* __restrict__ B,
                     const float* __restrict__ G, int D, const int32_t* __restrict__ users,
                     const int32_t* __restrict__ recent, const int32_t* __restrict__ items, const void* __restrict__ third,
                     int64_t batch, int loss_kind, float reg, float inv_b, float* __restrict__ gP, float* __restrict__ gQ,
                     float* __restrict__ gB, float* __restrict__ gG, int32_t* __restrict__ tP, int32_t* __restrict__ tQ,
                     int32_t* __restrict__ tB, int32_t stamp, float* __restrict__ work, float* __restrict__ loss) {
    __shared__ float s_g[kSeqWarps][kSeqMaxDim];
    __shared__ bool s_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float dg[kSeqPerLane];
#pragma unroll
    for (int c = 0; c < kSeqPerLane; ++c) dg[c] = 0.0f;
    float loss_acc = 0.0f;
    for (int64_t b = blockIdx.x * kSeqWarps + warp; b < batch; b += (int64_t)gridDim.x * kSeqWarps) {
        const int u = users[b], l = recent[b], i = items[b];
        const int j = PAIRWISE ? static_cast<const int32_t*>(third)[b] : 0;
        const size_t ou = (size_t)u * D, ol = (size_t)l * D, oi = (size_t)i * D, oj = (size_t)j * D;
        float di = 0.f, dj = 0.f, sq = 0.f;
#pragma unroll
        for (int c = 0; c < kSeqPerLane; ++c) {
            const int t = lane + c * kWarp;
            if (t < D) {
                const float p = P[ou + t], r = Q[ol + t], qi = Q[oi + t];
                const float x = (p + G[t]) + r;          // user + tile(global) + recent (TransRec.py:75-76)
                const float vi = x - qi;
                di = fmaf(vi, vi, di);
                sq += p * p + r * r + qi * qi;
                if (PAIRWISE) {
                    const float qj = Q[oj + t], vj = x - qj;
                    dj = fmaf(vj, vj, dj);
                    sq += qj * qj;
                }
            }
        }
        const float bi = B[i], bj = PAIRWISE ? B[j] : 0.0f;
        const float xi = bi - warp_sum(di);
        float lo, c;
        if (PAIRWISE) pairwise_loss_grad(loss_kind, xi - (bj - warp_sum(dj)), lo, c);
        else pointwise_loss_grad(loss_kind, xi, static_cast<const float*>(third)[b], inv_b, lo, c);
        if (reg != 0.0f) lo += reg * 0.5f * (warp_sum(sq) + bi * bi + bj * bj);
        loss_acc += lo;
        const float c2 = 2.0f * c;
#pragma unroll
        for (int k = 0; k < kSeqPerLane; ++k) {
            const int t = lane + k * kWarp;
            if (t < D) {
                const float p = P[ou + t], r = Q[ol + t], qi = Q[oi + t];
                const float x = (p + G[t]) + r;
                const float vi = x - qi;
                float e;                                 // dl/d(p + g + r) without the reg terms
                if (PAIRWISE) {
                    const float qj = Q[oj + t], vj = x - qj;
                    e = -c2 * (vi - vj);
                    atomicAdd(gQ + oj + t, -c2 * vj + reg * qj);
                } else {
                    e = -c2 * vi;
                }
                atomicAdd(gP + ou + t, e + reg * p);
                atomicAdd(gQ + ol + t, e + reg * r);
                atomicAdd(gQ + oi + t, c2 * vi + reg * qi);
                dg[k] += e;
            }
        }
        if (lane == 0) {
            atomicAdd(gB + i, c + reg * bi);
            tP[u] = stamp; tQ[l] = stamp; tQ[i] = stamp; tB[i] = stamp;
            if (PAIRWISE) {
                atomicAdd(gB + j, -c + reg * bj);
                tQ[j] = stamp; tB[j] = stamp;
            }
        }
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);

    // g's gradient: this CTA's warps in warp order -> work[blockIdx.x]; the last CTA sums the CTAs in CTA order
#pragma unroll
    for (int k = 0; k < kSeqPerLane; ++k) {
        const int t = lane + k * kWarp;
        if (t < D) s_g[warp][t] = dg[k];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < D; t += blockDim.x) {
        float s = 0.0f;
#pragma unroll
        for (int w = 0; w < kSeqWarps; ++w) s += s_g[w][t];
        work[(size_t)blockIdx.x * D + t] = s;
    }
    __threadfence();
    __syncthreads();
    unsigned* done = reinterpret_cast<unsigned*>(work + (size_t)kTransRecCtas * D);
    if (threadIdx.x == 0) s_last = atomicAdd(done, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int t = threadIdx.x; t < D; t += blockDim.x) {
        float s = 0.0f;
        for (unsigned k = 0; k < gridDim.x; ++k) s += __ldcg(work + (size_t)k * D + t);
        gG[t] += s + reg * G[t];
    }
    if (warp == 0 && reg != 0.0f && loss) {
        float sq = 0.0f;
        for (int t = lane; t < D; t += kWarp) sq += G[t] * G[t];
        sq = warp_sum(sq);
        if (lane == 0) atomicAdd(loss, reg * 0.5f * sq);
    }
    if (threadIdx.x == 0) *done = 0u;
}

// ---------------------------------------------------------------------------------------------
// Scores of every item for kScoreRows (user, recent item) rows per CTA, one item per thread; the rows' query vectors
// sit in shared memory.  grid = (row groups, item tiles of 256).
// ---------------------------------------------------------------------------------------------
// FPMC.predict (FPMC.py:140-165): out[r, j] = <UI_u, IU_j> + <IL_j, LI_l>
__global__ void __launch_bounds__(256)
fpmc_scores_kernel(const float* __restrict__ UI, const float* __restrict__ IU, const float* __restrict__ IL,
                   const float* __restrict__ LI, int D, int32_t num_items, const int32_t* __restrict__ users,
                   const int32_t* __restrict__ recent, int64_t rows, float* __restrict__ out) {
    __shared__ float s_u[kScoreRows][kSeqMaxDim], s_l[kScoreRows][kSeqMaxDim];
    const int64_t r0 = (int64_t)blockIdx.x * kScoreRows;
    const int nr = (rows - r0 < kScoreRows) ? (int)(rows - r0) : kScoreRows;
    for (int e = threadIdx.x; e < kScoreRows * D; e += blockDim.x) {
        const int r = e / D, k = e - r * D;
        const bool live = r < nr;
        s_u[r][k] = live ? UI[(size_t)users[r0 + r] * D + k] : 0.0f;
        s_l[r][k] = live ? LI[(size_t)recent[r0 + r] * D + k] : 0.0f;
    }
    __syncthreads();
    const int64_t j = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
    if (j >= num_items) return;
    const float* __restrict__ iu = IU + (size_t)j * D;
    const float* __restrict__ il = IL + (size_t)j * D;
    float acc[kScoreRows];
#pragma unroll
    for (int r = 0; r < kScoreRows; ++r) acc[r] = 0.0f;
    for (int k = 0; k < D; ++k) {
        const float a = __ldg(iu + k), c = __ldg(il + k);
#pragma unroll
        for (int r = 0; r < kScoreRows; ++r) acc[r] = fmaf(c, s_l[r][k], fmaf(s_u[r][k], a, acc[r]));
    }
#pragma unroll
    for (int r = 0; r < kScoreRows; ++r)
        if (r < nr) out[(size_t)(r0 + r) * num_items + j] = acc[r];
}

// TransRec's prediction graph (TransRec.py:102-107): out[r, j] = b_j - sqrt(sum_k (x_k - Q_jk)^2), x = (P_u + g) + Q_l.
// The squared distance is summed from the differences themselves (no |x|^2 - 2 x.q + |q|^2 expansion, which cancels
// when x is close to q), so x == Q_j gives exactly b_j.
__global__ void __launch_bounds__(256)
transrec_scores_kernel(const float* __restrict__ P, const float* __restrict__ Q, const float* __restrict__ B,
                       const float* __restrict__ G, int D, int32_t num_items, const int32_t* __restrict__ users,
                       const int32_t* __restrict__ recent, int64_t rows, float* __restrict__ out) {
    __shared__ float s_x[kScoreRows][kSeqMaxDim];
    const int64_t r0 = (int64_t)blockIdx.x * kScoreRows;
    const int nr = (rows - r0 < kScoreRows) ? (int)(rows - r0) : kScoreRows;
    for (int e = threadIdx.x; e < kScoreRows * D; e += blockDim.x) {
        const int r = e / D, k = e - r * D;
        s_x[r][k] = r < nr ? (P[(size_t)users[r0 + r] * D + k] + G[k]) + Q[(size_t)recent[r0 + r] * D + k] : 0.0f;
    }
    __syncthreads();
    const int64_t j = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
    if (j >= num_items) return;
    const float* __restrict__ q = Q + (size_t)j * D;
    float acc[kScoreRows];
#pragma unroll
    for (int r = 0; r < kScoreRows; ++r) acc[r] = 0.0f;
    for (int k = 0; k < D; ++k) {
        const float a = __ldg(q + k);
#pragma unroll
        for (int r = 0; r < kScoreRows; ++r) {
            const float v = s_x[r][k] - a;
            acc[r] = fmaf(v, v, acc[r]);
        }
    }
    const float bj = __ldg(B + j);
#pragma unroll
    for (int r = 0; r < kScoreRows; ++r)
        if (r < nr) out[(size_t)(r0 + r) * num_items + j] = bj - sqrtf(acc[r]);
}

// ---------------------------------------------------------------------------------------------
// HRM (HRM.py:62-91), pointwise.  recent is i32 [batch, L], oldest first; c = dl/dx;
//   s = pool_S(E[w_0], ..., E[w_{L-1}]),  h = pool_P(P_u, s),  x = <h, E_i>,
//   l(z, x) + reg * l2_loss(P_u, E[w], E_i)
// Both pools are elementwise: max (SMAX / PMAX) or mean.  Backward as TF: the mean passes grad / count
// (_MeanGrad); the max passes (1 / n) * grad to each of the n inputs equal to the maximum (_MinOrMaxGrad: ties split).
// The window is gathered twice (forward, backward); a lane keeps only its elements of s, the tie counts and dl/ds.
// ---------------------------------------------------------------------------------------------
template <bool SMAX, bool PMAX>
__global__ void __launch_bounds__(256)
hrm_grad_kernel(const float* __restrict__ P, const float* __restrict__ E, int D, int L,
                const int32_t* __restrict__ users, const int32_t* __restrict__ recent, const int32_t* __restrict__ items,
                const float* __restrict__ labels, int64_t batch, int loss_kind, float reg, float inv_b,
                float* __restrict__ gP, float* __restrict__ gE, int32_t* __restrict__ tP, int32_t* __restrict__ tE,
                int32_t stamp, float* __restrict__ loss) {
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    const float fl = (float)L;
    float loss_acc = 0.0f;
    for (int64_t b = blockIdx.x * wpb + (threadIdx.x >> 5); b < batch; b += (int64_t)gridDim.x * wpb) {
        const int u = users[b], i = items[b];
        const int32_t* __restrict__ w = recent + b * L;
        const size_t ou = (size_t)u * D, oi = (size_t)i * D;
        float s[kSeqPerLane], cnt[kSeqPerLane], ds[kSeqPerLane];
#pragma unroll
        for (int c = 0; c < kSeqPerLane; ++c) { s[c] = SMAX ? -INFINITY : 0.0f; cnt[c] = 0.0f; }
        float sq = 0.0f, x = 0.0f;
        for (int k = 0; k < L; ++k) {
            const size_t ow = (size_t)w[k] * D;
#pragma unroll
            for (int c = 0; c < kSeqPerLane; ++c) {
                const int t = lane + c * kWarp;
                if (t < D) {
                    const float v = E[ow + t];
                    sq = fmaf(v, v, sq);
                    if (SMAX) {
                        if (v > s[c]) { s[c] = v; cnt[c] = 1.0f; }
                        else if (v == s[c]) cnt[c] += 1.0f;
                    } else {
                        s[c] += v;
                    }
                }
            }
        }
#pragma unroll
        for (int c = 0; c < kSeqPerLane; ++c) {
            const int t = lane + c * kWarp;
            if (t < D) {
                if (!SMAX) s[c] = s[c] / fl;
                const float p = P[ou + t], e = E[oi + t];
                const float h = PMAX ? fmaxf(p, s[c]) : (p + s[c]) / 2.0f;
                x = fmaf(h, e, x);
                sq += p * p + e * e;
            }
        }
        x = warp_sum(x);
        float lo, g;
        pointwise_loss_grad(loss_kind, x, labels[b], inv_b, lo, g);
        if (reg != 0.0f) lo += reg * 0.5f * warp_sum(sq);
        loss_acc += lo;
#pragma unroll
        for (int c = 0; c < kSeqPerLane; ++c) {
            const int t = lane + c * kWarp;
            if (t < D) {
                const float p = P[ou + t], e = E[oi + t];
                const float h = PMAX ? fmaxf(p, s[c]) : (p + s[c]) / 2.0f;
                const float dh = g * e;
                float dp;
                if (PMAX) {
                    const float share = 1.0f / ((p == s[c]) ? 2.0f : 1.0f);
                    dp = (p == h) ? share * dh : 0.0f;
                    ds[c] = (s[c] == h) ? share * dh : 0.0f;
                } else {
                    dp = dh / 2.0f;
                    ds[c] = dh / 2.0f;
                }
                atomicAdd(gP + ou + t, dp + reg * p);
                atomicAdd(gE + oi + t, g * h + reg * e);
            }
        }
        for (int k = 0; k < L; ++k) {
            const int wk = w[k];
            const size_t ow = (size_t)wk * D;
#pragma unroll
            for (int c = 0; c < kSeqPerLane; ++c) {
                const int t = lane + c * kWarp;
                if (t < D) {
                    const float v = E[ow + t];
                    const float dv = SMAX ? ((v == s[c]) ? (1.0f / cnt[c]) * ds[c] : 0.0f) : ds[c] / fl;
                    atomicAdd(gE + ow + t, dv + reg * v);
                }
            }
            if (lane == 0) tE[wk] = stamp;
        }
        if (lane == 0) { tP[u] = stamp; tE[i] = stamp; }
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
}

// ---------------------------------------------------------------------------------------------
// NPE (NPE.py:54-71), pointwise.  recent is i32 [batch, L]; c = dl/dx;
//   ctx = sum_l IL[w_l] (in window order),  x = sum_k relu(UI_u)_k relu(IU_i)_k + relu(IU_i)_k relu(ctx)_k,
//   l(z, x) + reg * l2_loss(UI_u, IU_i, IL[w])
// relu's gradient is TF's ReluGrad: zero where the input is <= 0.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
npe_grad_kernel(const float* __restrict__ UI, const float* __restrict__ IU, const float* __restrict__ IL, int D, int L,
                const int32_t* __restrict__ users, const int32_t* __restrict__ recent, const int32_t* __restrict__ items,
                const float* __restrict__ labels, int64_t batch, int loss_kind, float reg, float inv_b,
                float* __restrict__ gUI, float* __restrict__ gIU, float* __restrict__ gIL, int32_t* __restrict__ tU,
                int32_t* __restrict__ tI, int32_t* __restrict__ tL, int32_t stamp, float* __restrict__ loss) {
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    float loss_acc = 0.0f;
    for (int64_t b = blockIdx.x * wpb + (threadIdx.x >> 5); b < batch; b += (int64_t)gridDim.x * wpb) {
        const int u = users[b], i = items[b];
        const int32_t* __restrict__ w = recent + b * L;
        const size_t ou = (size_t)u * D, oi = (size_t)i * D;
        float ctx[kSeqPerLane];
#pragma unroll
        for (int c = 0; c < kSeqPerLane; ++c) ctx[c] = 0.0f;
        float sq = 0.0f, x = 0.0f;
        for (int k = 0; k < L; ++k) {
            const size_t ow = (size_t)w[k] * D;
#pragma unroll
            for (int c = 0; c < kSeqPerLane; ++c) {
                const int t = lane + c * kWarp;
                if (t < D) {
                    const float v = IL[ow + t];
                    ctx[c] += v;
                    sq = fmaf(v, v, sq);
                }
            }
        }
#pragma unroll
        for (int c = 0; c < kSeqPerLane; ++c) {
            const int t = lane + c * kWarp;
            if (t < D) {
                const float a = UI[ou + t], q = IU[oi + t];
                const float ra = fmaxf(a, 0.0f), rq = fmaxf(q, 0.0f), rc = fmaxf(ctx[c], 0.0f);
                x += ra * rq + rq * rc;
                sq += a * a + q * q;
            }
        }
        x = warp_sum(x);
        float lo, g;
        pointwise_loss_grad(loss_kind, x, labels[b], inv_b, lo, g);
        if (reg != 0.0f) lo += reg * 0.5f * warp_sum(sq);
        loss_acc += lo;
#pragma unroll
        for (int c = 0; c < kSeqPerLane; ++c) {
            const int t = lane + c * kWarp;
            if (t < D) {
                const float a = UI[ou + t], q = IU[oi + t];
                const float ra = fmaxf(a, 0.0f), rq = fmaxf(q, 0.0f), rc = fmaxf(ctx[c], 0.0f);
                atomicAdd(gUI + ou + t, (a > 0.0f ? g * rq : 0.0f) + reg * a);
                atomicAdd(gIU + oi + t, (q > 0.0f ? g * ra + g * rc : 0.0f) + reg * q);
                ctx[c] = ctx[c] > 0.0f ? g * rq : 0.0f;          // dl/dctx from here on
            }
        }
        for (int k = 0; k < L; ++k) {
            const int wk = w[k];
            const size_t ow = (size_t)wk * D;
#pragma unroll
            for (int c = 0; c < kSeqPerLane; ++c) {
                const int t = lane + c * kWarp;
                if (t < D) {
                    const float v = IL[ow + t];
                    atomicAdd(gIL + ow + t, ctx[c] + reg * v);
                }
            }
            if (lane == 0) tL[wk] = stamp;
        }
        if (lane == 0) { tU[u] = stamp; tI[i] = stamp; }
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
}

// ---------------------------------------------------------------------------------------------
// Query rows of HRM / NPE predict, one thread per (row, element).  Row r is user u = users[r] with its window
// recent[u, 0 .. recent_len[u]) (a per-user table of width L); pools run over the window's actual length.
// ---------------------------------------------------------------------------------------------
// HRM: out[r] = h = pool_P(P_u, pool_S(E[window]))
template <bool SMAX, bool PMAX>
__global__ void __launch_bounds__(256)
hrm_query_kernel(const float* __restrict__ P, const float* __restrict__ E, int D, int L,
                 const int32_t* __restrict__ users, const int32_t* __restrict__ recent,
                 const int32_t* __restrict__ recent_len, int64_t rows, float* __restrict__ out) {
    const int64_t total = rows * D;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / D;
        const int t = (int)(e - r * D);
        const int u = users[r], n = recent_len[u];
        const int32_t* __restrict__ w = recent + (size_t)u * L;
        float s = SMAX ? -INFINITY : 0.0f;
        for (int k = 0; k < n; ++k) {
            const float v = E[(size_t)w[k] * D + t];
            s = SMAX ? fmaxf(s, v) : s + v;
        }
        if (!SMAX) s = s / (float)n;
        const float p = P[(size_t)u * D + t];
        out[e] = PMAX ? fmaxf(p, s) : (p + s) / 2.0f;
    }
}

// NPE: out[r] = relu(UI_u) + relu(sum of IL over the window), so that <out[r], relu(IU_j)> is the score
__global__ void __launch_bounds__(256)
npe_query_kernel(const float* __restrict__ UI, const float* __restrict__ IL, int D, int L,
                 const int32_t* __restrict__ users, const int32_t* __restrict__ recent,
                 const int32_t* __restrict__ recent_len, int64_t rows, float* __restrict__ out) {
    const int64_t total = rows * D;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / D;
        const int t = (int)(e - r * D);
        const int u = users[r], n = recent_len[u];
        const int32_t* __restrict__ w = recent + (size_t)u * L;
        float ctx = 0.0f;
        for (int k = 0; k < n; ++k) ctx += IL[(size_t)w[k] * D + t];
        out[e] = fmaxf(UI[(size_t)u * D + t], 0.0f) + fmaxf(ctx, 0.0f);
    }
}

__global__ void __launch_bounds__(256)
relu_kernel(const float* __restrict__ in, int64_t n, float* __restrict__ out) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        out[e] = fmaxf(in[e], 0.0f);
}

// ---------------------------------------------------------------------------------------------
// argument checks shared by the entry points (all of them before any CUDA call: a rejected call writes nothing)
// ---------------------------------------------------------------------------------------------
static int seq_check(int32_t dim, int32_t pairwise, int32_t loss_kind, int64_t batch) {
    NRC_REQUIRE(dim >= 1 && dim <= kSeqMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kSeqMaxDim);
    // learner.py:27-28 / 39-40
    if (pairwise)
        NRC_REQUIRE(loss_kind == NRC_LOSS_BPR || loss_kind == NRC_LOSS_HINGE || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                    "please choose a suitable loss function");
    else
        NRC_REQUIRE(loss_kind == NRC_LOSS_CROSS_ENTROPY || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                    "please choose a suitable loss function");
    NRC_REQUIRE(batch >= 0, NRC_E_VALUE, "batch >= 0 required");
    return NRC_OK;
}

static int seq_check_epoch(int32_t dim, int32_t pairwise, int32_t loss_kind, int64_t n, int32_t batch_size,
                           int32_t opt_kind, const float* lr_t_host, const float* hyper_host) {
    const int rc = seq_check(dim, pairwise, loss_kind, n);
    if (rc) return rc;
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    // learner.py:14-15
    NRC_REQUIRE(opt_kind >= NRC_OPT_GD && opt_kind <= NRC_OPT_MOMENTUM, NRC_E_VALUE, "please select a suitable optimizer");
    NRC_REQUIRE(lr_t_host && hyper_host, NRC_E_VALUE, "lr_t_host and hyper_host are required");
    return NRC_OK;
}

static int seq_check_window(int32_t window) {
    NRC_REQUIRE(window >= 1 && window <= kSeqMaxWindow, NRC_E_LIMIT, "window %d outside [1, %d]", window,
                kSeqMaxWindow);
    return NRC_OK;
}

static int seq_check_query(int32_t dim, int32_t window, int64_t rows) {
    NRC_REQUIRE(dim >= 1 && dim <= kSeqMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kSeqMaxDim);
    const int rc = seq_check_window(window);
    if (rc) return rc;
    NRC_REQUIRE(rows >= 0, NRC_E_VALUE, "rows >= 0 required");
    return NRC_OK;
}

// ---------------------------------------------------------------------------------------------
// FPMCplus (FPMCplus.py:53-119): FPMC whose recent-item term is attention over a window conditioned on the
// candidate.  Variables UI [U, d], IU, IL, LI [I, d], W [3d, w] = [W_U; W_I; W_L], b [w], h [w].  For user u,
// window l_1..l_L and item i:
//   z_k = (A + B_i) + C_k with A = UI_u W_U + b, B_i = IL_i W_I, C_k = LI_{l_k} W_L   (the concat [u, i, l] W + b)
//   e_k = <h, tanh(z_k)>,  a_k = exp(e_k) / sum_k exp(e_k)   (no max shift, as :87-91: exp overflows to NaN there)
//   x   = <UI_u, IU_i> + <IL_i, sum_k a_k LI_{l_k}>
//   pairwise   l(x_i - x_j) + reg_mf * l2_loss(UI_u, IU_i, IL_i, LI_w, IU_j, IL_j) + reg_w * l2_loss(W, h)
//   pointwise  l(z, x_i)    + reg_mf * l2_loss(UI_u, IU_i, IL_i, LI_w)
// Backward with c_s = dl/dx_s (c_j = -c in the pairwise form), q_k = <IL_s, LI_{l_k}>, y = sum_k a_k q_k:
//   de_k = c_s a_k (q_k - y),  dz_k = de_k h * (1 - tanh(z_k)^2)   (TF's TanhGrad)
//   dW_U += UI_u (x) sum_k dz_k,  dW_I += IL_s (x) sum_k dz_k,  dW_L += LI_{l_k} (x) dz_k,  db += sum_k dz_k,
//   dh += sum_k de_k tanh(z_k);  the rows get the transposed products W_U sum_k dz_k, W_I sum_k dz_k, W_L dz_k.
// W, b and h enter every sample.  Their gradients are not accumulated with atomics: the gradient kernel writes each
// sample's factors (the vectors above) to work, and fpmcplus_wgrad_kernel forms the outer products over the batch in
// chunks of kFpmcPlusChunk samples, each chunk's sum in sample order, then the chunks in chunk order -- one fixed
// order for a given batch, so the dense gradients are the same bits on every run.
// ---------------------------------------------------------------------------------------------
constexpr int kFpmcPlusMaxWeight = 128;                         // weight_size cap (registers of the gradient kernel)
constexpr int kFpmcPlusPerLane = kFpmcPlusMaxWeight / kWarp;    // w elements one lane holds at the cap
constexpr int kFpmcPlusChunk = 32;                              // samples per partial sum of the dense gradients
constexpr int kFpmcPlusPairItems = 256;                         // score kernel: items per CTA, one per thread
constexpr int kFpmcPlusPairSmemFloats = 25600;                  // score kernel: shared-memory budget of the rows

// Per-sample factors of the dense gradients in work: [gA = sum of dz over both sides (W_U, b), gI (W_I from IL_i),
// gJ (W_I from IL_j), gH (h), gL_k = dz_ik + dz_jk for every window position k (W_L)], each w floats.
__host__ __device__ inline int64_t fpmcplus_factor_floats(int Wd, int L) { return (int64_t)(4 + L) * Wd; }
// dense gradient elements: W [3d, w], b [w], h [w]
__host__ __device__ inline int64_t fpmcplus_dense_floats(int D, int Wd) { return 3 * (int64_t)D * Wd + 2 * (int64_t)Wd; }
static int64_t fpmcplus_counters(int D, int Wd) { return (fpmcplus_dense_floats(D, Wd) + 255) / 256; }
static int64_t fpmcplus_chunks(int64_t batch) { return (batch + kFpmcPlusChunk - 1) / kFpmcPlusChunk; }

// out[q] (+)= sum_r x_r Wb[r, lane + 32 q]: a row vector held by the warp's lanes (element lane + 32 p in x[p]) times
// a [D, Wd] block, into the lane layout of a w-vector.
__device__ __forceinline__ void fpmcplus_proj(const float (&x)[kSeqPerLane], const float* __restrict__ Wb, int D,
                                              int Wd, int lane, float (&out)[kFpmcPlusPerLane]) {
#pragma unroll
    for (int p = 0; p < kSeqPerLane; ++p) {
        if (p * kWarp >= D) break;
#pragma unroll 1
        for (int s = 0; s < kWarp; ++s) {
            const int r = p * kWarp + s;
            if (r >= D) break;
            const float xr = __shfl_sync(kFull, x[p], s);
#pragma unroll
            for (int q = 0; q < kFpmcPlusPerLane; ++q) {
                const int c = lane + q * kWarp;
                if (c < Wd) out[q] = fmaf(xr, __ldg(Wb + (size_t)r * Wd + c), out[q]);
            }
        }
    }
}

// out[p] = sum_c Wb[lane + 32 p, c] g_c: a [D, Wd] block times a w-vector held in the w lane layout.
__device__ __forceinline__ void fpmcplus_back(const float (&g)[kFpmcPlusPerLane], const float* __restrict__ Wb, int D,
                                              int Wd, int lane, float (&out)[kSeqPerLane]) {
#pragma unroll
    for (int p = 0; p < kSeqPerLane; ++p) out[p] = 0.0f;
#pragma unroll
    for (int q = 0; q < kFpmcPlusPerLane; ++q) {
        if (q * kWarp >= Wd) break;
#pragma unroll 1
        for (int s = 0; s < kWarp; ++s) {
            const int c = q * kWarp + s;
            if (c >= Wd) break;
            const float gc = __shfl_sync(kFull, g[q], s);
#pragma unroll
            for (int p = 0; p < kSeqPerLane; ++p) {
                const int t = lane + p * kWarp;
                if (t < D) out[p] = fmaf(__ldg(Wb + (size_t)t * Wd + c), gc, out[p]);
            }
        }
    }
}

// sum_q h_q tanh((A_q + B_q) + C_q) over the warp
__device__ __forceinline__ float fpmcplus_energy(const float (&A)[kFpmcPlusPerLane], const float (&B)[kFpmcPlusPerLane],
                                                 const float (&C)[kFpmcPlusPerLane], const float (&H)[kFpmcPlusPerLane],
                                                 int Wd, int lane) {
    float e = 0.0f;
#pragma unroll
    for (int q = 0; q < kFpmcPlusPerLane; ++q)
        if (lane + q * kWarp < Wd) e = fmaf(H[q], tanhf((A[q] + B[q]) + C[q]), e);
    return warp_sum(e);
}

// One warp per sample.  Window scalars (e_k, q_k, then a_k, de_k) live in lane k % 32, register k / 32.  work holds
// the per-sample factors at fac + b * fpmcplus_factor_floats; the gL_k slots first hold C_k between the two passes.
template <bool PAIRWISE>
__global__ void __launch_bounds__(256, 1)
fpmcplus_grad_kernel(const float* __restrict__ UI, const float* __restrict__ IU, const float* __restrict__ IL,
                     const float* __restrict__ LI, const float* __restrict__ W, const float* __restrict__ Bv,
                     const float* __restrict__ Hv, int D, int Wd, int L, const int32_t* __restrict__ users,
                     const int32_t* __restrict__ recent, const int32_t* __restrict__ items,
                     const void* __restrict__ third, int64_t batch, int loss_kind, float reg, float reg_w, float inv_b,
                     float* __restrict__ gUI, float* __restrict__ gIU, float* __restrict__ gIL, float* __restrict__ gLI,
                     int32_t* __restrict__ tU, int32_t* __restrict__ tI, int32_t* __restrict__ tL, int32_t stamp,
                     float* __restrict__ fac, float* __restrict__ loss) {
    constexpr int P = kSeqPerLane, Q = kFpmcPlusPerLane;
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    const float* __restrict__ WU = W;
    const float* __restrict__ WI = W + (size_t)D * Wd;
    const float* __restrict__ WL = W + 2 * (size_t)D * Wd;
    float H[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) H[q] = (lane + q * kWarp < Wd) ? Hv[lane + q * kWarp] : 0.0f;
    float loss_acc = 0.0f;
    for (int64_t b = blockIdx.x * wpb + (threadIdx.x >> 5); b < batch; b += (int64_t)gridDim.x * wpb) {
        const int u = users[b], i = items[b];
        const int j = PAIRWISE ? static_cast<const int32_t*>(third)[b] : 0;
        const int32_t* __restrict__ win = recent + b * L;
        float* __restrict__ f = fac + b * fpmcplus_factor_floats(Wd, L);
        const size_t ou = (size_t)u * D, oi = (size_t)i * D, oj = (size_t)j * D;
        float a[P], ili[P], ilj[P];
        float xi = 0.f, xj = 0.f, sq = 0.f;
#pragma unroll
        for (int p = 0; p < P; ++p) {
            const int t = lane + p * kWarp;
            a[p] = ili[p] = ilj[p] = 0.0f;
            if (t < D) {
                a[p] = UI[ou + t]; ili[p] = IL[oi + t];
                const float ui = IU[oi + t];
                xi = fmaf(a[p], ui, xi);
                sq += a[p] * a[p] + ui * ui + ili[p] * ili[p];
                if (PAIRWISE) {
                    ilj[p] = IL[oj + t];
                    const float uj = IU[oj + t];
                    xj = fmaf(a[p], uj, xj);
                    sq += uj * uj + ilj[p] * ilj[p];
                }
            }
        }
        float A[Q], Bi[Q], Bj[Q], C[Q];
#pragma unroll
        for (int q = 0; q < Q; ++q) { A[q] = Bi[q] = Bj[q] = 0.0f; }
        fpmcplus_proj(a, WU, D, Wd, lane, A);
#pragma unroll
        for (int q = 0; q < Q; ++q) if (lane + q * kWarp < Wd) A[q] += Bv[lane + q * kWarp];
        fpmcplus_proj(ili, WI, D, Wd, lane, Bi);
        if (PAIRWISE) fpmcplus_proj(ilj, WI, D, Wd, lane, Bj);
        // forward over the window: e_k and q_k per side; C_k parked in the gL_k slot for the backward pass
        float ei[2] = {0.f, 0.f}, ej[2] = {0.f, 0.f}, qi[2] = {0.f, 0.f}, qj[2] = {0.f, 0.f};
        for (int k = 0; k < L; ++k) {
            const size_t ol = (size_t)win[k] * D;
            float r[P];
            float di = 0.f, dj = 0.f;
#pragma unroll
            for (int p = 0; p < P; ++p) {
                const int t = lane + p * kWarp;
                r[p] = (t < D) ? LI[ol + t] : 0.0f;
                sq = fmaf(r[p], r[p], sq);
                di = fmaf(ili[p], r[p], di);
                if (PAIRWISE) dj = fmaf(ilj[p], r[p], dj);
            }
#pragma unroll
            for (int q = 0; q < Q; ++q) C[q] = 0.0f;
            fpmcplus_proj(r, WL, D, Wd, lane, C);
#pragma unroll
            for (int q = 0; q < Q; ++q) if (lane + q * kWarp < Wd) f[(4 + k) * Wd + lane + q * kWarp] = C[q];
            const float e_i = fpmcplus_energy(A, Bi, C, H, Wd, lane);
            const float q_i = warp_sum(di);
            const float e_j = PAIRWISE ? fpmcplus_energy(A, Bj, C, H, Wd, lane) : 0.0f;
            const float q_j = PAIRWISE ? warp_sum(dj) : 0.0f;
            if (lane == (k & 31)) {
                const int h = k >> 5;
                if (h == 0) { ei[0] = e_i; qi[0] = q_i; ej[0] = e_j; qj[0] = q_j; }
                else { ei[1] = e_i; qi[1] = q_i; ej[1] = e_j; qj[1] = q_j; }
            }
        }
        // softmax over the window (exp(e) / sum exp(e), :87-91) and x = <UI_u, IU_s> + sum_k a_k q_k
        float ai[2], aj[2];
        {
            const bool k0 = lane < L, k1 = lane + 32 < L;
            const float x0 = k0 ? expf(ei[0]) : 0.f, x1 = k1 ? expf(ei[1]) : 0.f;
            const float s = warp_sum(x0 + x1);
            ai[0] = k0 ? x0 / s : 0.f; ai[1] = k1 ? x1 / s : 0.f;
            if (PAIRWISE) {
                const float y0 = k0 ? expf(ej[0]) : 0.f, y1 = k1 ? expf(ej[1]) : 0.f;
                const float t = warp_sum(y0 + y1);
                aj[0] = k0 ? y0 / t : 0.f; aj[1] = k1 ? y1 / t : 0.f;
            }
        }
        const float yi = warp_sum(fmaf(ai[0], qi[0], ai[1] * qi[1]));
        const float yj = PAIRWISE ? warp_sum(fmaf(aj[0], qj[0], aj[1] * qj[1])) : 0.0f;
        xi = warp_sum(xi) + yi;
        float lo, c;
        if (PAIRWISE) pairwise_loss_grad(loss_kind, xi - (warp_sum(xj) + yj), lo, c);
        else pointwise_loss_grad(loss_kind, xi, static_cast<const float*>(third)[b], inv_b, lo, c);
        if (reg != 0.0f) lo += reg * 0.5f * warp_sum(sq);
        loss_acc += lo;
        // de_k = c_s a_k (q_k - y_s)
        float dei[2], dej[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            dei[h] = c * ai[h] * (qi[h] - yi);
            if (PAIRWISE) dej[h] = -c * aj[h] * (qj[h] - yj);
        }
        float si[P], sj[P], zi[Q], zj[Q], gh[Q];
#pragma unroll
        for (int p = 0; p < P; ++p) si[p] = sj[p] = 0.0f;
#pragma unroll
        for (int q = 0; q < Q; ++q) zi[q] = zj[q] = gh[q] = 0.0f;
        for (int k = 0; k < L; ++k) {
            const int lk = win[k];
            const size_t ol = (size_t)lk * D;
            const int src = k & 31, h = k >> 5;
            const float aik = __shfl_sync(kFull, h ? ai[1] : ai[0], src);
            const float deik = __shfl_sync(kFull, h ? dei[1] : dei[0], src);
            const float ajk = PAIRWISE ? __shfl_sync(kFull, h ? aj[1] : aj[0], src) : 0.0f;
            const float dejk = PAIRWISE ? __shfl_sync(kFull, h ? dej[1] : dej[0], src) : 0.0f;
            float gl[Q];
#pragma unroll
            for (int q = 0; q < Q; ++q) {
                const int cc = lane + q * kWarp;
                gl[q] = 0.0f;
                if (cc < Wd) {
                    const float ck = f[(4 + k) * Wd + cc];
                    const float ti = tanhf((A[q] + Bi[q]) + ck);
                    const float dzi = (deik * H[q]) * (1.0f - ti * ti);
                    zi[q] += dzi;
                    gh[q] = fmaf(deik, ti, gh[q]);
                    gl[q] = dzi;
                    if (PAIRWISE) {
                        const float tj = tanhf((A[q] + Bj[q]) + ck);
                        const float dzj = (dejk * H[q]) * (1.0f - tj * tj);
                        zj[q] += dzj;
                        gh[q] = fmaf(dejk, tj, gh[q]);
                        gl[q] += dzj;
                    }
                    f[(4 + k) * Wd + cc] = gl[q];
                }
            }
            float v[P];
            fpmcplus_back(gl, WL, D, Wd, lane, v);
#pragma unroll
            for (int p = 0; p < P; ++p) {
                const int t = lane + p * kWarp;
                if (t < D) {
                    const float r = LI[ol + t];
                    si[p] = fmaf(aik, r, si[p]);
                    float g = c * (aik * ili[p]);
                    if (PAIRWISE) { sj[p] = fmaf(ajk, r, sj[p]); g -= c * (ajk * ilj[p]); }
                    atomicAdd(gLI + ol + t, (g + v[p]) + reg * r);
                }
            }
            if (lane == 0) tL[lk] = stamp;
        }
        float gA[Q];
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const int cc = lane + q * kWarp;
            gA[q] = zi[q] + zj[q];
            if (cc < Wd) {
                f[cc] = gA[q]; f[Wd + cc] = zi[q]; f[2 * Wd + cc] = zj[q]; f[3 * Wd + cc] = gh[q];
            }
        }
        float vU[P], vI[P];
        fpmcplus_back(gA, WU, D, Wd, lane, vU);
        fpmcplus_back(zi, WI, D, Wd, lane, vI);
#pragma unroll
        for (int p = 0; p < P; ++p) {
            const int t = lane + p * kWarp;
            if (t < D) {
                const float ui = IU[oi + t];
                if (PAIRWISE) {
                    const float uj = IU[oj + t];
                    atomicAdd(gUI + ou + t, (c * (ui - uj) + vU[p]) + reg * a[p]);
                    atomicAdd(gIU + oj + t, -c * a[p] + reg * uj);
                } else {
                    atomicAdd(gUI + ou + t, (c * ui + vU[p]) + reg * a[p]);
                }
                atomicAdd(gIU + oi + t, c * a[p] + reg * ui);
                atomicAdd(gIL + oi + t, (c * si[p] + vI[p]) + reg * ili[p]);
            }
        }
        if (PAIRWISE) {
            fpmcplus_back(zj, WI, D, Wd, lane, vI);
#pragma unroll
            for (int p = 0; p < P; ++p) {
                const int t = lane + p * kWarp;
                if (t < D) atomicAdd(gIL + oj + t, (-c * sj[p] + vI[p]) + reg * ilj[p]);
            }
        }
        if (lane == 0) {
            tU[u] = stamp; tI[i] = stamp;
            if (PAIRWISE) tI[j] = stamp;
        }
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
    // reg_w * l2_loss(W, h) enters once per batch (pairwise only; reg_w = 0 otherwise)
    if (PAIRWISE && reg_w != 0.0f && loss && blockIdx.x == 0 && threadIdx.x < kWarp) {
        float s = 0.0f;
        for (int64_t e = lane; e < 3 * (int64_t)D * Wd; e += kWarp) s = fmaf(W[e], W[e], s);
        float t = 0.0f;
        for (int e = lane; e < Wd; e += kWarp) t = fmaf(Hv[e], Hv[e], t);
        s = warp_sum(s);
        t = warp_sum(t);
        if (lane == 0) atomicAdd(loss, reg_w * (0.5f * s + 0.5f * t));
    }
}

// Dense gradients from the per-sample factors.  grid = (element tiles of 256 over [W, b, h], chunks of kFpmcPlusChunk
// samples): each CTA sums its chunk in sample order into partial[chunk]; the last CTA of an element tile to finish
// adds the chunks in chunk order (plus reg_w * W and reg_w * h) into the gradients and resets the tile's counter.
__global__ void __launch_bounds__(256)
fpmcplus_wgrad_kernel(const float* __restrict__ UI, const float* __restrict__ IL, const float* __restrict__ LI,
                      const float* __restrict__ W, const float* __restrict__ Hv, int D, int Wd, int L,
                      const int32_t* __restrict__ users, const int32_t* __restrict__ recent,
                      const int32_t* __restrict__ items, const int32_t* __restrict__ negs, int64_t batch, float reg_w,
                      const float* __restrict__ fac, float* __restrict__ partial, unsigned* __restrict__ counters,
                      float* __restrict__ gW, float* __restrict__ gB, float* __restrict__ gH) {
    __shared__ bool s_last;
    const int64_t E = fpmcplus_dense_floats(D, Wd), EW = 3 * (int64_t)D * Wd;
    const int64_t stride = fpmcplus_factor_floats(Wd, L);
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t b0 = (int64_t)blockIdx.y * kFpmcPlusChunk;
    const int64_t b1 = (batch - b0 < kFpmcPlusChunk) ? batch : b0 + kFpmcPlusChunk;
    if (e < E) {
        float s = 0.0f;
        if (e < EW) {
            const int r = (int)(e / Wd), c = (int)(e - (int64_t)r * Wd);
            const int part = r / D, rr = r - part * D;
            if (part == 0) {
                for (int64_t b = b0; b < b1; ++b) s = fmaf(UI[(size_t)users[b] * D + rr], fac[b * stride + c], s);
            } else if (part == 1) {
                for (int64_t b = b0; b < b1; ++b) {
                    s = fmaf(IL[(size_t)items[b] * D + rr], fac[b * stride + Wd + c], s);
                    if (negs) s = fmaf(IL[(size_t)negs[b] * D + rr], fac[b * stride + 2 * Wd + c], s);
                }
            } else {
                for (int64_t b = b0; b < b1; ++b)
                    for (int k = 0; k < L; ++k)
                        s = fmaf(LI[(size_t)recent[b * L + k] * D + rr], fac[b * stride + (4 + k) * Wd + c], s);
            }
        } else {
            const int c = (int)((e - EW) % Wd), off = (e - EW < Wd) ? 0 : 3 * Wd;   // b: gA, h: gH
            for (int64_t b = b0; b < b1; ++b) s += fac[b * stride + off + c];
        }
        partial[(size_t)blockIdx.y * E + e] = s;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(counters + blockIdx.x, 1u) == gridDim.y - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (e < E) {
        float s = 0.0f;
        for (unsigned k = 0; k < gridDim.y; ++k) s += __ldcg(partial + (size_t)k * E + e);
        if (e < EW) gW[e] += s + reg_w * W[e];
        else if (e - EW < Wd) gB[e - EW] += s;
        else gH[e - EW - Wd] += s + reg_w * Hv[e - EW - Wd];
    }
    if (threadIdx.x == 0) counters[blockIdx.x] = 0u;
}

// Scoring, pass 1: the projections the pair kernel reads, into work.  Element ranges (one thread each):
//   Bt  [w, I]   IL W_I, transposed so that the pair kernel's item reads coalesce
//   ILt [d, I], IUt [d, I]   IL and IU transposed
//   A   [rows, w]            UI_u W_U + b
//   C   [rows, L, w]         LI_{l_k} W_L over each row's table window (0 past its length)
__global__ void __launch_bounds__(256)
fpmcplus_project_kernel(const float* __restrict__ UI, const float* __restrict__ IU, const float* __restrict__ IL,
                        const float* __restrict__ LI, const float* __restrict__ W, const float* __restrict__ Bv, int D,
                        int Wd, int L, int32_t I, const int32_t* __restrict__ users, const int32_t* __restrict__ recent,
                        const int32_t* __restrict__ recent_len, int64_t rows, float* __restrict__ work) {
    const int64_t nB = (int64_t)Wd * I, nT = (int64_t)D * I, nA = rows * Wd, nC = rows * L * Wd;
    const int64_t total = nB + 2 * nT + nA + nC;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        float v = 0.0f;
        if (e < nB) {
            const int c = (int)(e / I), j = (int)(e - (int64_t)c * I);
            const float* __restrict__ x = IL + (size_t)j * D;
            const float* __restrict__ Wb = W + (size_t)D * Wd + c;
            for (int r = 0; r < D; ++r) v = fmaf(x[r], Wb[(size_t)r * Wd], v);
        } else if (e < nB + 2 * nT) {
            const int64_t f = e - nB;
            const float* __restrict__ T = f < nT ? IL : IU;
            const int64_t g = f < nT ? f : f - nT;
            const int t = (int)(g / I), j = (int)(g - (int64_t)t * I);
            v = T[(size_t)j * D + t];
        } else if (e < nB + 2 * nT + nA) {
            const int64_t f = e - nB - 2 * nT;
            const int64_t r = f / Wd;
            const int c = (int)(f - r * Wd);
            const float* __restrict__ x = UI + (size_t)users[r] * D;
            for (int k = 0; k < D; ++k) v = fmaf(x[k], W[(size_t)k * Wd + c], v);
            v += Bv[c];
        } else {
            const int64_t f = e - nB - 2 * nT - nA;
            const int64_t rk = f / Wd;
            const int c = (int)(f - rk * Wd);
            const int64_t r = rk / L;
            const int k = (int)(rk - r * L);
            const int u = users[r];
            if (k < recent_len[u]) {
                const float* __restrict__ x = LI + (size_t)recent[(size_t)u * L + k] * D;
                const float* __restrict__ Wb = W + 2 * (size_t)D * Wd + c;
                for (int t = 0; t < D; ++t) v = fmaf(x[t], Wb[(size_t)t * Wd], v);
            }
        }
        work[e] = v;
    }
}

// Scoring, pass 2: out[r, j] for R rows per CTA (their A, C, LI window rows, UI row and h in shared memory) and one
// item per thread.  Per (row, item): L w tanh, L w FMAs and (L + 1) d FMAs.  The softmax is folded into one pass,
// y = (sum_k exp(e_k) q_k) / (sum_k exp(e_k)); where the denominator overflows, every a_k of the reference is
// exp(e_k) / inf, which is NaN if an exp(e_k) overflowed and 0 otherwise, and y follows it.
__global__ void __launch_bounds__(256)
fpmcplus_pair_kernel(const float* __restrict__ LI, const float* __restrict__ UI, const float* __restrict__ Hv, int D,
                     int Wd, int L, int32_t I, int R, const int32_t* __restrict__ users,
                     const int32_t* __restrict__ recent, const int32_t* __restrict__ recent_len, int64_t rows,
                     const float* __restrict__ work, float* __restrict__ out) {
    extern __shared__ float sm[];
    const int64_t nB = (int64_t)Wd * I, nT = (int64_t)D * I;
    const float* __restrict__ Bt = work;
    const float* __restrict__ ILt = work + nB;
    const float* __restrict__ IUt = work + nB + nT;
    const float* __restrict__ gA = work + nB + 2 * nT;
    const float* __restrict__ gC = gA + rows * Wd;
    float* sH = sm;
    float* sA = sH + Wd;
    float* sC = sA + (size_t)R * Wd;
    float* sL = sC + (size_t)R * L * Wd;
    float* sU = sL + (size_t)R * L * D;
    int* sN = reinterpret_cast<int*>(sU + (size_t)R * D);
    const int64_t r0 = (int64_t)blockIdx.x * R;
    const int nr = (rows - r0 < R) ? (int)(rows - r0) : R;
    for (int e = threadIdx.x; e < Wd; e += blockDim.x) sH[e] = Hv[e];
    for (int e = threadIdx.x; e < nr * Wd; e += blockDim.x) sA[e] = gA[r0 * Wd + e];
    for (int e = threadIdx.x; e < nr * L * Wd; e += blockDim.x) sC[e] = gC[r0 * L * Wd + e];
    for (int e = threadIdx.x; e < nr * L * D; e += blockDim.x) {
        const int r = e / (L * D), k = (e / D) % L, t = e % D;
        const int u = users[r0 + r];
        sL[e] = k < recent_len[u] ? LI[(size_t)recent[(size_t)u * L + k] * D + t] : 0.0f;
    }
    for (int e = threadIdx.x; e < nr * D; e += blockDim.x) {
        const int r = e / D, t = e % D;
        sU[e] = UI[(size_t)users[r0 + r] * D + t];
    }
    for (int r = threadIdx.x; r < nr; r += blockDim.x) sN[r] = recent_len[users[r0 + r]];
    __syncthreads();
    const int64_t j = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
    if (j >= I) return;
    for (int r = 0; r < nr; ++r) {
        float p = 0.0f;
        for (int t = 0; t < D; ++t) p = fmaf(sU[r * D + t], __ldg(IUt + (size_t)t * I + j), p);
        float S = 0.0f, N = 0.0f;
        bool inf = false;
        const int n = sN[r];
        for (int k = 0; k < n; ++k) {
            const float* c = sC + ((size_t)r * L + k) * Wd;
            const float* a = sA + (size_t)r * Wd;
            float e = 0.0f;
            for (int q = 0; q < Wd; ++q) e = fmaf(sH[q], tanhf((a[q] + __ldg(Bt + (size_t)q * I + j)) + c[q]), e);
            const float* l = sL + ((size_t)r * L + k) * D;
            float qk = 0.0f;
            for (int t = 0; t < D; ++t) qk = fmaf(__ldg(ILt + (size_t)t * I + j), l[t], qk);
            const float x = expf(e);
            S += x;
            N = fmaf(x, qk, N);
            inf |= isinf(x);
        }
        const float y = isinf(S) ? (inf ? __int_as_float(0x7fc00000) : 0.0f) : N / S;
        out[(size_t)(r0 + r) * I + j] = p + y;
    }
}

}  // namespace nrc

using namespace nrc;

extern "C" int nrc_fpmc_grad(const float* ui, const float* iu, const float* il, const float* li, int32_t dim,
                             const int32_t* users, const int32_t* recent, const int32_t* items, const void* third,
                             int64_t batch, int32_t pairwise, int32_t loss_kind, float reg, float* grad_ui,
                             float* grad_iu, float* grad_il, float* grad_li, int32_t* touched_user,
                             int32_t* touched_item, int32_t* touched_recent, int32_t stamp, float* loss, void* stream) {
    const int rc = seq_check(dim, pairwise, loss_kind, batch);
    if (rc) return rc;
    if (batch == 0) return NRC_OK;
    const int64_t cap = (int64_t)sm_count() * 8;
    const unsigned grid = seq_grad_grid(batch, cap);
    seq_route(kSeqFpmcGrad, pairwise ? 1 : 0, -1, -1, grid, -1, seq_grad_capped(batch, cap), -1);
    const float inv_b = 1.0f / (float)batch;
    if (pairwise)
        fpmc_grad_kernel<true><<<grid, 256, 0, as_stream(stream)>>>(ui, iu, il, li, dim, users, recent, items, third, batch,
                                                                     loss_kind, reg, inv_b, grad_ui, grad_iu, grad_il,
                                                                     grad_li, touched_user, touched_item, touched_recent,
                                                                     stamp, loss);
    else
        fpmc_grad_kernel<false><<<grid, 256, 0, as_stream(stream)>>>(ui, iu, il, li, dim, users, recent, items, third, batch,
                                                                      loss_kind, reg, inv_b, grad_ui, grad_iu, grad_il,
                                                                      grad_li, touched_user, touched_item, touched_recent,
                                                                      stamp, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_fpmc_train_epoch(float* ui, float* iu, float* il, float* li, int32_t num_users, int32_t num_items,
                                    int32_t dim, const int32_t* users, const int32_t* recent, const int32_t* items,
                                    const void* third, int64_t n, int32_t batch_size, int32_t pairwise, int32_t loss_kind,
                                    float reg, int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                                    float* grad_ui, float* grad_iu, float* grad_il, float* grad_li,
                                    int32_t* touched_user, int32_t* touched_item, int32_t* touched_recent,
                                    float* const* slot0, float* const* slot1, int32_t first_stamp, float* step_loss,
                                    void* stream) {
    int rc = seq_check_epoch(dim, pairwise, loss_kind, n, batch_size, opt_kind, lr_t_host, hyper_host);
    if (rc) return rc;
    NRC_REQUIRE(slot0 && slot1, NRC_E_VALUE, "slot0 and slot1 must list the four variables' slots");
    const size_t third_bytes = 4;       // i32 negatives or f32 labels
    return seq_epoch_loop(
        n, batch_size, opt_kind, lr_t_host, hyper_host, first_stamp, step_loss, as_stream(stream),
        [&](int64_t off, int64_t bs, int32_t stamp, float* loss) {
            return nrc_fpmc_grad(ui, iu, il, li, dim, users + off, recent + off, items + off,
                                 static_cast<const char*>(third) + off * third_bytes, bs, pairwise, loss_kind, reg,
                                 grad_ui, grad_iu, grad_il, grad_li, touched_user, touched_item, touched_recent, stamp,
                                 loss, stream);
        },
        [&](OptLaunch& L) {
            opt_launch_add(L, ui, grad_ui, slot0[0], slot1[0], touched_user, num_users, dim, 0);
            opt_launch_add(L, iu, grad_iu, slot0[1], slot1[1], touched_item, num_items, dim, 0);
            opt_launch_add(L, il, grad_il, slot0[2], slot1[2], touched_item, num_items, dim, 0);
            opt_launch_add(L, li, grad_li, slot0[3], slot1[3], touched_recent, num_items, dim, 0);
        });
}

extern "C" int64_t nrc_transrec_work_floats(int32_t dim) {
    NRC_REQUIRE(dim >= 1 && dim <= kSeqMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kSeqMaxDim);
    return (int64_t)kTransRecCtas * dim + 1;
}

extern "C" int nrc_transrec_grad(const float* user_table, const float* item_table, const float* item_bias,
                                 const float* global, int32_t dim, const int32_t* users, const int32_t* recent,
                                 const int32_t* items, const void* third, int64_t batch, int32_t pairwise,
                                 int32_t loss_kind, float reg, float* grad_user, float* grad_item, float* grad_bias,
                                 float* grad_global, int32_t* touched_user, int32_t* touched_item,
                                 int32_t* touched_bias, int32_t stamp, float* work, float* loss, void* stream) {
    const int rc = seq_check(dim, pairwise, loss_kind, batch);
    if (rc) return rc;
    NRC_REQUIRE(work, NRC_E_VALUE, "work (nrc_transrec_work_floats(dim) floats) is required");
    if (batch == 0) return NRC_OK;
    const unsigned grid = seq_grad_grid(batch, kTransRecCtas);
    seq_route(kSeqTransRecGrad, pairwise ? 1 : 0, -1, -1, grid, -1, seq_grad_capped(batch, kTransRecCtas), -1);
    const float inv_b = 1.0f / (float)batch;
    if (pairwise)
        transrec_grad_kernel<true><<<grid, 256, 0, as_stream(stream)>>>(
            user_table, item_table, item_bias, global, dim, users, recent, items, third, batch, loss_kind, reg, inv_b,
            grad_user, grad_item, grad_bias, grad_global, touched_user, touched_item, touched_bias, stamp, work, loss);
    else
        transrec_grad_kernel<false><<<grid, 256, 0, as_stream(stream)>>>(
            user_table, item_table, item_bias, global, dim, users, recent, items, third, batch, loss_kind, reg, inv_b,
            grad_user, grad_item, grad_bias, grad_global, touched_user, touched_item, touched_bias, stamp, work, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_transrec_train_epoch(float* user_table, float* item_table, float* item_bias, float* global,
                                        int32_t num_users, int32_t num_items, int32_t dim, const int32_t* users,
                                        const int32_t* recent, const int32_t* items, const void* third, int64_t n,
                                        int32_t batch_size, int32_t pairwise, int32_t loss_kind, float reg,
                                        int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                                        float* grad_user, float* grad_item, float* grad_bias, float* grad_global,
                                        int32_t* touched_user, int32_t* touched_item, int32_t* touched_bias,
                                        float* const* slot0, float* const* slot1, int32_t first_stamp, float* work,
                                        float* step_loss, void* stream) {
    int rc = seq_check_epoch(dim, pairwise, loss_kind, n, batch_size, opt_kind, lr_t_host, hyper_host);
    if (rc) return rc;
    NRC_REQUIRE(slot0 && slot1, NRC_E_VALUE, "slot0 and slot1 must list the four variables' slots");
    NRC_REQUIRE(work, NRC_E_VALUE, "work (nrc_transrec_work_floats(dim) floats) is required");
    const size_t third_bytes = 4;       // i32 negatives or f32 labels
    return seq_epoch_loop(
        n, batch_size, opt_kind, lr_t_host, hyper_host, first_stamp, step_loss, as_stream(stream),
        [&](int64_t off, int64_t bs, int32_t stamp, float* loss) {
            return nrc_transrec_grad(user_table, item_table, item_bias, global, dim, users + off, recent + off,
                                     items + off, static_cast<const char*>(third) + off * third_bytes, bs, pairwise,
                                     loss_kind, reg, grad_user, grad_item, grad_bias, grad_global, touched_user,
                                     touched_item, touched_bias, stamp, work, loss, stream);
        },
        [&](OptLaunch& L) {
            opt_launch_add(L, user_table, grad_user, slot0[0], slot1[0], touched_user, num_users, dim, 0);
            opt_launch_add(L, item_table, grad_item, slot0[1], slot1[1], touched_item, num_items, dim, 0);
            opt_launch_add(L, item_bias, grad_bias, slot0[2], slot1[2], touched_bias, num_items, 1, 0);
            // tf.tile makes g's gradient a dense tensor: the Apply* formulas, every element (TransRec.py:75)
            opt_launch_add(L, global, grad_global, slot0[3], slot1[3], nullptr, 1, dim, 1);
        });
}

static unsigned score_item_tiles(int32_t num_items) { return (unsigned)((num_items + 255) / 256); }

extern "C" int nrc_fpmc_scores(const float* ui, const float* iu, const float* il, const float* li, int32_t num_items,
                               int32_t dim, const int32_t* users, const int32_t* recent, int64_t rows, float* out,
                               void* stream) {
    NRC_REQUIRE(dim >= 1 && dim <= kSeqMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kSeqMaxDim);
    NRC_REQUIRE(num_items > 0 && rows >= 0, NRC_E_VALUE, "num_items > 0 and rows >= 0 required");
    NRC_REQUIRE(score_item_tiles(num_items) <= 65535u, NRC_E_LIMIT, "num_items %d above %d", num_items, 65535 * 256);
    if (rows == 0) return NRC_OK;
    const dim3 grid((unsigned)((rows + kScoreRows - 1) / kScoreRows), score_item_tiles(num_items));
    seq_route(kSeqFpmcScores, -1, -1, -1, grid.x, grid.y, -1, -1);
    fpmc_scores_kernel<<<grid, 256, 0, as_stream(stream)>>>(ui, iu, il, li, dim, num_items, users, recent, rows, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_transrec_scores(const float* user_table, const float* item_table, const float* item_bias,
                                   const float* global, int32_t num_items, int32_t dim, const int32_t* users,
                                   const int32_t* recent, int64_t rows, float* out, void* stream) {
    NRC_REQUIRE(dim >= 1 && dim <= kSeqMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kSeqMaxDim);
    NRC_REQUIRE(num_items > 0 && rows >= 0, NRC_E_VALUE, "num_items > 0 and rows >= 0 required");
    NRC_REQUIRE(score_item_tiles(num_items) <= 65535u, NRC_E_LIMIT, "num_items %d above %d", num_items, 65535 * 256);
    if (rows == 0) return NRC_OK;
    const dim3 grid((unsigned)((rows + kScoreRows - 1) / kScoreRows), score_item_tiles(num_items));
    seq_route(kSeqTransRecScores, -1, -1, -1, grid.x, grid.y, -1, -1);
    transrec_scores_kernel<<<grid, 256, 0, as_stream(stream)>>>(user_table, item_table, item_bias, global, dim,
                                                                 num_items, users, recent, rows, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// ---------------------------------------------------------------------------------------------
// HRM and NPE entry points
// ---------------------------------------------------------------------------------------------
extern "C" int nrc_hrm_grad(const float* user_table, const float* item_table, int32_t dim, int32_t window,
                            const int32_t* users, const int32_t* recent, const int32_t* items, const float* labels,
                            int64_t batch, int32_t pre_agg, int32_t session_agg, int32_t loss_kind, float reg,
                            float* grad_user, float* grad_item, int32_t* touched_user, int32_t* touched_item,
                            int32_t stamp, float* loss, void* stream) {
    int rc = seq_check(dim, 0, loss_kind, batch);
    if (rc) return rc;
    rc = seq_check_window(window);
    if (rc) return rc;
    if (batch == 0) return NRC_OK;
    const int64_t cap = (int64_t)sm_count() * 8;
    const unsigned grid = seq_grad_grid(batch, cap);
    seq_route(kSeqHrmGrad, 0, session_agg ? 1 : 0, pre_agg ? 1 : 0, grid, -1, seq_grad_capped(batch, cap), window);
    auto* kernel = session_agg ? (pre_agg ? hrm_grad_kernel<true, true> : hrm_grad_kernel<true, false>)
                               : (pre_agg ? hrm_grad_kernel<false, true> : hrm_grad_kernel<false, false>);
    kernel<<<grid, 256, 0, as_stream(stream)>>>(user_table, item_table, dim, window, users, recent, items, labels,
                                                batch, loss_kind, reg, 1.0f / (float)batch, grad_user, grad_item,
                                                touched_user, touched_item, stamp, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_hrm_train_epoch(float* user_table, float* item_table, int32_t num_users, int32_t num_items,
                                   int32_t dim, int32_t window, const int32_t* users, const int32_t* recent,
                                   const int32_t* items, const float* labels, int64_t n, int32_t batch_size,
                                   int32_t pre_agg, int32_t session_agg, int32_t loss_kind, float reg,
                                   int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                                   float* grad_user, float* grad_item, int32_t* touched_user, int32_t* touched_item,
                                   float* const* slot0, float* const* slot1, int32_t first_stamp, float* step_loss,
                                   void* stream) {
    int rc = seq_check_window(window);
    if (rc) return rc;
    rc = seq_check_epoch(dim, 0, loss_kind, n, batch_size, opt_kind, lr_t_host, hyper_host);
    if (rc) return rc;
    NRC_REQUIRE(slot0 && slot1, NRC_E_VALUE, "slot0 and slot1 must list the two variables' slots");
    return seq_epoch_loop(
        n, batch_size, opt_kind, lr_t_host, hyper_host, first_stamp, step_loss, as_stream(stream),
        [&](int64_t off, int64_t bs, int32_t stamp, float* loss) {
            return nrc_hrm_grad(user_table, item_table, dim, window, users + off, recent + off * window, items + off,
                                labels + off, bs, pre_agg, session_agg, loss_kind, reg, grad_user, grad_item,
                                touched_user, touched_item, stamp, loss, stream);
        },
        [&](OptLaunch& L) {
            opt_launch_add(L, user_table, grad_user, slot0[0], slot1[0], touched_user, num_users, dim, 0);
            opt_launch_add(L, item_table, grad_item, slot0[1], slot1[1], touched_item, num_items, dim, 0);
        });
}

extern "C" int nrc_hrm_query(const float* user_table, const float* item_table, int32_t dim, int32_t window,
                             const int32_t* users, int64_t rows, const int32_t* recent, const int32_t* recent_len,
                             int32_t pre_agg, int32_t session_agg, float* out, void* stream) {
    const int rc = seq_check_query(dim, window, rows);
    if (rc) return rc;
    if (rows == 0) return NRC_OK;
    auto* kernel = session_agg ? (pre_agg ? hrm_query_kernel<true, true> : hrm_query_kernel<true, false>)
                               : (pre_agg ? hrm_query_kernel<false, true> : hrm_query_kernel<false, false>);
    const unsigned grid = elementwise_grid(rows * dim);
    seq_route(kSeqHrmQuery, -1, session_agg ? 1 : 0, pre_agg ? 1 : 0, grid, -1, elementwise_capped(rows * dim),
              window);
    kernel<<<grid, 256, 0, as_stream(stream)>>>(user_table, item_table, dim, window, users, recent, recent_len, rows,
                                                out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_npe_grad(const float* ui, const float* iu, const float* il, int32_t dim, int32_t window,
                            const int32_t* users, const int32_t* recent, const int32_t* items, const float* labels,
                            int64_t batch, int32_t loss_kind, float reg, float* grad_ui, float* grad_iu,
                            float* grad_il, int32_t* touched_user, int32_t* touched_item, int32_t* touched_recent,
                            int32_t stamp, float* loss, void* stream) {
    int rc = seq_check(dim, 0, loss_kind, batch);
    if (rc) return rc;
    rc = seq_check_window(window);
    if (rc) return rc;
    if (batch == 0) return NRC_OK;
    const int64_t cap = (int64_t)sm_count() * 8;
    const unsigned grid = seq_grad_grid(batch, cap);
    seq_route(kSeqNpeGrad, 0, -1, -1, grid, -1, seq_grad_capped(batch, cap), window);
    npe_grad_kernel<<<grid, 256, 0, as_stream(stream)>>>(ui, iu, il, dim, window, users, recent, items, labels, batch,
                                                         loss_kind, reg, 1.0f / (float)batch, grad_ui, grad_iu,
                                                         grad_il, touched_user, touched_item, touched_recent, stamp,
                                                         loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_npe_train_epoch(float* ui, float* iu, float* il, int32_t num_users, int32_t num_items, int32_t dim,
                                   int32_t window, const int32_t* users, const int32_t* recent, const int32_t* items,
                                   const float* labels, int64_t n, int32_t batch_size, int32_t loss_kind, float reg,
                                   int32_t opt_kind, const float* lr_t_host, const float* hyper_host, float* grad_ui,
                                   float* grad_iu, float* grad_il, int32_t* touched_user, int32_t* touched_item,
                                   int32_t* touched_recent, float* const* slot0, float* const* slot1,
                                   int32_t first_stamp, float* step_loss, void* stream) {
    int rc = seq_check_window(window);
    if (rc) return rc;
    rc = seq_check_epoch(dim, 0, loss_kind, n, batch_size, opt_kind, lr_t_host, hyper_host);
    if (rc) return rc;
    NRC_REQUIRE(slot0 && slot1, NRC_E_VALUE, "slot0 and slot1 must list the three variables' slots");
    return seq_epoch_loop(
        n, batch_size, opt_kind, lr_t_host, hyper_host, first_stamp, step_loss, as_stream(stream),
        [&](int64_t off, int64_t bs, int32_t stamp, float* loss) {
            return nrc_npe_grad(ui, iu, il, dim, window, users + off, recent + off * window, items + off, labels + off,
                                bs, loss_kind, reg, grad_ui, grad_iu, grad_il, touched_user, touched_item,
                                touched_recent, stamp, loss, stream);
        },
        [&](OptLaunch& L) {
            opt_launch_add(L, ui, grad_ui, slot0[0], slot1[0], touched_user, num_users, dim, 0);
            opt_launch_add(L, iu, grad_iu, slot0[1], slot1[1], touched_item, num_items, dim, 0);
            opt_launch_add(L, il, grad_il, slot0[2], slot1[2], touched_recent, num_items, dim, 0);
        });
}

extern "C" int nrc_npe_query(const float* ui, const float* iu, const float* il, int32_t num_items, int32_t dim,
                             int32_t window, const int32_t* users, int64_t rows, const int32_t* recent,
                             const int32_t* recent_len, float* out, float* out_items, void* stream) {
    const int rc = seq_check_query(dim, window, rows);
    if (rc) return rc;
    NRC_REQUIRE(num_items > 0 || !out_items, NRC_E_VALUE, "num_items > 0 required with out_items");
    cudaStream_t st = as_stream(stream);
    if (rows > 0) {
        const unsigned grid = elementwise_grid(rows * dim);
        seq_route(kSeqNpeQuery, -1, -1, -1, grid, -1, elementwise_capped(rows * dim), window);
        npe_query_kernel<<<grid, 256, 0, st>>>(ui, il, dim, window, users, recent, recent_len, rows, out);
        NRC_CUDA_CHECK(cudaGetLastError());
    }
    if (out_items) {
        const int64_t total = (int64_t)num_items * dim;
        const unsigned grid = elementwise_grid(total);
        seq_route(kSeqNpeRelu, -1, -1, -1, grid, -1, elementwise_capped(total), -1);
        relu_kernel<<<grid, 256, 0, st>>>(iu, total, out_items);
        NRC_CUDA_CHECK(cudaGetLastError());
    }
    return NRC_OK;
}

// ---------------------------------------------------------------------------------------------
// FPMCplus entry points
// ---------------------------------------------------------------------------------------------
// Host record of FPMCplus's launches, for nrc_fpmcplus_last_routes (see the header); -1 as for g_seq_routes.
enum FpmcPlusKernel { kFpGrad, kFpWgrad, kFpProject, kFpPair, kFpKernels };
enum FpmcPlusField { kFpPairwise, kFpGridX, kFpGridY, kFpCapped, kFpWindow, kFpRows, kFpFields };
static struct FpmcPlusRoutes {
    int32_t r[kFpKernels][kFpFields];
    FpmcPlusRoutes() { for (auto& k : r) for (auto& f : k) f = -1; }
} g_fpmcplus_routes;

static void fpmcplus_route(int kernel, int pairwise, int64_t grid_x, int64_t grid_y, int capped, int window,
                           int rows) {
    int32_t* r = g_fpmcplus_routes.r[kernel];
    r[kFpPairwise] = pairwise; r[kFpGridX] = (int32_t)grid_x; r[kFpGridY] = (int32_t)grid_y;
    r[kFpCapped] = capped; r[kFpWindow] = window; r[kFpRows] = rows;
}

static int fpmcplus_check_shape(int32_t dim, int32_t weight_size, int32_t window) {
    NRC_REQUIRE(dim >= 1 && dim <= kSeqMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kSeqMaxDim);
    NRC_REQUIRE(weight_size >= 1 && weight_size <= kFpmcPlusMaxWeight, NRC_E_LIMIT, "weight_size %d outside [1, %d]",
                weight_size, kFpmcPlusMaxWeight);
    return seq_check_window(window);
}

static int fpmcplus_check_batch(int64_t batch) {
    NRC_REQUIRE(fpmcplus_chunks(batch) <= 65535, NRC_E_LIMIT, "batch %lld above %d", (long long)batch,
                65535 * kFpmcPlusChunk);
    return NRC_OK;
}

// rows per CTA of the pair kernel: as many as the shared-memory budget holds, at most kScoreRows
static int fpmcplus_pair_rows(int32_t dim, int32_t weight_size, int32_t window) {
    const int64_t per_row = (int64_t)weight_size * (1 + window) + (int64_t)dim * (1 + window) + 1;
    int64_t r = (kFpmcPlusPairSmemFloats - weight_size) / per_row;
    return (int)(r > kScoreRows ? kScoreRows : r);
}

extern "C" int64_t nrc_fpmcplus_work_floats(int32_t dim, int32_t weight_size, int32_t window, int32_t batch_size) {
    const int rc = fpmcplus_check_shape(dim, weight_size, window);
    if (rc) return rc;
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    const int rb = fpmcplus_check_batch(batch_size);
    if (rb) return rb;
    return fpmcplus_counters(dim, weight_size) + (int64_t)batch_size * fpmcplus_factor_floats(weight_size, window) +
           fpmcplus_chunks(batch_size) * fpmcplus_dense_floats(dim, weight_size);
}

extern "C" int nrc_fpmcplus_grad(const float* ui, const float* iu, const float* il, const float* li, const float* w,
                                 const float* b, const float* h, int32_t dim, int32_t weight_size, int32_t window,
                                 const int32_t* users, const int32_t* recent, const int32_t* items, const void* third,
                                 int64_t batch, int32_t pairwise, int32_t loss_kind, float reg_mf, float reg_w,
                                 float* grad_ui, float* grad_iu, float* grad_il, float* grad_li, float* grad_w,
                                 float* grad_b, float* grad_h, int32_t* touched_user, int32_t* touched_item,
                                 int32_t* touched_recent, int32_t stamp, float* work, float* loss, void* stream) {
    int rc = fpmcplus_check_shape(dim, weight_size, window);
    if (rc) return rc;
    rc = seq_check(dim, pairwise, loss_kind, batch);
    if (rc) return rc;
    rc = fpmcplus_check_batch(batch);
    if (rc) return rc;
    NRC_REQUIRE(ui && iu && il && li && w && b && h && users && recent && items && third, NRC_E_VALUE,
                "tables, weights and the batch are required");
    NRC_REQUIRE(grad_ui && grad_iu && grad_il && grad_li && grad_w && grad_b && grad_h && touched_user &&
                touched_item && touched_recent, NRC_E_VALUE, "gradients and touched arrays are required");
    NRC_REQUIRE(work, NRC_E_VALUE, "work (nrc_fpmcplus_work_floats floats) is required");
    if (batch == 0) return NRC_OK;
    cudaStream_t st = as_stream(stream);
    const float rw = pairwise ? reg_w : 0.0f;      // the pointwise loss has no reg_w term (FPMCplus.py:118-119)
    unsigned* counters = reinterpret_cast<unsigned*>(work);
    float* fac = work + fpmcplus_counters(dim, weight_size);
    float* partial = fac + batch * fpmcplus_factor_floats(weight_size, window);
    const int64_t cap = (int64_t)sm_count() * 8;
    const unsigned grid = seq_grad_grid(batch, cap);
    fpmcplus_route(kFpGrad, pairwise ? 1 : 0, grid, -1, seq_grad_capped(batch, cap), window, -1);
    const float inv_b = 1.0f / (float)batch;
    if (pairwise)
        fpmcplus_grad_kernel<true><<<grid, 256, 0, st>>>(ui, iu, il, li, w, b, h, dim, weight_size, window, users,
                                                          recent, items, third, batch, loss_kind, reg_mf, rw, inv_b,
                                                          grad_ui, grad_iu, grad_il, grad_li, touched_user,
                                                          touched_item, touched_recent, stamp, fac, loss);
    else
        fpmcplus_grad_kernel<false><<<grid, 256, 0, st>>>(ui, iu, il, li, w, b, h, dim, weight_size, window, users,
                                                           recent, items, third, batch, loss_kind, reg_mf, rw, inv_b,
                                                           grad_ui, grad_iu, grad_il, grad_li, touched_user,
                                                           touched_item, touched_recent, stamp, fac, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    const dim3 wgrid((unsigned)fpmcplus_counters(dim, weight_size), (unsigned)fpmcplus_chunks(batch));
    fpmcplus_route(kFpWgrad, pairwise ? 1 : 0, wgrid.x, wgrid.y, -1, window, -1);
    fpmcplus_wgrad_kernel<<<wgrid, 256, 0, st>>>(ui, il, li, w, h, dim, weight_size, window, users, recent, items,
                                                 pairwise ? static_cast<const int32_t*>(third) : nullptr, batch, rw,
                                                 fac, partial, counters, grad_w, grad_b, grad_h);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_fpmcplus_train_epoch(float* ui, float* iu, float* il, float* li, float* w, float* b, float* h,
                                        int32_t num_users, int32_t num_items, int32_t dim, int32_t weight_size,
                                        int32_t window, const int32_t* users, const int32_t* recent,
                                        const int32_t* items, const void* third, int64_t n, int32_t batch_size,
                                        int32_t pairwise, int32_t loss_kind, float reg_mf, float reg_w,
                                        int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                                        float* grad_ui, float* grad_iu, float* grad_il, float* grad_li, float* grad_w,
                                        float* grad_b, float* grad_h, int32_t* touched_user, int32_t* touched_item,
                                        int32_t* touched_recent, float* const* slot0, float* const* slot1,
                                        int32_t first_stamp, float* work, float* step_loss, void* stream) {
    int rc = fpmcplus_check_shape(dim, weight_size, window);
    if (rc) return rc;
    rc = seq_check_epoch(dim, pairwise, loss_kind, n, batch_size, opt_kind, lr_t_host, hyper_host);
    if (rc) return rc;
    rc = fpmcplus_check_batch(batch_size);
    if (rc) return rc;
    NRC_REQUIRE(slot0 && slot1, NRC_E_VALUE, "slot0 and slot1 must list the seven variables' slots");
    NRC_REQUIRE(work && step_loss, NRC_E_VALUE, "work (nrc_fpmcplus_work_floats floats) and step_loss are required");
    const size_t third_bytes = 4;       // i32 negatives or f32 labels
    return seq_epoch_loop(
        n, batch_size, opt_kind, lr_t_host, hyper_host, first_stamp, step_loss, as_stream(stream),
        [&](int64_t off, int64_t bs, int32_t stamp, float* loss) {
            return nrc_fpmcplus_grad(ui, iu, il, li, w, b, h, dim, weight_size, window, users + off,
                                     recent + off * window, items + off,
                                     static_cast<const char*>(third) + off * third_bytes, bs, pairwise, loss_kind,
                                     reg_mf, reg_w, grad_ui, grad_iu, grad_il, grad_li, grad_w, grad_b, grad_h,
                                     touched_user, touched_item, touched_recent, stamp, work, loss, stream);
        },
        [&](OptLaunch& L) {
            opt_launch_add(L, ui, grad_ui, slot0[0], slot1[0], touched_user, num_users, dim, 0);
            opt_launch_add(L, iu, grad_iu, slot0[1], slot1[1], touched_item, num_items, dim, 0);
            opt_launch_add(L, il, grad_il, slot0[2], slot1[2], touched_item, num_items, dim, 0);
            opt_launch_add(L, li, grad_li, slot0[3], slot1[3], touched_recent, num_items, dim, 0);
            // W, b and h enter through matmuls: dense gradients, the Apply* formulas on every element
            opt_launch_add(L, w, grad_w, slot0[4], slot1[4], nullptr, 3 * (int64_t)dim, weight_size, 1);
            opt_launch_add(L, b, grad_b, slot0[5], slot1[5], nullptr, 1, weight_size, 1);
            opt_launch_add(L, h, grad_h, slot0[6], slot1[6], nullptr, weight_size, 1, 1);
        });
}

extern "C" int64_t nrc_fpmcplus_score_work_floats(int32_t num_items, int32_t dim, int32_t weight_size, int32_t window,
                                                  int64_t rows) {
    const int rc = fpmcplus_check_shape(dim, weight_size, window);
    if (rc) return rc;
    NRC_REQUIRE(num_items > 0 && rows >= 0, NRC_E_VALUE, "num_items > 0 and rows >= 0 required");
    return (int64_t)num_items * (weight_size + 2 * (int64_t)dim) + rows * (1 + (int64_t)window) * weight_size;
}

extern "C" int nrc_fpmcplus_scores(const float* ui, const float* iu, const float* il, const float* li, const float* w,
                                   const float* b, const float* h, int32_t num_items, int32_t dim, int32_t weight_size,
                                   int32_t window, const int32_t* users, int64_t rows, const int32_t* recent,
                                   const int32_t* recent_len, float* work, float* out, void* stream) {
    int rc = fpmcplus_check_shape(dim, weight_size, window);
    if (rc) return rc;
    NRC_REQUIRE(num_items > 0 && rows >= 0, NRC_E_VALUE, "num_items > 0 and rows >= 0 required");
    NRC_REQUIRE((num_items + kFpmcPlusPairItems - 1) / kFpmcPlusPairItems <= 65535, NRC_E_LIMIT, "num_items %d above %d",
                num_items, 65535 * kFpmcPlusPairItems);
    NRC_REQUIRE(ui && iu && il && li && w && b && h && work && out, NRC_E_VALUE,
                "tables, weights, work and out are required");
    NRC_REQUIRE(rows == 0 || (users && recent && recent_len), NRC_E_VALUE, "users, recent and recent_len are required");
    if (rows == 0) return NRC_OK;
    cudaStream_t st = as_stream(stream);
    const int64_t total = (int64_t)num_items * (weight_size + 2 * (int64_t)dim) + rows * (1 + (int64_t)window) * weight_size;
    const unsigned pgrid = elementwise_grid(total);
    fpmcplus_route(kFpProject, -1, pgrid, -1, elementwise_capped(total), window, -1);
    fpmcplus_project_kernel<<<pgrid, 256, 0, st>>>(ui, iu, il, li, w, b, dim, weight_size, window, num_items, users,
                                                    recent, recent_len, rows, work);
    NRC_CUDA_CHECK(cudaGetLastError());
    const int R = fpmcplus_pair_rows(dim, weight_size, window);
    const size_t smem = ((size_t)weight_size + (size_t)R * ((1 + window) * (size_t)(weight_size + dim)) + R) *
                        sizeof(float);
    NRC_CUDA_CHECK(cudaFuncSetAttribute(fpmcplus_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        kFpmcPlusPairSmemFloats * (int)sizeof(float)));
    const dim3 grid((unsigned)((rows + R - 1) / R), (unsigned)((num_items + kFpmcPlusPairItems - 1) / kFpmcPlusPairItems));
    fpmcplus_route(kFpPair, -1, grid.x, grid.y, -1, window, R);
    fpmcplus_pair_kernel<<<grid, kFpmcPlusPairItems, smem, st>>>(li, ui, h, dim, weight_size, window, num_items, R,
                                                                 users, recent, recent_len, rows, work, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// Host bookkeeping of the routes the most recent FPMCplus launches took (see the header); no device work.
extern "C" int nrc_fpmcplus_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "out is NULL");
    for (int k = 0; k < kFpKernels; ++k)
        for (int f = 0; f < kFpFields; ++f) out[k * kFpFields + f] = g_fpmcplus_routes.r[k][f];
    return NRC_OK;
}

// Host bookkeeping of the routes the most recent sequential launches took (see the header); no device work.
extern "C" int nrc_seq_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "out is NULL");
    for (int k = 0; k < kSeqKernels; ++k)
        for (int f = 0; f < kSeqFields; ++f) out[k * kSeqFields + f] = g_seq_routes.r[k][f];
    return NRC_OK;
}
