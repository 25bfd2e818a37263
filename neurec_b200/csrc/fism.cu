// FISM: factored item similarity.  A user is the sum of the c1 rows of its train history; a sample's score is that
// sum against the target's Q row, scaled by a power of the history's count.
//
// Replaces (reference paths):
//   model/general_recommender/FISM.py:55-88     variables c1, embedding_Q, bias; the inference and loss graphs
//   model/general_recommender/FISM.py:100-144   train_model's batch loop (sess.run((loss, optimizer)) per batch)
//   model/general_recommender/FISM.py:154-180   predict (the history is the user's whole train row)
//
// Variables c1 [I, d], Q [I, d] (embedding_Q), b [I] (bias).  The reference pads histories with id I, which reads the
// constant zero row c2 concatenated after c1; a pad adds nothing and takes no gradient, so pads are not materialised
// here.  One sample is (history row r of a history CSR, an excluded item e or -1, the count n, the target i, a label
// z or a negative j):
//   p = sum_{h in H_r, h != e} c1_h,   x = n^(-alpha) * <p, Q_i> + b_i          (the coefficient multiplies the dot)
//   pointwise  l(z, x) + lambda * l2_loss(p) + gamma * l2_loss(Q_i)
//   pairwise   l(x_i - x_j) + lambda * l2_loss(p) + gamma * (l2_loss(Q_j) + l2_loss(Q_i)), where x_j uses the same
//              history with its own count n_j
// Every occurrence of h in the history takes dl/dp = g n^(-alpha) Q_i [- g n_j^(-alpha) Q_j] + lambda p, so a
// pairwise sample gathers and scatters its history once for both sides.  All three variables take IndexedSlices
// gradients: c1's too, because TF 1.12's ConcatV2 gradient keeps IndexedSlices at axis 0 (read from TF's source, not
// pinned by a run of the reference).
//
// The hot path is the history: one warp per sample reads every row of it twice (the sum, then the gradient's RED.ADD
// into the dense accumulator).  The warp takes 32 history ids with one coalesced load and broadcasts them by shuffle;
// each row is read by a group of lanes_per_row lanes with float4 loads when d % 4 == 0, so 32 / lanes_per_row rows go
// in one warp load (eight at d = 16).  The groups' partial sums meet by shuffle at the end.
#include "common.cuh"
#include "learner.cuh"
#include "optim.cuh"
#include "seq_epoch.cuh"

namespace nrc {

constexpr int kFismMaxDim = 256;
constexpr int kFismPerLane = 8;          // floats of a row one lane holds: 256 / 32
constexpr int kFismWarps = 2;            // warps of a gradient / query CTA (64 threads: a 256-sample step fills 128 SMs)
constexpr int kFismCtasPerSm = 32;       // gradient / query grid cap: 64 samples per SM in flight
constexpr int kFismScoreRows = 8;        // score kernel: users per CTA

// How a warp splits a row of d floats: units of VEC floats, lanes_per_row lanes per row (a power of two), rows per
// warp load = 32 / lanes_per_row, chunks = units a lane owns.
struct FismLanes {
    int vec, units, lpr, rows, chunks;
};

static FismLanes fism_lanes(int d) {
    FismLanes L;
    L.vec = d % 4 == 0 ? 4 : 1;
    L.units = d / L.vec;
    L.lpr = 1;
    while (L.lpr < L.units && L.lpr < kWarp) L.lpr <<= 1;
    L.rows = kWarp / L.lpr;
    L.chunks = (L.units + L.lpr - 1) / L.lpr;
    return L;
}

// p[c * VEC + v] += c1[h, (c * lpr + s) * VEC + v] over the history ids [beg, end) other than excl, for this lane's
// group (sub = lane / lpr) and slot s = lane % lpr; then the groups' sums are added by shuffle, so every lane holds
// the whole sum of its slots.
template <int VEC>
__device__ __forceinline__ void fism_gather(const float* __restrict__ C1, int d, int units, int lpr, int chunks,
                                            const int32_t* __restrict__ idx, int64_t beg, int64_t end, int excl,
                                            float (&p)[kFismPerLane]) {
    const int lane = threadIdx.x & 31, R = kWarp / lpr, sub = lane / lpr, s = lane & (lpr - 1);
#pragma unroll
    for (int e = 0; e < kFismPerLane; ++e) p[e] = 0.0f;
    for (int64_t base = beg; base < end; base += kWarp) {
        const int m = end - base < kWarp ? (int)(end - base) : kWarp;
        const int mine = lane < m ? __ldg(idx + base + lane) : -1;
#pragma unroll(VEC == 4 ? 4 : 2)
        for (int r = 0; r < m; r += R) {
            const int k = r + sub;
            const int h = __shfl_sync(kFull, mine, k);
            if (k < m && h != excl) {
                const float* row = C1 + (size_t)h * d;
#pragma unroll
                for (int c = 0; c < kFismPerLane / VEC; ++c) {
                    const int u = c * lpr + s;
                    if (c < chunks && u < units) {
                        float v[VEC];
                        ld_vec<VEC>(row + u * VEC, v);
#pragma unroll
                        for (int t = 0; t < VEC; ++t) p[c * VEC + t] += v[t];
                    }
                }
            }
        }
    }
    for (int o = lpr; o < kWarp; o <<= 1)
#pragma unroll
        for (int e = 0; e < kFismPerLane; ++e) p[e] += __shfl_xor_sync(kFull, p[e], o);
}

// sum over the lanes of one group (every group holds the same values, so every lane gets the whole sum)
__device__ __forceinline__ float fism_group_sum(float v, int lpr) {
    for (int o = lpr >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// One warp per sample (grid-strided).  third: labels (f32) or negatives (i32); num_neg: n_j (pairwise).
template <int VEC, bool PAIRWISE>
__global__ void __launch_bounds__(kFismWarps * 32)
fism_grad_kernel(const float* __restrict__ C1, const float* __restrict__ Q, const float* __restrict__ B, int d,
                 int units, int lpr, int chunks, const int64_t* __restrict__ ptr, const int32_t* __restrict__ idx,
                 const int32_t* __restrict__ rows, const int32_t* __restrict__ excl, const int32_t* __restrict__ num,
                 const int32_t* __restrict__ items, const void* __restrict__ third,
                 const int32_t* __restrict__ num_neg, int64_t batch, int loss_kind, float alpha, float lambda,
                 float gamma, float inv_b, float* __restrict__ gC1, float* __restrict__ gQ, float* __restrict__ gB,
                 int32_t* __restrict__ tC, int32_t* __restrict__ tQ, int32_t stamp, float* __restrict__ loss) {
    const int lane = threadIdx.x & 31, R = kWarp / lpr, sub = lane / lpr, s = lane & (lpr - 1);
    const int64_t wpb = blockDim.x >> 5;
    float loss_acc = 0.0f;
    for (int64_t b = blockIdx.x * wpb + (threadIdx.x >> 5); b < batch; b += (int64_t)gridDim.x * wpb) {
        const int r = rows[b], i = items[b], ex = excl ? excl[b] : -1;
        const int j = PAIRWISE ? static_cast<const int32_t*>(third)[b] : 0;
        const int64_t beg = ptr[r], end = ptr[r + 1];
        float p[kFismPerLane];
        fism_gather<VEC>(C1, d, units, lpr, chunks, idx, beg, end, ex, p);
        float qi[kFismPerLane], qj[kFismPerLane];
        float di = 0.0f, dj = 0.0f, sp = 0.0f, sq = 0.0f;
#pragma unroll
        for (int c = 0; c < kFismPerLane / VEC; ++c) {
            const int u = c * lpr + s;
            if (c < chunks && u < units) {
                float v[VEC], w[VEC];
                ld_vec<VEC>(Q + (size_t)i * d + u * VEC, v);
                if (PAIRWISE) ld_vec<VEC>(Q + (size_t)j * d + u * VEC, w);
#pragma unroll
                for (int t = 0; t < VEC; ++t) {
                    const int e = c * VEC + t;
                    qi[e] = v[t];
                    di = fmaf(p[e], v[t], di);
                    sp = fmaf(p[e], p[e], sp);
                    sq = fmaf(v[t], v[t], sq);
                    if (PAIRWISE) {
                        qj[e] = w[t];
                        dj = fmaf(p[e], w[t], dj);
                        sq = fmaf(w[t], w[t], sq);
                    }
                }
            } else {
#pragma unroll
                for (int t = 0; t < VEC; ++t) { qi[c * VEC + t] = 0.0f; qj[c * VEC + t] = 0.0f; }
            }
        }
        di = fism_group_sum(di, lpr);
        const float ci = powf((float)num[b], -alpha);
        const float xi = ci * di + B[i];
        float lo, g, cj = 0.0f;
        if (PAIRWISE) {
            dj = fism_group_sum(dj, lpr);
            cj = powf((float)num_neg[b], -alpha);
            pairwise_loss_grad(loss_kind, xi - (cj * dj + B[j]), lo, g);
        } else {
            pointwise_loss_grad(loss_kind, xi, static_cast<const float*>(third)[b], inv_b, lo, g);
        }
        lo += lambda * 0.5f * fism_group_sum(sp, lpr) + gamma * 0.5f * fism_group_sum(sq, lpr);
        loss_acc += lo;
        const float gi = g * ci, gj = -g * cj;
        // the targets' rows and biases: one group writes them
        float gp[kFismPerLane];
#pragma unroll
        for (int c = 0; c < kFismPerLane / VEC; ++c) {
            const int u = c * lpr + s;
            float ai[VEC], aj[VEC];
#pragma unroll
            for (int t = 0; t < VEC; ++t) {
                const int e = c * VEC + t;
                ai[t] = gi * p[e] + gamma * qi[e];
                if (PAIRWISE) {
                    aj[t] = gj * p[e] + gamma * qj[e];
                    gp[e] = (gi * qi[e] + gj * qj[e]) + lambda * p[e];
                } else {
                    gp[e] = gi * qi[e] + lambda * p[e];
                }
            }
            if (sub == 0 && c < chunks && u < units) {
                red_vec<VEC>(gQ + (size_t)i * d + u * VEC, ai);
                if (PAIRWISE) red_vec<VEC>(gQ + (size_t)j * d + u * VEC, aj);
            }
        }
        if (lane == 0) {
            atomicAdd(gB + i, g);
            tQ[i] = stamp;
            if (PAIRWISE) {
                atomicAdd(gB + j, -g);
                tQ[j] = stamp;
            }
        }
        // every history row (once for both sides of a pair) takes dl/dp
        for (int64_t base = beg; base < end; base += kWarp) {
            const int m = end - base < kWarp ? (int)(end - base) : kWarp;
            const int mine = lane < m ? __ldg(idx + base + lane) : -1;
#pragma unroll 4
            for (int q = 0; q < m; q += R) {
                const int k = q + sub;
                const int h = __shfl_sync(kFull, mine, k);
                if (k < m && h != ex) {
                    float* row = gC1 + (size_t)h * d;
#pragma unroll
                    for (int c = 0; c < kFismPerLane / VEC; ++c) {
                        const int u = c * lpr + s;
                        if (c < chunks && u < units) {
                            float v[VEC];
#pragma unroll
                            for (int t = 0; t < VEC; ++t) v[t] = gp[c * VEC + t];
                            red_vec<VEC>(row + u * VEC, v);
                        }
                    }
                    if (s == 0) tC[h] = stamp;
                }
            }
        }
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
}

// p_u over user users[r]'s whole history row, one warp per row (grid-strided): out [rows, d].
template <int VEC>
__global__ void __launch_bounds__(kFismWarps * 32)
fism_query_kernel(const float* __restrict__ C1, int d, int units, int lpr, int chunks, const int64_t* __restrict__ ptr,
                  const int32_t* __restrict__ idx, const int32_t* __restrict__ users, int64_t rows,
                  float* __restrict__ out) {
    const int lane = threadIdx.x & 31, s = lane & (lpr - 1);
    const int64_t wpb = blockDim.x >> 5;
    for (int64_t r = blockIdx.x * wpb + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.x * wpb) {
        const int u = users[r];
        float p[kFismPerLane];
        fism_gather<VEC>(C1, d, units, lpr, chunks, idx, ptr[u], ptr[u + 1], -1, p);
        if (lane < lpr) {
#pragma unroll
            for (int c = 0; c < kFismPerLane / VEC; ++c) {
                const int un = c * lpr + s;
                if (c < chunks && un < units) {
                    float v[VEC];
#pragma unroll
                    for (int t = 0; t < VEC; ++t) v[t] = p[c * VEC + t];
                    st_vec<VEC>(out + (size_t)r * d + un * VEC, v);
                }
            }
        }
    }
}

// out[r, j] = n_r^(-alpha) * <query[r], Q_j> + b_j with n_r the length of user users[r]'s history row: kFismScoreRows
// rows per CTA in shared memory, one item per thread, grid = (row groups, item tiles of 256).  The coefficient and the
// bias are applied in the kernel that forms the dot, as the reference's graph does, so the [rows, I] scores are
// written once.
template <int VEC>
__global__ void __launch_bounds__(256)
fism_scores_kernel(const float* __restrict__ query, const float* __restrict__ Q, const float* __restrict__ B, int d,
                   int32_t num_items, float alpha, const int64_t* __restrict__ ptr, const int32_t* __restrict__ users,
                   int64_t rows, float* __restrict__ out) {
    __shared__ float s_p[kFismScoreRows][kFismMaxDim];
    __shared__ float s_c[kFismScoreRows];
    const int64_t r0 = (int64_t)blockIdx.x * kFismScoreRows;
    const int nr = (rows - r0 < kFismScoreRows) ? (int)(rows - r0) : kFismScoreRows;
    for (int e = threadIdx.x; e < kFismScoreRows * d; e += blockDim.x) {
        const int r = e / d, k = e - r * d;
        s_p[r][k] = r < nr ? query[(size_t)(r0 + r) * d + k] : 0.0f;
    }
    if (threadIdx.x < kFismScoreRows) {
        const int r = threadIdx.x;
        float c = 0.0f;
        if (r < nr) {
            const int u = users[r0 + r];
            c = powf((float)(ptr[u + 1] - ptr[u]), -alpha);
        }
        s_c[r] = c;
    }
    __syncthreads();
    const int64_t j = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
    if (j >= num_items) return;
    const float* __restrict__ q = Q + (size_t)j * d;
    float acc[kFismScoreRows];
#pragma unroll
    for (int r = 0; r < kFismScoreRows; ++r) acc[r] = 0.0f;
    for (int k = 0; k < d; k += VEC) {
        float v[VEC];
        ld_vec<VEC>(q + k, v);
#pragma unroll
        for (int t = 0; t < VEC; ++t)
#pragma unroll
            for (int r = 0; r < kFismScoreRows; ++r) acc[r] = fmaf(s_p[r][k + t], v[t], acc[r]);
    }
    const float bj = __ldg(B + j);
#pragma unroll
    for (int r = 0; r < kFismScoreRows; ++r)
        if (r < nr) out[(size_t)(r0 + r) * num_items + j] = s_c[r] * acc[r] + bj;
}

}  // namespace nrc

using namespace nrc;

// Host record of FISM's launches, for nrc_fism_last_routes (see the header); -1 = no such launch yet, or a field the
// kernel does not decide.  Written just before the launch.
enum FismKernel { kFiGrad, kFiQuery, kFiScores, kFiKernels };
enum FismField { kFiPairwise, kFiVec, kFiLanes, kFiGridX, kFiGridY, kFiCapped, kFiFields };
static struct FismRoutes {
    int32_t r[kFiKernels][kFiFields];
    FismRoutes() { for (auto& k : r) for (auto& f : k) f = -1; }
} g_fism_routes;

static void fism_route(int kernel, int pairwise, int vec, int lanes, int64_t grid_x, int64_t grid_y, int capped) {
    int32_t* r = g_fism_routes.r[kernel];
    r[kFiPairwise] = pairwise; r[kFiVec] = vec; r[kFiLanes] = lanes; r[kFiGridX] = (int32_t)grid_x;
    r[kFiGridY] = (int32_t)grid_y; r[kFiCapped] = capped;
}

// CTAs of a warp-per-sample launch over `work` samples or rows, and whether the cap made a warp take more than one
static unsigned fism_grid(int64_t work, int* capped) {
    int64_t blocks = (work + kFismWarps - 1) / kFismWarps;
    const int64_t cap = (int64_t)sm_count() * kFismCtasPerSm;
    *capped = blocks > cap ? 1 : 0;
    if (blocks > cap) blocks = cap;
    return (unsigned)(blocks < 1 ? 1 : blocks);
}

static int fism_check(int32_t num_items, int32_t dim, int32_t pairwise, int32_t loss_kind, int64_t batch,
                      float alpha) {
    NRC_REQUIRE(dim >= 1 && dim <= kFismMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kFismMaxDim);
    NRC_REQUIRE(num_items >= 1, NRC_E_VALUE, "num_items >= 1 required");
    // learner.py:27-28 / 39-40
    if (pairwise)
        NRC_REQUIRE(loss_kind == NRC_LOSS_BPR || loss_kind == NRC_LOSS_HINGE || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                    "please choose a suitable loss function");
    else
        NRC_REQUIRE(loss_kind == NRC_LOSS_CROSS_ENTROPY || loss_kind == NRC_LOSS_SQUARE, NRC_E_VALUE,
                    "please choose a suitable loss function");
    NRC_REQUIRE(batch >= 0, NRC_E_VALUE, "batch >= 0 required");
    NRC_REQUIRE(alpha == alpha && alpha > -INFINITY && alpha < INFINITY, NRC_E_VALUE, "alpha must be finite");
    return NRC_OK;
}

extern "C" int nrc_fism_grad(const float* c1, const float* q, const float* bias, int32_t num_items, int32_t dim,
                             const int64_t* hist_ptr, const int32_t* hist_idx, const int32_t* rows,
                             const int32_t* excl, const int32_t* num, const int32_t* items, const void* third,
                             const int32_t* num_neg, int64_t batch, int32_t pairwise, int32_t loss_kind, float alpha,
                             float lambda, float gamma, float* grad_c1, float* grad_q, float* grad_bias,
                             int32_t* touched_c1, int32_t* touched_item, int32_t stamp, float* loss, void* stream) {
    const int rc = fism_check(num_items, dim, pairwise, loss_kind, batch, alpha);
    if (rc) return rc;
    // an empty batch launches nothing and may come without arrays, as in nrc_fism_query
    NRC_REQUIRE(batch == 0 || (c1 && q && bias && hist_ptr && hist_idx && rows && num && items && third), NRC_E_VALUE,
                "tables, the history CSR and the batch are required");
    NRC_REQUIRE(batch == 0 || !pairwise || num_neg, NRC_E_VALUE, "num_neg is required in the pairwise form");
    NRC_REQUIRE(grad_c1 && grad_q && grad_bias && touched_c1 && touched_item, NRC_E_VALUE,
                "gradients and touched stamps are required");
    if (batch == 0) return NRC_OK;
    const FismLanes L = fism_lanes(dim);
    int capped;
    const unsigned grid = fism_grid(batch, &capped);
    fism_route(kFiGrad, pairwise ? 1 : 0, L.vec, L.lpr, grid, -1, capped);
    const float inv_b = 1.0f / (float)batch;
    cudaStream_t st = as_stream(stream);
#define FISM_GRAD(V, P)                                                                                                \
    fism_grad_kernel<V, P><<<grid, kFismWarps * 32, 0, st>>>(                                                          \
        c1, q, bias, dim, L.units, L.lpr, L.chunks, hist_ptr, hist_idx, rows, excl, num, items, third, num_neg, batch, \
        loss_kind, alpha, lambda, gamma, inv_b, grad_c1, grad_q, grad_bias, touched_c1, touched_item, stamp, loss)
    if (L.vec == 4) {
        if (pairwise) FISM_GRAD(4, true); else FISM_GRAD(4, false);
    } else {
        if (pairwise) FISM_GRAD(1, true); else FISM_GRAD(1, false);
    }
#undef FISM_GRAD
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_fism_train_epoch(float* c1, float* q, float* bias, int32_t num_items, int32_t dim,
                                    const int64_t* hist_ptr, const int32_t* hist_idx, const int32_t* rows,
                                    const int32_t* excl, const int32_t* num, const int32_t* items, const void* third,
                                    const int32_t* num_neg, int64_t n, int32_t batch_size, int32_t pairwise,
                                    int32_t loss_kind, float alpha, float lambda, float gamma, int32_t opt_kind,
                                    const float* lr_t_host, const float* hyper_host, float* grad_c1, float* grad_q,
                                    float* grad_bias, int32_t* touched_c1, int32_t* touched_item,
                                    float* const* slot0, float* const* slot1, int32_t first_stamp, float* step_loss,
                                    void* stream) {
    int rc = fism_check(num_items, dim, pairwise, loss_kind, n, alpha);
    if (rc) return rc;
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    // learner.py:14-15
    NRC_REQUIRE(opt_kind >= NRC_OPT_GD && opt_kind <= NRC_OPT_MOMENTUM, NRC_E_VALUE, "please select a suitable optimizer");
    NRC_REQUIRE(lr_t_host && hyper_host && slot0 && slot1 && step_loss, NRC_E_VALUE,
                "lr_t_host, hyper_host, slot0, slot1 (the three variables' slots) and step_loss are required");
    // an empty epoch may come without arrays: seq_epoch_loop runs no gradient step and no optimizer pass at n = 0
    NRC_REQUIRE(n == 0 || (c1 && q && bias && hist_ptr && hist_idx && rows && num && items && third), NRC_E_VALUE,
                "tables, the history CSR and the samples are required");
    NRC_REQUIRE(n == 0 || !pairwise || num_neg, NRC_E_VALUE, "num_neg is required in the pairwise form");
    NRC_REQUIRE(grad_c1 && grad_q && grad_bias && touched_c1 && touched_item, NRC_E_VALUE,
                "gradients and touched stamps are required");
    const size_t tsz = pairwise ? sizeof(int32_t) : sizeof(float);
    return seq_epoch_loop(
        n, batch_size, opt_kind, lr_t_host, hyper_host, first_stamp, step_loss, as_stream(stream),
        [&](int64_t off, int64_t bs, int32_t stamp, float* loss) {
            return nrc_fism_grad(c1, q, bias, num_items, dim, hist_ptr, hist_idx, rows + off, excl ? excl + off : nullptr,
                                 num + off, items + off, static_cast<const char*>(third) + off * tsz,
                                 pairwise ? num_neg + off : nullptr, bs, pairwise, loss_kind, alpha, lambda, gamma,
                                 grad_c1, grad_q, grad_bias, touched_c1, touched_item, stamp, loss, stream);
        },
        [&](OptLaunch& Lo) {
            // IndexedSlices gradients: touched rows for adagrad / rmsprop / momentum, Adam's sparse form on every row
            opt_launch_add(Lo, c1, grad_c1, slot0[0], slot1[0], touched_c1, num_items, dim, 0);
            opt_launch_add(Lo, q, grad_q, slot0[1], slot1[1], touched_item, num_items, dim, 0);
            opt_launch_add(Lo, bias, grad_bias, slot0[2], slot1[2], touched_item, num_items, 1, 0);
        });
}

extern "C" int nrc_fism_query(const float* c1, int32_t num_items, int32_t dim, const int64_t* hist_ptr,
                              const int32_t* hist_idx, const int32_t* users, int64_t rows, float* out, void* stream) {
    NRC_REQUIRE(dim >= 1 && dim <= kFismMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kFismMaxDim);
    NRC_REQUIRE(num_items >= 1 && rows >= 0, NRC_E_VALUE, "num_items >= 1 and rows >= 0 required");
    NRC_REQUIRE(rows == 0 || (c1 && hist_ptr && hist_idx && users && out), NRC_E_VALUE,
                "c1, the history CSR, users and out are required");
    if (rows == 0) return NRC_OK;
    const FismLanes L = fism_lanes(dim);
    int capped;
    const unsigned grid = fism_grid(rows, &capped);
    fism_route(kFiQuery, -1, L.vec, L.lpr, grid, -1, capped);
    cudaStream_t st = as_stream(stream);
    if (L.vec == 4)
        fism_query_kernel<4><<<grid, kFismWarps * 32, 0, st>>>(c1, dim, L.units, L.lpr, L.chunks, hist_ptr, hist_idx,
                                                               users, rows, out);
    else
        fism_query_kernel<1><<<grid, kFismWarps * 32, 0, st>>>(c1, dim, L.units, L.lpr, L.chunks, hist_ptr, hist_idx,
                                                               users, rows, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_fism_scores(const float* query, const float* q, const float* bias, int32_t num_items, int32_t dim,
                               float alpha, const int64_t* hist_ptr, const int32_t* users, int64_t rows, float* out,
                               void* stream) {
    NRC_REQUIRE(dim >= 1 && dim <= kFismMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kFismMaxDim);
    NRC_REQUIRE(num_items >= 1 && rows >= 0, NRC_E_VALUE, "num_items >= 1 and rows >= 0 required");
    NRC_REQUIRE(alpha == alpha && alpha > -INFINITY && alpha < INFINITY, NRC_E_VALUE, "alpha must be finite");
    NRC_REQUIRE(rows == 0 || (query && q && bias && hist_ptr && users && out), NRC_E_VALUE,
                "query, Q, bias, the history row pointers, users and out are required");
    const int64_t groups = (rows + kFismScoreRows - 1) / kFismScoreRows;
    NRC_REQUIRE(groups <= 0x7fffffff, NRC_E_LIMIT, "rows %lld above %lld", (long long)rows,
                (long long)0x7fffffff * kFismScoreRows);
    NRC_REQUIRE((num_items + 255) / 256 <= 65535, NRC_E_LIMIT, "num_items %d above %d", num_items, 65535 * 256);
    if (rows == 0) return NRC_OK;
    const int vec = dim % 4 == 0 ? 4 : 1;
    const dim3 grid((unsigned)groups, (unsigned)((num_items + 255) / 256));
    fism_route(kFiScores, -1, vec, -1, grid.x, grid.y, 0);
    cudaStream_t st = as_stream(stream);
    if (vec == 4)
        fism_scores_kernel<4><<<grid, 256, 0, st>>>(query, q, bias, dim, num_items, alpha, hist_ptr, users, rows, out);
    else
        fism_scores_kernel<1><<<grid, 256, 0, st>>>(query, q, bias, dim, num_items, alpha, hist_ptr, users, rows, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// Host bookkeeping of the routes the most recent FISM launches took (see the header); no device work.
extern "C" int nrc_fism_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "out is NULL");
    for (int k = 0; k < kFiKernels; ++k)
        for (int f = 0; f < kFiFields; ++f) out[k * kFiFields + f] = g_fism_routes.r[k][f];
    return NRC_OK;
}
