// Caser: a vertical and a horizontal convolution over the embeddings of the last L items, a max-pool over time,
// dropout and a dense layer, whose output joins the user's row to score the next T items against sampled negatives.
//
// Replaces (reference paths):
//   model/sequential_recommender/Caser.py:37-122   variables, the convolutional graph, loss and Adam
//   model/sequential_recommender/Caser.py:124-142  train_model's batch loop (sess.run(train_opt) per batch)
//   model/sequential_recommender/Caser.py:194-209  predict's user vectors (scores by nrc_mf_scores, without the biases)
//
// Variables: P [U, d] (user_embeddings), E [I, d] (seq_item_embeddings; id I is the pad id and reads a zero row),
// W2 [I, 2d] (item_embeddings), b2 [I] (item_biases) and the dense block (see nrc_caser_dense_floats in the header
// for its layout).  For a sample with user u, window w_0..w_{L-1} and image X[l] = E[w_l]:
//   out_v[k nv + f]       = sum_l X[l, k] Kv[l, f] + bv[f]
//   out_h[(h-1) nh + f]   = max_t relu(sum_{l<h, k} X[t + l, k] Kh_h[l, k, f] + bh_h[f])        h = 1..L
//   o = dropout([out_v, out_h]) = ([out_v, out_h] / keep) * mask,   z = relu(o W1 + b1)
//   x_j = <[z, P_u], W2[j]> + b2[j] over the T positives and N negatives (a pad target reads a zero row and bias)
//   loss = mean_pos(-log(sigmoid(x) + 1e-24)) + mean_neg(-log(1 - sigmoid(x) + 1e-24)) + l2_reg * l2_loss(P, E, W2, b2)
// Backward as TF: the max passes grad / n to each of the n tied maxima, relu passes where its output is > 0, dropout
// passes (grad * mask) / keep.  The tables' row gradients go to dense accumulators with atomics; the l2 term enters
// through caser_reg_kernel, which sets every table's accumulator to l2_reg * var before the gradient kernel runs.  The
// dense block's gradient takes no atomics: the gradient kernel writes each sample's layer inputs and output gradients
// to work, and caser_wgrad_kernel forms the products in chunks of kCaserChunk samples, each chunk in sample order and
// then the chunks in chunk order -- the same bits on every call.
#include "common.cuh"
#include "optim.cuh"
#include "seq_epoch.cuh"

namespace nrc {

constexpr int kCaserMaxDim = 256;
constexpr int kCaserMaxL = 16;
constexpr int kCaserMaxFilters = 64;          // nv and nh
constexpr int kCaserMaxTargets = 64;          // T + N
constexpr int kCaserChunk = 32;               // samples per partial sum of the dense gradient
constexpr int kCaserSmemFloats = 56 * 1024;   // dynamic shared memory of one CTA (224 KB of the 227 KB opt-in)

struct CaserDims {
    int d, L, nv, nh, T, N, I;
    int F;     // nv d + nh L: width of the pooled features
    int NH;    // nh L (L + 1) / 2: conv_h outputs over every height and position
    int Dn;    // floats of the dense block
};

// first conv_h output position of height h (1-based) in the [height, position] order: sum_{h' < h} (L - h' + 1)
__host__ __device__ inline int caser_pos_off(int L, int h) { return (h - 1) * (L + 1) - (h - 1) * h / 2; }
// offset of Kh_h in the dense block; bh_h follows it at + h d nh
__host__ __device__ inline int caser_kh_off(const CaserDims& D, int h) {
    return D.L * D.nv + D.nv + (h - 1) * h / 2 * D.d * D.nh + (h - 1) * D.nh;
}
__host__ __device__ inline int caser_w1_off(const CaserDims& D) { return caser_kh_off(D, D.L + 1); }

static CaserDims caser_dims(int d, int L, int nv, int nh, int T, int N, int I) {
    CaserDims D;
    D.d = d; D.L = L; D.nv = nv; D.nh = nh; D.T = T; D.N = N; D.I = I;
    D.F = nv * d + nh * L;
    D.NH = nh * L * (L + 1) / 2;
    D.Dn = caser_w1_off(D) + D.F * d + d;
    return D;
}

// Per-sample factors in work: [X: L d][o: F][dz: d (gradient at o W1 + b1)][gv: L nv + nv (the sample's Kv and bv
// gradients, summed over d in the gradient kernel)][dh: NH (gradient at the conv_h pre-activations)].
__host__ __device__ inline int64_t caser_factor_floats(const CaserDims& D) {
    return (int64_t)D.L * D.d + D.F + D.d + (int64_t)(D.L + 1) * D.nv + D.NH;
}
// Shared memory of the gradient and query kernels besides the staged weights: X, the conv_h outputs, o, [z, P_u], the
// pre-activation of z and the target coefficients.
static int64_t caser_smem_work(const CaserDims& D) {
    return (int64_t)D.L * D.d + D.NH + D.F + 3 * (int64_t)D.d + kCaserMaxTargets;
}
static bool caser_staged(const CaserDims& D) { return D.Dn + caser_smem_work(D) <= kCaserSmemFloats; }
static size_t caser_smem_bytes(const CaserDims& D) {
    return (size_t)((caser_staged(D) ? D.Dn : 0) + caser_smem_work(D)) * sizeof(float);
}
static int64_t caser_counters(const CaserDims& D) { return (D.Dn + 255) / 256; }
static int64_t caser_chunks(int64_t batch) { return (batch + kCaserChunk - 1) / kCaserChunk; }

// Copies the dense block into shared memory when it fits (the staged route); returns where the CTA reads it from.
__device__ __forceinline__ const float* caser_weights(const CaserDims& D, const float* __restrict__ dense, bool staged,
                                                      float* sW) {
    if (!staged) return dense;
    for (int e = threadIdx.x; e < D.Dn; e += blockDim.x) sW[e] = dense[e];
    __syncthreads();
    return sW;
}

// Loads X (pad id -> zero row) and P_u into shared memory; X also to the sample's factors when fX is not NULL.
__device__ __forceinline__ void caser_gather(const CaserDims& D, const float* __restrict__ P, const float* __restrict__ E,
                                             int u, const int32_t* __restrict__ win, float* sX, float* sU,
                                             float* __restrict__ fX) {
    for (int e = threadIdx.x; e < D.L * D.d; e += blockDim.x) {
        const int l = e / D.d, k = e - l * D.d;
        const int id = win[l];
        const float v = id == D.I ? 0.0f : E[(size_t)id * D.d + k];
        sX[e] = v;
        if (fX) fX[e] = v;
    }
    for (int k = threadIdx.x; k < D.d; k += blockDim.x) sU[D.d + k] = P[(size_t)u * D.d + k];
    __syncthreads();
}

// The forward pass of one sample from X in shared memory: conv_h outputs to act, the (dropped-out) features to o,
// the pre-activation of z to zp and z to u[0, d).  mask = NULL: no dropout.
__device__ void caser_forward(const CaserDims& D, const float* W, const float* sX, float* act, float* o, float* zp,
                              float* u, const float* __restrict__ mask, float keep) {
    const int d = D.d, L = D.L, nv = D.nv, nh = D.nh;
    for (int e = threadIdx.x; e < nv * d; e += blockDim.x) {
        const int k = e / nv, f = e - k * nv;
        float s = 0.0f;
        for (int l = 0; l < L; ++l) s = fmaf(sX[l * d + k], W[l * nv + f], s);
        s += W[L * nv + f];
        o[e] = mask ? (s / keep) * mask[e] : s;
    }
    for (int e = threadIdx.x; e < D.NH; e += blockDim.x) {
        const int p = e / nh, f = e - p * nh;
        int h = 1;
        while (p >= caser_pos_off(L, h + 1)) ++h;
        const int t = p - caser_pos_off(L, h);
        const float* Kh = W + caser_kh_off(D, h);
        float s = 0.0f;
        for (int l = 0; l < h; ++l)
            for (int k = 0; k < d; ++k) s = fmaf(sX[(t + l) * d + k], Kh[(l * d + k) * nh + f], s);
        act[e] = fmaxf(s + Kh[h * d * nh + f], 0.0f);
    }
    __syncthreads();
    for (int e = threadIdx.x; e < nh * L; e += blockDim.x) {
        const int h = e / nh + 1, f = e - (h - 1) * nh;
        const float* a = act + caser_pos_off(L, h) * nh + f;
        float m = a[0];
        for (int t = 1; t <= L - h; ++t) m = fmaxf(m, a[t * nh]);
        const int r = nv * d + e;
        o[r] = mask ? (m / keep) * mask[r] : m;
    }
    __syncthreads();
    // z = relu(o W1 + b1): one warp per column, the lanes over the rows, a fixed shuffle order
    const float* W1 = W + caser_w1_off(D);
    const int lane = threadIdx.x & 31;
    for (int c = threadIdx.x >> 5; c < d; c += blockDim.x >> 5) {
        float s = 0.0f;
        for (int r = lane; r < D.F; r += kWarp) s = fmaf(o[r], W1[(size_t)r * d + c], s);
        s = warp_sum(s);
        if (lane == 0) {
            s += W1[(size_t)D.F * d + c];
            zp[c] = s;
            u[c] = fmaxf(s, 0.0f);
        }
    }
    __syncthreads();
}

// One CTA per sample (grid-strided).  fac: the per-sample factors (caser_factor_floats each).
__global__ void __launch_bounds__(256)
caser_grad_kernel(CaserDims D, const float* __restrict__ P, const float* __restrict__ E, const float* __restrict__ W2,
                  const float* __restrict__ B2, const float* __restrict__ dense, bool staged,
                  const int32_t* __restrict__ users, const int32_t* __restrict__ seqs, const int32_t* __restrict__ pos,
                  const int32_t* __restrict__ neg, int64_t batch, const float* __restrict__ mask, float keep,
                  float inv_bt, float inv_bn, float* __restrict__ gP, float* __restrict__ gE, float* __restrict__ gW2,
                  float* __restrict__ gB2, float* __restrict__ fac, float* __restrict__ loss) {
    extern __shared__ float sm[];
    const int d = D.d, L = D.L, nv = D.nv, nh = D.nh, F = D.F, nt = D.T + D.N, d2 = 2 * D.d;
    float* sX = sm + (staged ? D.Dn : 0);
    float* act = sX + L * d;
    float* o = act + D.NH;
    float* u = o + F;
    float* zp = u + d2;
    float* cj = zp + d;
    const float* W = caser_weights(D, dense, staged, sm);
    const float* W1 = W + caser_w1_off(D);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int64_t S = caser_factor_floats(D);
    float loss_acc = 0.0f;
    for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
        const int uid = users[b];
        const int32_t* win = seqs + b * L;
        float* f = fac + b * S;
        float* fO = f + L * d;
        float* fDz = fO + F;
        float* fGv = fDz + d;
        float* fDh = fGv + (L + 1) * nv;
        const float* m = mask ? mask + b * F : nullptr;
        caser_gather(D, P, E, uid, win, sX, u, f);
        caser_forward(D, W, sX, act, o, zp, u, m, keep);
        // targets: one warp each; c_j = dloss / dx_j
        for (int j = warp; j < nt; j += nwarps) {
            const int id = j < D.T ? pos[b * D.T + j] : neg[b * D.N + (j - D.T)];
            float x = 0.0f;
            if (id != D.I) {
                for (int k = lane; k < d2; k += kWarp) x = fmaf(u[k], W2[(size_t)id * d2 + k], x);
                x = warp_sum(x) + B2[id];
            }
            if (lane == 0) {
                const float s = 1.0f / (1.0f + expf(-x));
                float c;
                if (j < D.T) {
                    loss_acc += -logf(s + 1e-24f) * inv_bt;
                    c = ((-inv_bt) * (1.0f / (s + 1e-24f))) * s * (1.0f - s);
                } else {
                    loss_acc += -logf((1.0f - s) + 1e-24f) * inv_bn;
                    c = (inv_bn * (1.0f / ((1.0f - s) + 1e-24f))) * s * (1.0f - s);
                }
                cj[j] = c;
            }
        }
        __syncthreads();
        // targets' rows and biases; the gradient at [z, P_u]: P_u's to its row, z's through relu into zp
        for (int e = threadIdx.x; e < nt * d2; e += blockDim.x) {
            const int j = e / d2, k = e - j * d2;
            const int id = j < D.T ? pos[b * D.T + j] : neg[b * D.N + (j - D.T)];
            if (id != D.I) atomicAdd(gW2 + (size_t)id * d2 + k, cj[j] * u[k]);
        }
        for (int j = threadIdx.x; j < nt; j += blockDim.x) {
            const int id = j < D.T ? pos[b * D.T + j] : neg[b * D.N + (j - D.T)];
            if (id != D.I) atomicAdd(gB2 + id, cj[j]);
        }
        for (int k = threadIdx.x; k < d2; k += blockDim.x) {
            float g = 0.0f;
            for (int j = 0; j < nt; ++j) {
                const int id = j < D.T ? pos[b * D.T + j] : neg[b * D.N + (j - D.T)];
                if (id != D.I) g = fmaf(cj[j], W2[(size_t)id * d2 + k], g);
            }
            if (k >= d) {
                atomicAdd(gP + (size_t)uid * d + (k - d), g);
            } else {
                const float dz = u[k] > 0.0f ? g : 0.0f;
                zp[k] = dz;
                fDz[k] = dz;
            }
        }
        __syncthreads();
        // the gradient at o (W1 dz), then through dropout; o itself goes to the factors first
        for (int r = threadIdx.x; r < F; r += blockDim.x) {
            float g = 0.0f;
            for (int c = 0; c < d; ++c) g = fmaf(W1[(size_t)r * d + c], zp[c], g);
            fO[r] = o[r];
            const float dr = m ? (g * m[r]) / keep : g;
            o[r] = dr;
        }
        __syncthreads();
        // the sample's Kv and bv gradients from out_v's gradient (o[0, nv d)), summed over k in order
        for (int e = threadIdx.x; e < (L + 1) * nv; e += blockDim.x) {
            const int l = e / nv, fi = e - l * nv;
            float g = 0.0f;
            if (l < L)
                for (int k = 0; k < d; ++k) g = fmaf(sX[l * d + k], o[k * nv + fi], g);
            else
                for (int k = 0; k < d; ++k) g += o[k * nv + fi];
            fGv[e] = g;
        }
        // max-pool and relu backward, in place over the conv_h outputs: act becomes the gradient at the pre-activations
        for (int e = threadIdx.x; e < nh * L; e += blockDim.x) {
            const int h = e / nh + 1, fi = e - (h - 1) * nh;
            float* a = act + caser_pos_off(L, h) * nh + fi;
            float mx = a[0];
            for (int t = 1; t <= L - h; ++t) mx = fmaxf(mx, a[t * nh]);
            int ties = 0;
            for (int t = 0; t <= L - h; ++t) ties += a[t * nh] == mx;
            const float g = (1.0f / (float)ties) * o[nv * d + e];
            for (int t = 0; t <= L - h; ++t) {
                const float av = a[t * nh];
                const float gt = (av == mx && av > 0.0f) ? g : 0.0f;
                a[t * nh] = gt;
                fDh[(caser_pos_off(L, h) + t) * nh + fi] = gt;
            }
        }
        __syncthreads();
        // the window rows: conv_v's and every conv_h's transposed products
        for (int e = threadIdx.x; e < L * d; e += blockDim.x) {
            const int lp = e / d, k = e - lp * d;
            const int id = win[lp];
            if (id == D.I) continue;
            float g = 0.0f;
            for (int fi = 0; fi < nv; ++fi) g = fmaf(o[k * nv + fi], W[lp * nv + fi], g);
            for (int h = 1; h <= L; ++h) {
                const float* Kh = W + caser_kh_off(D, h);
                const float* a = act + caser_pos_off(L, h) * nh;
                const int l0 = lp - (L - h) > 0 ? lp - (L - h) : 0, l1 = lp < h - 1 ? lp : h - 1;
                for (int l = l0; l <= l1; ++l) {
                    const int t = lp - l;
                    for (int fi = 0; fi < nh; ++fi) g = fmaf(a[t * nh + fi], Kh[(l * d + k) * nh + fi], g);
                }
            }
            atomicAdd(gE + (size_t)id * d + k, g);
        }
        __syncthreads();
    }
    if (lane == 0 && loss && loss_acc != 0.0f) atomicAdd(loss, loss_acc);
}

// The dense block's gradient from the per-sample factors.  grid = (element tiles of 256, chunks of kCaserChunk
// samples): each CTA sums its chunk in sample order into partial[chunk]; the last CTA of an element tile to finish
// writes the sum of the chunks in chunk order to grad and resets the tile's counter.
__global__ void __launch_bounds__(256)
caser_wgrad_kernel(CaserDims D, int64_t batch, const float* __restrict__ fac, float* __restrict__ partial,
                   unsigned* __restrict__ counters, float* __restrict__ grad) {
    __shared__ bool s_last;
    const int d = D.d, L = D.L, nv = D.nv, nh = D.nh;
    const int64_t S = caser_factor_floats(D);
    const int oO = L * d, oDz = oO + D.F, oGv = oDz + d, oDh = oGv + (L + 1) * nv;
    const int oW1 = caser_w1_off(D);
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t b0 = (int64_t)blockIdx.y * kCaserChunk;
    const int64_t b1 = (batch - b0 < kCaserChunk) ? batch : b0 + kCaserChunk;
    if (e < D.Dn) {
        float s = 0.0f;
        const int q = (int)e;
        if (q < (L + 1) * nv) {                             // Kv[l, f] and bv[f]: the samples' own sums
            for (int64_t b = b0; b < b1; ++b) s += fac[b * S + oGv + q];
        } else if (q < oW1) {                               // Kh_h[l, k, f] and bh_h[f]
            int h = 1;
            while (q >= caser_kh_off(D, h + 1)) ++h;
            const int r = q - caser_kh_off(D, h), np = L - h + 1, p0 = caser_pos_off(L, h);
            if (r < h * d * nh) {
                const int l = r / (d * nh), k = (r / nh) % d, f = r % nh;
                for (int64_t b = b0; b < b1; ++b) {
                    const float* x = fac + b * S;
                    for (int t = 0; t < np; ++t) s = fmaf(x[(t + l) * d + k], x[oDh + (p0 + t) * nh + f], s);
                }
            } else {
                const int f = r - h * d * nh;
                for (int64_t b = b0; b < b1; ++b)
                    for (int t = 0; t < np; ++t) s += fac[b * S + oDh + (p0 + t) * nh + f];
            }
        } else if (q < oW1 + D.F * d) {                     // W1[r, c]
            const int r = (q - oW1) / d, c = (q - oW1) - r * d;
            for (int64_t b = b0; b < b1; ++b) s = fmaf(fac[b * S + oO + r], fac[b * S + oDz + c], s);
        } else {                                            // b1[c]
            const int c = q - oW1 - D.F * d;
            for (int64_t b = b0; b < b1; ++b) s += fac[b * S + oDz + c];
        }
        partial[(size_t)blockIdx.y * D.Dn + e] = s;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(counters + blockIdx.x, 1u) == gridDim.y - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (e < D.Dn) {
        float s = 0.0f;
        for (unsigned k = 0; k < gridDim.y; ++k) s += __ldcg(partial + (size_t)k * D.Dn + e);
        grad[e] = s;
    }
    if (threadIdx.x == 0) counters[blockIdx.x] = 0u;
}

// Every table's gradient accumulator <- l2_reg * var (0 when l2_reg = 0): the dense reg term of the step.
struct CaserRegSegs {
    const float* var[4];
    float* grad[4];
    int64_t n[4];
};

__global__ void __launch_bounds__(256)
caser_reg_kernel(CaserRegSegs S, int64_t total, float reg) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        int64_t q = e;
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            if (q >= 0 && q < S.n[s]) S.grad[s][q] = reg != 0.0f ? reg * S.var[s][q] : 0.0f;
            q -= S.n[s];
        }
    }
}

// The user vectors [z, P_u] without dropout, one CTA per row (grid-strided).
__global__ void __launch_bounds__(256)
caser_query_kernel(CaserDims D, const float* __restrict__ P, const float* __restrict__ E,
                   const float* __restrict__ dense, bool staged, const int32_t* __restrict__ users, int64_t rows,
                   const int32_t* __restrict__ windows, float* __restrict__ out) {
    extern __shared__ float sm[];
    const int d = D.d, L = D.L;
    float* sX = sm + (staged ? D.Dn : 0);
    float* act = sX + L * d;
    float* o = act + D.NH;
    float* u = o + D.F;
    float* zp = u + 2 * d;
    const float* W = caser_weights(D, dense, staged, sm);
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const int uid = users[r];
        caser_gather(D, P, E, uid, windows + (size_t)uid * L, sX, u, nullptr);
        caser_forward(D, W, sX, act, o, zp, u, nullptr, 1.0f);
        for (int k = threadIdx.x; k < 2 * d; k += blockDim.x) out[(size_t)r * 2 * d + k] = u[k];
        __syncthreads();
    }
}

}  // namespace nrc

using namespace nrc;

// Host record of Caser's launches, for nrc_caser_last_routes (see the header); -1 = no such launch yet, or a field the
// kernel does not decide.  Written just before the launch.
enum CaserKernel { kCaGrad, kCaWgrad, kCaQuery, kCaReg, kCaKernels };
enum CaserField { kCaStaged, kCaGridX, kCaGridY, kCaCapped, kCaWindow, kCaMasked, kCaFields };
static struct CaserRoutes {
    int32_t r[kCaKernels][kCaFields];
    CaserRoutes() { for (auto& k : r) for (auto& f : k) f = -1; }
} g_caser_routes;

static void caser_route(int kernel, int staged, int64_t grid_x, int64_t grid_y, int capped, int window, int masked) {
    int32_t* r = g_caser_routes.r[kernel];
    r[kCaStaged] = staged; r[kCaGridX] = (int32_t)grid_x; r[kCaGridY] = (int32_t)grid_y; r[kCaCapped] = capped;
    r[kCaWindow] = window; r[kCaMasked] = masked;
}

static int caser_check_shape(int32_t dim, int32_t seq_L, int32_t nv, int32_t nh) {
    NRC_REQUIRE(dim >= 1 && dim <= kCaserMaxDim, NRC_E_LIMIT, "dim %d outside [1, %d]", dim, kCaserMaxDim);
    NRC_REQUIRE(seq_L >= 1 && seq_L <= kCaserMaxL, NRC_E_LIMIT, "seq_L %d outside [1, %d]", seq_L, kCaserMaxL);
    NRC_REQUIRE(nv >= 1 && nv <= kCaserMaxFilters && nh >= 1 && nh <= kCaserMaxFilters, NRC_E_LIMIT,
                "nv %d and nh %d must lie in [1, %d]", nv, nh, kCaserMaxFilters);
    return NRC_OK;
}

static int caser_check_targets(int32_t seq_T, int32_t neg_samples) {
    NRC_REQUIRE(seq_T >= 1 && neg_samples >= 1, NRC_E_VALUE, "seq_T and neg_samples must be positive");
    NRC_REQUIRE(seq_T + neg_samples <= kCaserMaxTargets, NRC_E_LIMIT, "seq_T + neg_samples = %d above %d",
                seq_T + neg_samples, kCaserMaxTargets);
    return NRC_OK;
}

static int caser_check_batch(int64_t batch) {
    NRC_REQUIRE(batch >= 0, NRC_E_VALUE, "batch >= 0 required");
    NRC_REQUIRE(caser_chunks(batch) <= 65535, NRC_E_LIMIT, "batch %lld above %d", (long long)batch,
                65535 * kCaserChunk);
    return NRC_OK;
}

extern "C" int64_t nrc_caser_dense_floats(int32_t dim, int32_t seq_L, int32_t nv, int32_t nh) {
    const int rc = caser_check_shape(dim, seq_L, nv, nh);
    if (rc) return rc;
    return caser_dims(dim, seq_L, nv, nh, 1, 1, 0).Dn;
}

extern "C" int64_t nrc_caser_work_floats(int32_t dim, int32_t seq_L, int32_t nv, int32_t nh, int32_t batch_size) {
    const int rc = caser_check_shape(dim, seq_L, nv, nh);
    if (rc) return rc;
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    const int rb = caser_check_batch(batch_size);
    if (rb) return rb;
    const CaserDims D = caser_dims(dim, seq_L, nv, nh, 1, 1, 0);
    return caser_counters(D) + (int64_t)batch_size * caser_factor_floats(D) + caser_chunks(batch_size) * D.Dn +
           (int64_t)batch_size * D.F;
}

extern "C" int nrc_caser_grad(const float* user_table, const float* seq_table, const float* item_table,
                              const float* item_bias, const float* dense, int32_t num_items, int32_t dim,
                              int32_t seq_L, int32_t seq_T, int32_t nv, int32_t nh, int32_t neg_samples,
                              const int32_t* users, const int32_t* seqs, const int32_t* pos, const int32_t* neg,
                              int64_t batch, const float* mask, float keep, float* grad_user, float* grad_seq,
                              float* grad_item, float* grad_bias, float* grad_dense, float* work, float* loss,
                              void* stream) {
    int rc = caser_check_shape(dim, seq_L, nv, nh);
    if (rc) return rc;
    rc = caser_check_targets(seq_T, neg_samples);
    if (rc) return rc;
    rc = caser_check_batch(batch);
    if (rc) return rc;
    NRC_REQUIRE(num_items >= 1, NRC_E_VALUE, "num_items >= 1 required");
    NRC_REQUIRE(!mask || (keep > 0.0f && keep <= 1.0f), NRC_E_VALUE, "keep in (0, 1] required with a mask");
    NRC_REQUIRE(user_table && seq_table && item_table && item_bias && dense && users && seqs && pos && neg, NRC_E_VALUE,
                "tables, the dense block and the batch are required");
    NRC_REQUIRE(grad_user && grad_seq && grad_item && grad_bias && grad_dense && work, NRC_E_VALUE,
                "gradients and work (nrc_caser_work_floats floats) are required");
    if (batch == 0) return NRC_OK;
    cudaStream_t st = as_stream(stream);
    const CaserDims D = caser_dims(dim, seq_L, nv, nh, seq_T, neg_samples, num_items);
    unsigned* counters = reinterpret_cast<unsigned*>(work);
    float* fac = work + caser_counters(D);
    float* partial = fac + batch * caser_factor_floats(D);
    const bool staged = caser_staged(D);
    const size_t smem = caser_smem_bytes(D);
    NRC_CUDA_CHECK(cudaFuncSetAttribute(caser_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t cap = (int64_t)sm_count() * 2;
    const unsigned grid = (unsigned)(batch < cap ? batch : cap);
    caser_route(kCaGrad, staged ? 1 : 0, grid, -1, batch > cap ? 1 : 0, seq_L, mask ? 1 : 0);
    caser_grad_kernel<<<grid, 256, smem, st>>>(D, user_table, seq_table, item_table, item_bias, dense, staged, users,
                                               seqs, pos, neg, batch, mask, mask ? keep : 1.0f,
                                               1.0f / (float)(batch * seq_T), 1.0f / (float)(batch * neg_samples),
                                               grad_user, grad_seq, grad_item, grad_bias, fac, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    const dim3 wgrid((unsigned)caser_counters(D), (unsigned)caser_chunks(batch));
    caser_route(kCaWgrad, -1, wgrid.x, wgrid.y, -1, seq_L, -1);
    caser_wgrad_kernel<<<wgrid, 256, 0, st>>>(D, batch, fac, partial, counters, grad_dense);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_caser_train_epoch(float* user_table, float* seq_table, float* item_table, float* item_bias,
                                     float* dense, int32_t num_users, int32_t num_items, int32_t dim, int32_t seq_L,
                                     int32_t seq_T, int32_t nv, int32_t nh, int32_t neg_samples, const int32_t* users,
                                     const int32_t* seqs, const int32_t* pos, const int32_t* neg, int64_t n,
                                     int32_t batch_size, float keep, float l2_reg, uint64_t seed, uint64_t epoch,
                                     const float* lr_t_host, const float* hyper_host, float* grad_user,
                                     float* grad_seq, float* grad_item, float* grad_bias, float* grad_dense,
                                     float* const* slot0, float* const* slot1, float* work, float* step_loss,
                                     void* stream) {
    int rc = caser_check_shape(dim, seq_L, nv, nh);
    if (rc) return rc;
    rc = caser_check_targets(seq_T, neg_samples);
    if (rc) return rc;
    NRC_REQUIRE(n >= 0, NRC_E_VALUE, "n >= 0 required");
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    rc = caser_check_batch(batch_size);
    if (rc) return rc;
    NRC_REQUIRE(num_users >= 1 && num_items >= 1, NRC_E_VALUE, "num_users and num_items >= 1 required");
    NRC_REQUIRE(keep > 0.0f && keep <= 1.0f, NRC_E_VALUE, "keep = 1 - dropout must lie in (0, 1]");
    NRC_REQUIRE(lr_t_host && hyper_host && slot0 && slot1 && work && step_loss, NRC_E_VALUE,
                "lr_t_host, hyper_host, slot0, slot1 (the five variables' Adam slots), work and step_loss are required");
    NRC_REQUIRE(user_table && seq_table && item_table && item_bias && dense && grad_user && grad_seq && grad_item &&
                grad_bias && grad_dense, NRC_E_VALUE, "variables and gradients are required");
    cudaStream_t st = as_stream(stream);
    const CaserDims D = caser_dims(dim, seq_L, nv, nh, seq_T, neg_samples, num_items);
    float* mask = work + caser_counters(D) + (int64_t)batch_size * caser_factor_floats(D) +
                  caser_chunks(batch_size) * D.Dn;
    CaserRegSegs R;
    R.var[0] = user_table; R.grad[0] = grad_user; R.n[0] = (int64_t)num_users * dim;
    R.var[1] = seq_table; R.grad[1] = grad_seq; R.n[1] = (int64_t)num_items * dim;
    R.var[2] = item_table; R.grad[2] = grad_item; R.n[2] = (int64_t)num_items * 2 * dim;
    R.var[3] = item_bias; R.grad[3] = grad_bias; R.n[3] = num_items;
    const int64_t total = R.n[0] + R.n[1] + R.n[2] + R.n[3];
    int64_t step = 0;
    return seq_epoch_loop(
        n, batch_size, NRC_OPT_ADAM, lr_t_host, hyper_host, 0, step_loss, st,
        [&](int64_t off, int64_t bs, int32_t, float* loss) {
            // the step's dropout mask: nrc_dropout_mask keyed by (seed, epoch << 32 | step)
            int r = nrc_dropout_mask(bs * D.F, keep, seed, (epoch << 32) | (uint64_t)step++, mask, stream);
            if (r) return r;
            const unsigned grid = elementwise_grid(total);
            caser_route(kCaReg, -1, grid, -1, elementwise_capped(total), -1, -1);
            caser_reg_kernel<<<grid, 256, 0, st>>>(R, total, l2_reg);
            NRC_CUDA_CHECK(cudaGetLastError());
            return nrc_caser_grad(user_table, seq_table, item_table, item_bias, dense, num_items, dim, seq_L, seq_T,
                                  nv, nh, neg_samples, users + off, seqs + off * seq_L, pos + off * seq_T,
                                  neg + off * neg_samples, bs, mask, keep, grad_user, grad_seq, grad_item, grad_bias,
                                  grad_dense, work, loss, stream);
        },
        [&](OptLaunch& L) {
            // the tables: IndexedSlices gradients on every row (Adam's sparse form); the dense block: ApplyAdam
            opt_launch_add(L, user_table, grad_user, slot0[0], slot1[0], nullptr, num_users, dim, 0);
            opt_launch_add(L, seq_table, grad_seq, slot0[1], slot1[1], nullptr, num_items, dim, 0);
            opt_launch_add(L, item_table, grad_item, slot0[2], slot1[2], nullptr, num_items, 2 * dim, 0);
            opt_launch_add(L, item_bias, grad_bias, slot0[3], slot1[3], nullptr, num_items, 1, 0);
            opt_launch_add(L, dense, grad_dense, slot0[4], slot1[4], nullptr, D.Dn, 1, 1);
        });
}

extern "C" int nrc_caser_query(const float* user_table, const float* seq_table, const float* dense, int32_t num_items,
                               int32_t dim, int32_t seq_L, int32_t nv, int32_t nh, const int32_t* users, int64_t rows,
                               const int32_t* windows, float* out, void* stream) {
    const int rc = caser_check_shape(dim, seq_L, nv, nh);
    if (rc) return rc;
    NRC_REQUIRE(num_items >= 1 && rows >= 0, NRC_E_VALUE, "num_items >= 1 and rows >= 0 required");
    NRC_REQUIRE(rows == 0 || (user_table && seq_table && dense && users && windows && out), NRC_E_VALUE,
                "tables, the dense block, users, windows and out are required");
    if (rows == 0) return NRC_OK;
    const CaserDims D = caser_dims(dim, seq_L, nv, nh, 1, 1, num_items);
    const bool staged = caser_staged(D);
    const size_t smem = caser_smem_bytes(D);
    NRC_CUDA_CHECK(cudaFuncSetAttribute(caser_query_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t cap = (int64_t)sm_count() * 2;
    const unsigned grid = (unsigned)(rows < cap ? rows : cap);
    caser_route(kCaQuery, staged ? 1 : 0, grid, -1, rows > cap ? 1 : 0, seq_L, 0);
    caser_query_kernel<<<grid, 256, smem, as_stream(stream)>>>(D, user_table, seq_table, dense, staged, users, rows,
                                                               windows, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// Host bookkeeping of the routes the most recent Caser launches took (see the header); no device work.
extern "C" int nrc_caser_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "out is NULL");
    for (int k = 0; k < kCaKernels; ++k)
        for (int f = 0; f < kCaFields; ++f) out[k * kCaFields + f] = g_caser_routes.r[k][f];
    return NRC_OK;
}
