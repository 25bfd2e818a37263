// MF's loss and gradient of one triplet / sample (model/general_recommender/MF.py:62-72), by one warp: shared by
// the per-step gradient kernel (train_mf.cu) and the persistent epoch kernel (epoch.cu).
#pragma once
#include "common.cuh"
#include "learner.cuh"

namespace nrc {

// Returns the sample's loss (including reg * l2_loss of its rows); adds the row gradients into the dense
// accumulators gU / gV with RED.ADD (duplicates sum) and stamps the rows.  t is the negative item (PAIRWISE) or the
// label's bits.  VEC > 0: D == 32 * VEC, the lane keeps its slice of the rows in registers; VEC == 0: any D,
// strided loop.  CG: table loads through L2 only (ld_vec).
template <bool PAIRWISE, int VEC, bool CG>
__device__ __forceinline__ float mf_sample_grad(const float* __restrict__ U, const float* __restrict__ V,
                                                float* __restrict__ gU, float* __restrict__ gV,
                                                int32_t* __restrict__ tU, int32_t* __restrict__ tV, int D, float reg,
                                                int loss_kind, int lane, int32_t u, int32_t i, int32_t t, float inv_b,
                                                int32_t stamp) {
    const float* pu = U + (size_t)u * D;
    const float* qi = V + (size_t)i * D;
    const float* qj = PAIRWISE ? V + (size_t)t * D : nullptr;
    float* gu = gU + (size_t)u * D;
    float* gi = gV + (size_t)i * D;
    float* gj = PAIRWISE ? gV + (size_t)t * D : nullptr;
    float l, g;
    if constexpr (VEC > 0) {
        const int k0 = lane * VEC;
        float a[VEC], bi[VEC], bj[VEC];
        ld_vec<VEC, CG>(pu + k0, a);
        ld_vec<VEC, CG>(qi + k0, bi);
        if constexpr (PAIRWISE) ld_vec<VEC, CG>(qj + k0, bj);
        float di = 0.0f, dj = 0.0f, sq = 0.0f;
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
            di = fmaf(a[c], bi[c], di);
            if constexpr (PAIRWISE) { dj = fmaf(a[c], bj[c], dj); sq += a[c] * a[c] + bi[c] * bi[c] + bj[c] * bj[c]; }
            else sq += a[c] * a[c] + bi[c] * bi[c];
        }
        di = warp_sum(di);
        if constexpr (PAIRWISE) pairwise_loss_grad(loss_kind, di - warp_sum(dj), l, g);   // MF.py:66
        else pointwise_loss_grad(loss_kind, di, __int_as_float(t), inv_b, l, g);
        if (reg != 0.0f) l += reg * 0.5f * warp_sum(sq);                                 // MF.py:67,72
        float du[VEC], dvi[VEC], dvj[VEC];
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
            if constexpr (PAIRWISE) {
                du[c] = g * (bi[c] - bj[c]) + reg * a[c];
                dvi[c] = g * a[c] + reg * bi[c];
                dvj[c] = -g * a[c] + reg * bj[c];
            } else {
                du[c] = g * bi[c] + reg * a[c];
                dvi[c] = g * a[c] + reg * bi[c];
            }
        }
        red_vec<VEC>(gu + k0, du);
        red_vec<VEC>(gi + k0, dvi);
        if constexpr (PAIRWISE) red_vec<VEC>(gj + k0, dvj);
    } else {
        float di = 0.0f, dj = 0.0f, sq = 0.0f;
        for (int k = lane; k < D; k += kWarp) {
            const float a = ld<CG>(pu + k), bi = ld<CG>(qi + k);
            di = fmaf(a, bi, di);
            if constexpr (PAIRWISE) {
                const float bj = ld<CG>(qj + k);
                dj = fmaf(a, bj, dj);
                sq += a * a + bi * bi + bj * bj;
            } else sq += a * a + bi * bi;
        }
        di = warp_sum(di);
        if constexpr (PAIRWISE) pairwise_loss_grad(loss_kind, di - warp_sum(dj), l, g);
        else pointwise_loss_grad(loss_kind, di, __int_as_float(t), inv_b, l, g);
        if (reg != 0.0f) l += reg * 0.5f * warp_sum(sq);
        for (int k = lane; k < D; k += kWarp) {
            const float a = ld<CG>(pu + k), bi = ld<CG>(qi + k);
            if constexpr (PAIRWISE) {
                const float bj = ld<CG>(qj + k);
                atomicAdd(gu + k, g * (bi - bj) + reg * a);
                atomicAdd(gi + k, g * a + reg * bi);
                atomicAdd(gj + k, -g * a + reg * bj);
            } else {
                atomicAdd(gu + k, g * bi + reg * a);
                atomicAdd(gi + k, g * a + reg * bi);
            }
        }
    }
    if (lane == 0) {
        tU[u] = stamp;
        tV[i] = stamp;
        if constexpr (PAIRWISE) tV[t] = stamp;
    }
    return l;
}

}  // namespace nrc
