// The reference's losses, value and derivative: util/learner.py:21-38 (and util/tool.py:224), defined once for
// every training kernel.
#pragma once
#include "common.cuh"

namespace nrc {

// softplus(-x) = -log_sigmoid(x)  (learner.py:22, tool.py:224)
__device__ __forceinline__ float neg_log_sigmoid(float x) {
    return (x >= 0.0f) ? log1pf(expf(-x)) : (-x + log1pf(expf(x)));
}

// d/dx of neg_log_sigmoid(x) = -sigmoid(-x)
__device__ __forceinline__ float neg_log_sigmoid_grad(float x) { return -1.0f / (1.0f + expf(x)); }

// loss l(x) and dl/dx of one pair; x = score(positive) - score(negative)
__device__ __forceinline__ void pairwise_loss_grad(int kind, float x, float& l, float& g) {
    if (kind == NRC_LOSS_BPR) {           // learner.py:21-22  -sum(log_sigmoid(y))
        l = neg_log_sigmoid(x);
        g = neg_log_sigmoid_grad(x);
    } else if (kind == NRC_LOSS_HINGE) {  // learner.py:23-24  sum(max(y + margin, 0)) [sic]
        const float t = x + 1.0f;
        l = fmaxf(t, 0.0f);
        g = (t > 0.0f) ? 1.0f : 0.0f;
    } else {                              // learner.py:25-26  sum((1 - y)^2)
        const float t = 1.0f - x;
        l = t * t;
        g = -2.0f * t;
    }
}

// loss l(x) and dl/dx of one sample; x = score, z = label, inv_b = 1 / batch size
__device__ __forceinline__ void pointwise_loss_grad(int kind, float x, float z, float inv_b, float& l, float& g) {
    if (kind == NRC_LOSS_CROSS_ENTROPY) {
        // learner.py:33-34 tf.losses.sigmoid_cross_entropy: mean_b of max(x,0) - x*z + log1p(exp(-|x|))
        const float e = expf(-fabsf(x));
        l = (fmaxf(x, 0.0f) - x * z + log1pf(e)) * inv_b;
        const float s = (x >= 0.0f) ? 1.0f / (1.0f + e) : e / (1.0f + e);
        g = (s - z) * inv_b;
    } else {                              // learner.py:37-38  sum((y_rea - y_pre)^2)
        const float t = z - x;
        l = t * t;
        g = -2.0f * t;
    }
}

}  // namespace nrc
