// TensorFlow-1.12 optimizer update rules (util/learner.py:2-15 selects them).
//
// Third-party arithmetic (tensorflow==1.12.3, python/training/*.py + core/kernels/training_ops.cc;
// not vendored in the reference, restated from its published algorithm -- see DESIGN.md):
//
//  IndexedSlices gradients (embedding rows; `dense_var == 0`), g = de-duplicated row gradient
//    gd        var -= g * lr                                     (touched rows; g = 0 elsewhere)
//    adam      m = m*b1 + g*(1-b1); v = v*b2 + (g*g)*(1-b2);     EVERY row: _apply_sparse_shared
//              var -= (lr_t * m) / (sqrt(v) + eps)               assigns m*b1, v*b2 densely
//    adagrad   a += g*g; var -= (lr * g) * (1/sqrt(a))           touched rows only
//    rmsprop   ms = ms*rho + (g*g)*(1-rho); mom = mom*mu + ((1/sqrt(ms+eps))*lr)*g; var -= mom   (SparseApplyRMSProp)
//    momentum  a = a*mu + g; var -= a*lr                         touched rows only
//  Dense gradients (`dense_var == 1`): the Apply* functors
//    adam      m += (g - m)*(1-b1); v += (g*g - v)*(1-b2); var -= (m*lr_t) / (sqrt(v) + eps)
//    rmsprop   ms += (g*g - ms)*(1-rho); mom = mom*mu + (lr*g)*(1/sqrt(ms+eps)); var -= mom     (ApplyRMSProp)
//    others    same formulas as above applied to every element.
//
// Every fp32 operation is written with a non-contracting intrinsic so the result is the
// same sequence of IEEE roundings numpy produces in oracle/tf_math.py (bit-exact given the
// same gradient).
#include "optim.cuh"

#include "mf_routes.cuh"

namespace nrc {

struct OptParams {
    OptSeg seg[kMaxOptSegs];
    int nseg;
    int kind;
    float h0, h1, h2, h3;
    const float* h0_src;   // optional device-resident lr / lr_t (captured step graphs)
    int32_t stamp;
    int64_t total;
};

__global__ void __launch_bounds__(256) opt_apply_kernel(const OptParams P) {
    const bool has0 = P.kind != NRC_OPT_GD;
    const bool has1 = P.kind == NRC_OPT_ADAM || P.kind == NRC_OPT_RMSPROP;
    const float h0 = P.h0_src ? __ldg(P.h0_src) : P.h0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < P.total;
         e += (int64_t)gridDim.x * blockDim.x) {
        int s = 0;
#pragma unroll 1
        while (s + 1 < P.nseg && e >= P.seg[s + 1].begin) ++s;
        const OptSeg& sg = P.seg[s];
        const int64_t i = e - sg.begin;
        const float g = sg.grad[i];
        bool touched = true;
        if (!sg.dense_var && sg.touched) touched = (sg.touched[i / sg.dim] == P.stamp);
        float var = sg.var[i];
        float s0 = has0 ? sg.s0[i] : 0.0f;
        float s1 = has1 ? sg.s1[i] : 0.0f;
        opt_update(P.kind, sg.dense_var, touched, h0, P.h1, P.h2, P.h3, var, g, s0, s1);
        sg.var[i] = var;
        if (has0) sg.s0[i] = s0;
        if (has1) sg.s1[i] = s1;
        sg.grad[i] = 0.0f;
    }
}

static thread_local const float* g_lr_src = nullptr;

int opt_launch_init(OptLaunch& L, int opt_kind, const float* hyper_host) {
    // learner.py:14-15 raises ValueError("please select a suitable optimizer")
    NRC_REQUIRE(opt_kind >= NRC_OPT_GD && opt_kind <= NRC_OPT_MOMENTUM, NRC_E_VALUE,
                "please select a suitable optimizer");
    L.nseg = 0;
    L.kind = opt_kind;
    L.total = 0;
    for (int i = 0; i < 4; ++i) L.h[i] = hyper_host ? hyper_host[i] : 0.0f;
    return NRC_OK;
}

int opt_launch_add(OptLaunch& L, float* var, float* grad, float* s0, float* s1,
                   const int32_t* touched, int64_t rows, int dim, int dense_var) {
    NRC_REQUIRE(L.nseg < kMaxOptSegs, NRC_E_LIMIT, "too many optimizer segments");
    NRC_REQUIRE(rows >= 0 && dim > 0, NRC_E_VALUE, "bad table shape");
    OptSeg& s = L.seg[L.nseg++];
    s.var = var; s.grad = grad; s.s0 = s0; s.s1 = s1; s.touched = touched;
    s.elems = rows * dim; s.begin = L.total; s.dim = dim; s.dense_var = dense_var;
    L.total += s.elems;
    return NRC_OK;
}

int opt_launch_run(const OptLaunch& L, int32_t stamp, cudaStream_t st) {
    if (L.total == 0) return NRC_OK;
    OptParams P;
    for (int i = 0; i < L.nseg; ++i) P.seg[i] = L.seg[i];
    P.nseg = L.nseg; P.kind = L.kind;
    P.h0 = L.h[0]; P.h1 = L.h[1]; P.h2 = L.h[2]; P.h3 = L.h[3];
    P.h0_src = g_lr_src;
    P.stamp = stamp; P.total = L.total;
    int64_t blocks = (L.total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    const bool capped = blocks > cap;
    if (blocks > cap) blocks = cap;
    mf_route(kMfOptApply, -1, -1, -1, -1, blocks, capped, -1);
    opt_apply_kernel<<<(unsigned)blocks, 256, 0, st>>>(P);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

}  // namespace nrc

// While a non-NULL source is set, every optimizer launch of this thread reads hyper[0] (lr, or
// Adam's lr_t) from that device float instead of the by-value argument -- what lets a captured
// CUDA graph of a training step be replayed with a different lr_t each step.
extern "C" int nrc_opt_set_lr_source(const float* lr_dev) {
    nrc::g_lr_src = lr_dev;
    return NRC_OK;
}
