// What the sequential models' fused epoch calls share (sequential.cu, caser.cu): the batch loop of every
// *_train_epoch and the grid of their elementwise passes.
#pragma once
#include "common.cuh"
#include "optim.cuh"

namespace nrc {

// The batch loop of every *_train_epoch: batch s covers samples [s * batch_size, min(n, (s + 1) * batch_size)) and
// gets stamp first_stamp + s.  grad(off, bs, stamp, loss) runs the model's gradient call for it; add(L) lists the
// model's variables in the optimizer launch that follows (one launch per batch).
template <class Grad, class Add>
static int seq_epoch_loop(int64_t n, int32_t batch_size, int32_t opt_kind, const float* lr_t_host,
                          const float* hyper_host, int32_t first_stamp, float* step_loss, cudaStream_t st, Grad grad,
                          Add add) {
    const int64_t steps = (n + batch_size - 1) / batch_size;
    if (steps == 0) return NRC_OK;
    NRC_CUDA_CHECK(cudaMemsetAsync(step_loss, 0, (size_t)steps * sizeof(float), st));
    float hyper[4] = {hyper_host[0], hyper_host[1], hyper_host[2], hyper_host[3]};
    for (int64_t s = 0; s < steps; ++s) {
        const int64_t off = s * batch_size;
        const int64_t bs = (n - off < batch_size) ? (n - off) : batch_size;
        const int32_t stamp = first_stamp + (int32_t)s;
        int rc = grad(off, bs, stamp, step_loss + s);
        if (rc) return rc;
        if (opt_kind == NRC_OPT_ADAM) hyper[0] = lr_t_host[s];
        OptLaunch L;
        rc = opt_launch_init(L, opt_kind, hyper);
        if (rc) return rc;
        add(L);
        rc = opt_launch_run(L, stamp, st);
        if (rc) return rc;
    }
    return NRC_OK;
}

// Grid of an elementwise pass: one 256-thread CTA per 256 elements, at most 16 per SM.
static unsigned elementwise_grid(int64_t total) {
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    return (unsigned)(blocks < 1 ? 1 : blocks);
}

// 1 when elementwise_grid capped the grid, so a thread takes more than one element
static int elementwise_capped(int64_t total) { return (total + 255) / 256 > (int64_t)sm_count() * 16 ? 1 : 0; }

}  // namespace nrc
