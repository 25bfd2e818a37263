// Route bookkeeping of the MF training kernels (train_mf.cu, epoch.cu, optim.cu) for nrc_mf_last_routes.
#pragma once
#include <stdint.h>

namespace nrc {

// Host record of what the most recent launch of each kernel group decided (see the header); -1 = no such launch yet,
// or a field the group does not decide.  Written just before the launch, so a call that fails its checks leaves it as
// it was.
enum MfKernel { kMfGrad, kMfSgdIds, kMfSgdCsr, kMfLazyAdam, kMfEpoch, kMfOptApply, kMfKernels };
enum MfRouteField { kMfVec, kMfSharded, kMfUserOnce, kMfTierRows, kMfGrid, kMfCapped, kMfOptVec4, kMfFields };
extern int32_t g_mf_routes[kMfKernels][kMfFields];

inline void mf_route(int kernel, int vec, int sharded, int user_once, int tier_rows, int64_t grid, bool capped,
                     int opt_vec4) {
    int32_t* r = g_mf_routes[kernel];
    r[kMfVec] = vec; r[kMfSharded] = sharded; r[kMfUserOnce] = user_once; r[kMfTierRows] = tier_rows;
    r[kMfGrid] = (int32_t)grid; r[kMfCapped] = capped ? 1 : 0; r[kMfOptVec4] = opt_vec4;
}

}  // namespace nrc
