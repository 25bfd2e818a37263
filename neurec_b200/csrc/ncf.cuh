// Shapes shared by the NCF kernels (ncf.cu, ncf_epoch.cu).
#pragma once
#include "common.cuh"

namespace nrc {

constexpr int kNcfMaxLayers = 4;
constexpr int kNcfThreads = 128;   // threads per sample CTA
constexpr int kNcfWarps = 8;       // warps per CTA of the score kernel
constexpr int kWgradSlices = 16;   // batch slices of the weight-gradient kernel

struct NcfDev {
    int mf_dim, mlp_dim, n_layers, n_towers;
    int in_dim[kNcfMaxLayers], out_dim[kNcfMaxLayers];
    int w_off[kNcfMaxLayers], b_off[kNcfMaxLayers];      // offsets in the packed dense buffer
    int sw_off[kNcfMaxLayers], sb_off[kNcfMaxLayers];    // offsets in the padded smem copy (scores)
    int a_off[kNcfMaxLayers + 1];                        // activation offsets (a_0 = input)
    int tower_size, s_tower_size, act_size;
};

struct NcfPtrs {
    const float* mf_user; const float* mf_item; const float* mlp_user; const float* mlp_item;
    const float* dense;
    float* g_mf_user; float* g_mf_item; float* g_mlp_user; float* g_mlp_item; float* g_dense;
    int32_t* t_user; int32_t* t_item;
};

int ncf_make(NcfDev& S, const nrc_ncf_shape* sh);

// Layer forms of the epoch kernel's tower (ncf_epoch.cu fwd_layer / bwd_layer), one copy for the kernel and
// for the route hook.  Forward split: the k-range of a layer is divided over kNcfThreads / out thread groups.
// Backward split: kNcfThreads / in threads (at most a warp) share each input row k.  Macros, not functions:
// with the same condition behind a __host__ __device__ function nvcc 12.9 compiled a different, larger
// ncf_epoch_kernel; the macros leave its SASS as it was with the conditions written inline.
#define NCF_FWD_SPLIT(in, out) ((out) <= kNcfThreads && kNcfThreads % (out) == 0 && (in) % (kNcfThreads / (out)) == 0)
#define NCF_BWD_SPLIT(in, out) \
    ((in) <= kNcfThreads && kNcfThreads % (in) == 0 && (kNcfThreads / (in)) <= 32 && (out) % (kNcfThreads / (in)) == 0)

// Routes of the most recent NCF launch (nrc_ncf_last_routes); -1 = not decided by that call.
enum NcfRoute { kRouteSampleFast, kRouteWgradSlices, kRouteEpochDwBlocked, kRouteEpochTablesVec4, kRouteFwdSplit,
                kRouteBwdSplit, kRouteScoresTile, kNcfRoutes };
extern int32_t g_ncf_routes[kNcfRoutes];
void ncf_routes_reset();

}  // namespace nrc
