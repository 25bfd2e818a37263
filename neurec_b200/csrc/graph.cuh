// Route bookkeeping of the graph kernels (lightgcn.cu, ngcf.cu, spectral.cu) for nrc_graph_last_routes.
#pragma once
#include <stdint.h>

namespace nrc {

// Host record of what the most recent graph calls decided (see the header); -1 = not decided by the call that last
// wrote the group.  Written just before a call launches, so a call that fails its checks leaves it as it was.
enum GraphRoute { kRouteSpmmFast, kRouteSpmmWidth, kRouteSpmmCapped, kRouteNgcfFwdRows, kRouteNgcfBwdTiles,
                  kRouteNgcfBprTriplets, kRouteSpecFwdSplit, kRouteSpecBwdSplit, kRouteSpecDwSplit, kGraphRoutes };
extern int32_t g_graph_routes[kGraphRoutes];

}  // namespace nrc
