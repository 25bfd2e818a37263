// Route bookkeeping of the data-side kernels (extras.cu), the negative samplers (sampler.cu) and LightGCN's BPR
// gradient (lightgcn.cu) for nrc_extras_last_routes (see the header).
#pragma once
#include <stdint.h>

namespace nrc {

enum ExtrasKernel { kExL2Normalize, kExGatherRows, kExSbprEpochBuild, kExSbprGrad, kExCsrFromCoo, kExSplit, kExCsrRowIds,
                    kExSampleNegatives, kExBatchChoice, kExLightgcnGrad, kExKernels };
enum ExtrasField { kExGrid, kExCapped, kExRowGrid, kExRowCapped, kExScanChunks, kExReplace, kExFields };

// Written just before a launch, so a call that fails its checks or launches nothing leaves the record as it was.
// -1 = a field the group does not decide.
void extras_route(int kernel, int64_t grid, int capped, int64_t row_grid = -1, int row_capped = -1,
                  int64_t scan_chunks = -1, int replace = -1);

}  // namespace nrc
