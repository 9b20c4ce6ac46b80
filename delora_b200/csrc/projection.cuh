// Projection pieces shared by projection.cu and the fused projection + normals path in normals.cu (sm_90a).
#pragma once
#include "common.cuh"

namespace delora {

// Depth key of an empty pixel: every key buffer is all-ones between calls.
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

// Enqueue project_scatter_kernel: one 64-bit atomicMin of (range_bits << 32 | point_index) per in-FOV point into
// `keys` ([B, H*W], all-ones on entry).  The kernel lets its programmatic dependent launch as soon as all of its CTAs
// have started.  Check the launch with DELORA_CHECK_LAUNCH.
void launch_project_scatter(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                            const GridParams& g, unsigned long long* keys, cudaStream_t st);

}  // namespace delora
