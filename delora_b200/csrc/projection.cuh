// Projection pieces shared by projection.cu and the fused projection + normals path in normals.cu (sm_90a).  Every
// scatter (of raw points, and of grid cells in delora_project_grids_fwd) computes its pixel and key with
// project_pixel and depth_key, so the two cannot drift apart.
#pragma once
#include "common.cuh"

namespace delora {

// Depth key of an empty pixel: every key buffer is all-ones between calls.
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

// The pixel id v * W + u a point projects to: (u, v) rounded half to even (torch.round) and the field-of-view test of
// src/utility/projection.py:74-77.  -1 outside the image, NaN coordinates included.
__device__ __forceinline__ int project_pixel(const GridParams& g, float x, float y, float z) {
    float u, v;
    pixel_coords(g, x, y, z, u, v);
    const float ru = rintf(u), rv = rintf(v);
    const bool inside = (ru <= g.wm1) && (ru >= 0.0f) && (rv <= g.hm1) && (rv >= 0.0f);
    return inside ? (int)rv * g.W + (int)ru : -1;
}

// The depth key of a point: its range bits over a tie-break id.  A range is never negative, so the key order is the
// (range, id) order, and one 64-bit atomicMin per point leaves the closest point in a pixel, the lowest id among
// equal ranges.
__device__ __forceinline__ unsigned long long depth_key(float x, float y, float z, unsigned id) {
    return ((unsigned long long)__float_as_uint(range3(x, y, z)) << 32) | id;
}

// Enqueue project_scatter_kernel: one 64-bit atomicMin of (range_bits << 32 | point_index) per in-FOV point into
// `keys` ([B, H*W], all-ones on entry).  The kernel lets its programmatic dependent launch as soon as all of its CTAs
// have started.  Check the launch with DELORA_CHECK_LAUNCH.
void launch_project_scatter(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                            const GridParams& g, unsigned long long* keys, cudaStream_t st);

}  // namespace delora
