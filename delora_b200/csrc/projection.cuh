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

// A coordinate of a scaled projection: v / f correctly rounded (torch's tensor-by-tensor division), the value itself
// when the projection is not scaled or the channel is not a coordinate.
template <bool kScaled>
__device__ __forceinline__ float scaled(float v, float f, bool coordinate = true) {
    return (kScaled && coordinate) ? __fdiv_rn(v, f) : v;
}

// Enqueue project_scatter_kernel: one 64-bit atomicMin of (range_bits << 32 | point_index) per in-FOV point into
// `keys` ([B, H*W], all-ones on entry).  The kernel lets its programmatic dependent launch as soon as all of its CTAs
// have started.  Check the launch with DELORA_CHECK_LAUNCH.  factor [fB] or NULL: scan b's coordinates are divided by
// factor[b % fB] first (a separate instantiation; NULL runs the unscaled kernel).
void launch_project_scatter(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                            const GridParams& g, unsigned long long* keys, cudaStream_t st,
                            const float* factor = nullptr, int fB = 0);

// delora_normalization_factors' kernel on points [2B, 3, n_stride], counts [2B] (clamped to [0, n_stride] on the device)
// -> factor [B].  Arguments are not checked.
int launch_normalization_factors(const float* points, const int32_t* n_points, int B, int n_stride, float* factor,
                                 cudaStream_t st);

// The same factor of B pairs from the valid cells of the dense grids [2B, n_cells] float4 (delora_normals_fwd's layout:
// w = pixel-id bits >= 0 for a valid cell), the points the reference's preprocessing stored.  Arguments are not checked.
int launch_grid_normalization_factors(const delora_f4* grid, int B, int n_cells, float* factor, cudaStream_t st);

// delora_project_grids_fwd's two passes (g: the model's H x W grid), optionally with scan s's cell coordinates divided
// by factor[s % fB] (factor NULL: the unscaled kernels).  Arguments are not checked.
int project_grids_fwd(const delora_f4* pts_grid_pre, const delora_f4* nrm_grid_pre, int S, int Wp, const GridParams& g,
                      uint64_t* keys, float* image, int32_t* index_map, delora_f4* pts_grid, delora_f4* nrm_grid,
                      const float* factor, int fB, cudaStream_t st);

// delora_project_fwd's scatter and resolve passes, optionally scaled as above.  Arguments are not checked.
int project_fwd(const float* points, const int32_t* n_points, int B, int C, int n_stride, const GridParams& g,
                uint64_t* keys, float* image, int32_t* index_map, const float* factor, int fB, cudaStream_t st);

}  // namespace delora
