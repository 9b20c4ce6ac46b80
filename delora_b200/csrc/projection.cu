// Spherical projection of raw LiDAR scans to H x W range images (sm_90a).
//
// Replaces utility.projection.ImageProjectionLayer.project_to_img
// (reference: src/utility/projection.py:48-106).  The reference sorts the cloud by range
// (:63), walks it serially keeping the first point that lands in each pixel (:34-43, numba on
// the CPU) and scatters the survivors (:98-103).  "First in range order" == "minimum range",
// so here every point does one 64-bit atomicMin of (range_bits << 32 | point_index) on its
// pixel (equal ranges: lowest index wins == a stable sort); a second pass resolves the winners
// into the image and the pixel -> point index map and re-arms the key buffer.  delora_project_normals_fwd
// (normals.cu) runs the same scatter and resolves the keys inside its 7x11 normals kernel instead.
// delora_project_grids_fwd re-projects the dense grids of such a projection at another width with the same per-point
// arithmetic (project_pixel, depth_key in projection.cuh) and the same two passes.
//
// HBM/L2 traffic per scan: read 12 N (xyz) [+ 8 HW key RMW in L2] ; write 4 (C+1) HW + 4 HW.
#include <cooperative_groups.h>

#include "projection.cuh"

namespace delora {

constexpr int kScatterThreads = 256;
constexpr int kScatterPPT = 4;       // points per thread (independent loads in flight)

// kScaled: scan b's coordinates are divided by factor[b % fB] (delora_odometry_pairs_normalized) before any other use,
// so the keys are those of a pre-divided copy of the points; without it the factor arguments are not read.
template <bool kScaled>
__global__ void __launch_bounds__(kScatterThreads)
project_scatter_kernel(const float* __restrict__ points, const int32_t* __restrict__ n_points,
                       int C, int n_stride, GridParams g, unsigned long long* __restrict__ keys,
                       const float* __restrict__ factor, int fB) {
    // A programmatic dependent (project_normals_7x11_kernel) may start its key-independent prologue on SMs this grid
    // frees; it waits for this whole grid before it reads a key.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int b = blockIdx.y;
    const int n = n_points[b];
    const int base = blockIdx.x * (kScatterThreads * kScatterPPT) + threadIdx.x;
    if (blockIdx.x * (kScatterThreads * kScatterPPT) >= n) return;   // whole block past the end
    const float* __restrict__ px = points + (size_t)b * C * n_stride;
    const float* __restrict__ py = px + n_stride;
    const float* __restrict__ pz = py + n_stride;
    unsigned long long* __restrict__ kb = keys + (size_t)b * g.H * g.W;

    const float f = kScaled ? __ldg(factor + b % fB) : 1.0f;
    float x[kScatterPPT], y[kScatterPPT], z[kScatterPPT];
#pragma unroll
    for (int i = 0; i < kScatterPPT; ++i) {
        const int idx = base + i * kScatterThreads;
        const bool ok = idx < n;
        x[i] = ok ? scaled<kScaled>(__ldg(px + idx), f) : 0.0f;
        y[i] = ok ? scaled<kScaled>(__ldg(py + idx), f) : 0.0f;
        z[i] = ok ? scaled<kScaled>(__ldg(pz + idx), f) : 0.0f;
    }
#pragma unroll
    for (int i = 0; i < kScatterPPT; ++i) {
        const int idx = base + i * kScatterThreads;
        const int pix = project_pixel(g, x[i], y[i], z[i]);
        if (idx < n && pix >= 0) {
            // One 64-bit atomicMin (a fire-and-forget RED at L2) per in-FOV point.  A match.any /
            // redux.min warp aggregation does not pay here: redux with per-group masks serialises
            // once per distinct pixel (~28 groups per warp at W = 2048), while 2 M atomics per step
            // are far below the L2 atomic rate.
            atomicMin(kb + pix, depth_key(x[i], y[i], z[i], (unsigned)idx));
        }
    }
}

// One thread resolves 4 consecutive pixels: 2 x 16-byte key loads, float4 stores per channel.
// CT = compile-time channel count (3: xyz, 4: xyz + reflectance) so that all 4 x CT gathers are issued before
// the first store (the kernel is latency-bound on them); CT = 0: generic loop.  kScaled: x, y, z are divided by the
// scan's factor as in project_scatter_kernel<true> (further channels are not coordinates and are copied).
template <int CT, bool kScaled>
__global__ void __launch_bounds__(256)
project_resolve_kernel(const float* __restrict__ points, int C, int n_stride, int HW,
                       unsigned long long* __restrict__ keys, float* __restrict__ image,
                       int32_t* __restrict__ index_map, const float* __restrict__ factor, int fB) {
    const int b = blockIdx.y;
    const float f = kScaled ? __ldg(factor + b % fB) : 1.0f;
    const int p0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    if (p0 >= HW) return;
    const float* __restrict__ pb = points + (size_t)b * C * n_stride;
    unsigned long long* __restrict__ kb = keys + (size_t)b * HW;
    float* __restrict__ ib = image + (size_t)b * (C + 1) * HW;
    int32_t* __restrict__ mb = index_map + (size_t)b * HW;

    unsigned long long k[4];
    if (p0 + 3 < HW) {
        const ulonglong2 k01 = *reinterpret_cast<const ulonglong2*>(kb + p0);
        const ulonglong2 k23 = *reinterpret_cast<const ulonglong2*>(kb + p0 + 2);
        k[0] = k01.x; k[1] = k01.y; k[2] = k23.x; k[3] = k23.y;
        const ulonglong2 e = make_ulonglong2(kEmptyKey, kEmptyKey);
        *reinterpret_cast<ulonglong2*>(kb + p0) = e;          // re-arm for the next call
        *reinterpret_cast<ulonglong2*>(kb + p0 + 2) = e;
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            k[j] = (p0 + j < HW) ? kb[p0 + j] : kEmptyKey;
            if (p0 + j < HW) kb[p0 + j] = kEmptyKey;
        }
    }
    int idx[4];
    float rng[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const bool hit = k[j] != kEmptyKey;
        idx[j] = hit ? (int)(unsigned)(k[j] & 0xffffffffull) : -1;
        rng[j] = hit ? __uint_as_float((unsigned)(k[j] >> 32)) : 0.0f;
    }
    const bool vec = (p0 + 3 < HW) && ((HW & 3) == 0);
    if (CT > 0) {
        float val[CT > 0 ? CT : 1][4];
#pragma unroll
        for (int c = 0; c < CT; ++c)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                val[c][j] = idx[j] >= 0 ? scaled<kScaled>(__ldg(pb + (size_t)c * n_stride + idx[j]), f, c < 3) : 0.0f;
#pragma unroll
        for (int c = 0; c < CT; ++c) {
            if (vec) {
                *reinterpret_cast<float4*>(ib + (size_t)c * HW + p0) = make_float4(val[c][0], val[c][1], val[c][2], val[c][3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) if (p0 + j < HW) ib[(size_t)c * HW + p0 + j] = val[c][j];
            }
        }
    } else {
        for (int c = 0; c < C; ++c) {
            float val[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                val[j] = idx[j] >= 0 ? scaled<kScaled>(__ldg(pb + (size_t)c * n_stride + idx[j]), f, c < 3) : 0.0f;
            if (vec) {
                *reinterpret_cast<float4*>(ib + (size_t)c * HW + p0) = make_float4(val[0], val[1], val[2], val[3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) if (p0 + j < HW) ib[(size_t)c * HW + p0 + j] = val[j];
            }
        }
    }
    if (vec) {
        *reinterpret_cast<float4*>(ib + (size_t)C * HW + p0) = make_float4(rng[0], rng[1], rng[2], rng[3]);
        *reinterpret_cast<int4*>(mb + p0) = make_int4(idx[0], idx[1], idx[2], idx[3]);
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) if (p0 + j < HW) { ib[(size_t)C * HW + p0 + j] = rng[j]; mb[p0 + j] = idx[j]; }
    }
}

__global__ void __launch_bounds__(256)
project_uv_kernel(const float* __restrict__ points, const int32_t* __restrict__ n_points, int C,
                  int n_stride, GridParams g, float* __restrict__ u_out, float* __restrict__ v_out,
                  float* __restrict__ r_out) {
    const int b = blockIdx.y;
    const int idx = blockIdx.x * 256 + threadIdx.x;
    if (idx >= n_points[b]) return;
    const float* __restrict__ px = points + (size_t)b * C * n_stride;
    const float x = __ldg(px + idx), y = __ldg(px + n_stride + idx), z = __ldg(px + 2 * (size_t)n_stride + idx);
    float u, v;
    pixel_coords(g, x, y, z, u, v);
    u_out[(size_t)b * n_stride + idx] = u;
    v_out[(size_t)b * n_stride + idx] = v;
    if (r_out) r_out[(size_t)b * n_stride + idx] = range3(x, y, z);
}

void launch_project_scatter(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                            const GridParams& g, unsigned long long* keys, cudaStream_t st, const float* factor, int fB) {
    const int per_block = kScatterThreads * kScatterPPT;
    dim3 grid((n_stride + per_block - 1) / per_block, B);
    if (factor)
        project_scatter_kernel<true><<<grid, kScatterThreads, 0, st>>>(points, n_points, C, n_stride, g, keys, factor, fB);
    else
        project_scatter_kernel<false><<<grid, kScatterThreads, 0, st>>>(points, n_points, C, n_stride, g, keys, nullptr, 0);
}

int project_fwd(const float* points, const int32_t* n_points, int B, int C, int n_stride, const GridParams& g,
                uint64_t* keys, float* image, int32_t* index_map, const float* factor, int fB, cudaStream_t st) {
    launch_project_scatter(points, n_points, B, C, n_stride, g, (unsigned long long*)keys, st, factor, fB);
    DELORA_CHECK_LAUNCH("project_scatter_kernel");
    const int HW = g.H * g.W;
    dim3 grid2((HW + 1023) / 1024, B);
    unsigned long long* k = (unsigned long long*)keys;
    if (factor) {
        if (C == 3)
            project_resolve_kernel<3, true><<<grid2, 256, 0, st>>>(points, C, n_stride, HW, k, image, index_map, factor, fB);
        else if (C == 4)
            project_resolve_kernel<4, true><<<grid2, 256, 0, st>>>(points, C, n_stride, HW, k, image, index_map, factor, fB);
        else
            project_resolve_kernel<0, true><<<grid2, 256, 0, st>>>(points, C, n_stride, HW, k, image, index_map, factor, fB);
    } else {
        if (C == 3)
            project_resolve_kernel<3, false><<<grid2, 256, 0, st>>>(points, C, n_stride, HW, k, image, index_map, nullptr, 0);
        else if (C == 4)
            project_resolve_kernel<4, false><<<grid2, 256, 0, st>>>(points, C, n_stride, HW, k, image, index_map, nullptr, 0);
        else
            project_resolve_kernel<0, false><<<grid2, 256, 0, st>>>(points, C, n_stride, HW, k, image, index_map, nullptr, 0);
    }
    DELORA_CHECK_LAUNCH("project_resolve_kernel");
    return 0;
}

// ---- delora_project_grids_fwd: the dense grids of a projection at one width, re-projected at another.
// The preprocessing-resolution grids hold one point per pixel, and a valid cell's pixel id grows with its row-major
// position, which is the point's index in the list delora_lists_from_images would make of them.  So the cell id serves
// as the depth key's tie-break id, and the result is the list path's (lists -> delora_project_fwd ->
// delora_grids_from_projection) without building the list.
// Scatter: one atomicMin per valid cell, kScatterPPT independent 16-byte loads in flight per thread.
// kScaled: scan b's cell coordinates are divided by factor[b % fB] first (the training step of a normalised model:
// the stored points are divided, src/deploy/deployer.py:222-235, the normals are not).
template <bool kScaled>
__global__ void __launch_bounds__(kScatterThreads)
grids_scatter_kernel(const float4* __restrict__ pts_pre, int HWp, GridParams g, unsigned long long* __restrict__ keys,
                     const float* __restrict__ factor, int fB) {
    const int b = blockIdx.y;
    const float f = kScaled ? __ldg(factor + b % fB) : 1.0f;
    const int base = blockIdx.x * (kScatterThreads * kScatterPPT) + threadIdx.x;
    const float4* __restrict__ pb = pts_pre + (size_t)b * HWp;
    unsigned long long* __restrict__ kb = keys + (size_t)b * g.H * g.W;
    float4 p[kScatterPPT];
#pragma unroll
    for (int i = 0; i < kScatterPPT; ++i) {
        const int cell = base + i * kScatterThreads;
        p[i] = cell < HWp ? __ldg(pb + cell) : make_float4(0.0f, 0.0f, 0.0f, __int_as_float(-1));
        p[i].x = scaled<kScaled>(p[i].x, f); p[i].y = scaled<kScaled>(p[i].y, f); p[i].z = scaled<kScaled>(p[i].z, f);
    }
#pragma unroll
    for (int i = 0; i < kScatterPPT; ++i) {
        if (__float_as_int(p[i].w) < 0) continue;                          // empty cell: (+inf, +inf, +inf, -1)
        const int pix = project_pixel(g, p[i].x, p[i].y, p[i].z);
        if (pix >= 0) atomicMin(kb + pix, depth_key(p[i].x, p[i].y, p[i].z, (unsigned)(base + i * kScatterThreads)));
    }
}

// Resolve: one model pixel per thread.  The values and empty conventions of project_resolve_kernel<3> (image) and
// grids_from_projection_kernel (grids); the index map holds the preprocessing cell of the kept point.
template <bool kScaled>
__global__ void __launch_bounds__(256)
grids_resolve_kernel(const float4* __restrict__ pts_pre, const float4* __restrict__ nrm_pre, int HWp, int HW,
                     unsigned long long* __restrict__ keys, float* __restrict__ image, int32_t* __restrict__ index_map,
                     float4* __restrict__ pts_grid, float4* __restrict__ nrm_grid, const float* __restrict__ factor,
                     int fB) {
    const int b = blockIdx.y, pix = blockIdx.x * 256 + threadIdx.x;
    if (pix >= HW) return;
    const size_t o = (size_t)b * HW + pix;
    const unsigned long long k = keys[o];
    keys[o] = kEmptyKey;                                                   // re-arm for the next call
    const float inf = __int_as_float(0x7f800000);
    float4 c = make_float4(0.0f, 0.0f, 0.0f, 0.0f), q = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    float rng = 0.0f;
    int cell = -1;
    if (k != kEmptyKey) {
        cell = (int)(unsigned)(k & 0xffffffffull);
        c = __ldg(pts_pre + (size_t)b * HWp + cell);
        if (kScaled) {
            const float f = __ldg(factor + b % fB);
            c.x = scaled<kScaled>(c.x, f); c.y = scaled<kScaled>(c.y, f); c.z = scaled<kScaled>(c.z, f);
        }
        const float4 n = __ldg(nrm_pre + (size_t)b * HWp + cell);
        const bool has = (n.x != 0.0f) | (n.y != 0.0f) | (n.z != 0.0f);    // icp_losses.py:48-52
        q = make_float4(n.x, n.y, n.z, has ? 1.0f : 0.0f);
        rng = __uint_as_float((unsigned)(k >> 32));
    }
    float* __restrict__ ib = image + (size_t)b * 4 * HW;
    ib[pix] = c.x;
    ib[HW + pix] = c.y;
    ib[2 * (size_t)HW + pix] = c.z;
    ib[3 * (size_t)HW + pix] = rng;
    if (index_map) index_map[o] = cell;
    pts_grid[o] = cell >= 0 ? make_float4(c.x, c.y, c.z, __int_as_float(pix)) : make_float4(inf, inf, inf, __int_as_float(-1));
    nrm_grid[o] = q;
}

// ---- delora_normalization_factors: the Deployer's normalize_input factor of B pairs, deterministic.
// One cluster of 2 x kFactorParts CTAs per pair: CTA r sums the ranges of scan (r / kFactorParts) of the pair, the points
// i = (r % kFactorParts) * kFactorThreads + thread + k * kFactorParts * kFactorThreads, k = 0, 1, ... in order, in
// float64; the warps' sums meet in an xor butterfly, the CTA's 32 warp sums in warp order, and CTA 0 adds the parts of
// each scan in rank order through distributed shared memory.  The order depends on neither B nor the launch, so the
// factor is bit-identical from run to run.  Reads 12 bytes per point.
// kGrid (the training step's preprocessing grids): the points are the valid cells of [2B, n] float4 grids (w = pixel-id
// bits, >= 0; empty cells (+inf, +inf, +inf, -1) are skipped and not counted), in cell order: the row-major lists the
// reference's preprocessing stored.  Reads 16 bytes per cell.
// The kernel is bound by the latency of each thread's chain of loads, so a pair gets 8 full CTAs and every thread keeps
// 8 points' loads in flight.
constexpr int kFactorThreads = 1024;
constexpr int kFactorParts = 4;
constexpr int kFactorUnroll = 8;       // independent point loads in flight per thread

template <bool kGrid>
__global__ void __cluster_dims__(2 * kFactorParts, 1, 1) __launch_bounds__(kFactorThreads)
normalization_factor_kernel(const float* __restrict__ points, const int32_t* __restrict__ n_points,
                            const float4* __restrict__ grid, int B, int n_stride, float* __restrict__ factor) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ double s_warp[kFactorThreads / 32];
    __shared__ int s_warp_n[kFactorThreads / 32];
    __shared__ double s_part;
    __shared__ int s_part_n;
    const int rank = (int)cluster.block_rank();
    const int pair = blockIdx.x / (2 * kFactorParts);
    const int side = rank / kFactorParts, part = rank % kFactorParts;
    const int scan = side * B + pair;
    const int n = kGrid ? n_stride : min(max(n_points[scan], 0), n_stride);
    const float* __restrict__ px = points + (size_t)scan * 3 * n_stride;
    const float* __restrict__ py = px + n_stride;
    const float* __restrict__ pz = py + n_stride;
    const float4* __restrict__ pg = grid + (size_t)scan * n_stride;
    constexpr int kStep = kFactorParts * kFactorThreads;
    double acc = 0.0;
    int cnt = 0;
    for (int base = part * kFactorThreads + threadIdx.x; base < n; base += kFactorUnroll * kStep) {
        float r[kFactorUnroll];
        bool ok[kFactorUnroll];
#pragma unroll
        for (int u = 0; u < kFactorUnroll; ++u) {
            const int i = base + u * kStep;
            if (kGrid) {
                const float4 c = i < n ? __ldg(pg + i) : make_float4(0.0f, 0.0f, 0.0f, __int_as_float(-1));
                ok[u] = __float_as_int(c.w) >= 0;
                r[u] = ok[u] ? range3(c.x, c.y, c.z) : 0.0f;
            } else {
                ok[u] = i < n;
                r[u] = ok[u] ? range3(__ldg(px + i), __ldg(py + i), __ldg(pz + i)) : 0.0f;
            }
        }
#pragma unroll
        for (int u = 0; u < kFactorUnroll; ++u) {
            acc += (double)r[u];
            cnt += ok[u] ? 1 : 0;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        acc += __shfl_xor_sync(0xffffffffu, acc, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((threadIdx.x & 31) == 0) { s_warp[threadIdx.x >> 5] = acc; s_warp_n[threadIdx.x >> 5] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        int c = 0;
        for (int w = 0; w < kFactorThreads / 32; ++w) { t += s_warp[w]; c += s_warp_n[w]; }
        s_part = t;
        s_part_n = c;
    }
    cluster.sync();
    if (rank == 0 && threadIdx.x == 0) {
        float m[2];
        for (int sd = 0; sd < 2; ++sd) {
            double t = 0.0;
            int ns = 0;
            for (int q = 0; q < kFactorParts; ++q) {
                t += *cluster.map_shared_rank(&s_part, sd * kFactorParts + q);
                ns += *cluster.map_shared_rank(&s_part_n, sd * kFactorParts + q);
            }
            m[sd] = (float)(t / (double)ns);           // an empty scan gives 0 / 0 = NaN, as torch.mean of nothing
        }
        factor[pair] = __fdiv_rn(__fadd_rn(m[0], m[1]), 2.0f);
    }
    cluster.sync();                                     // keep every CTA's partials alive until rank 0 has read them
}

int launch_normalization_factors(const float* points, const int32_t* n_points, int B, int n_stride, float* factor,
                                 cudaStream_t st) {
    normalization_factor_kernel<false><<<2 * kFactorParts * B, kFactorThreads, 0, st>>>(points, n_points, nullptr, B,
                                                                                        n_stride, factor);
    DELORA_CHECK_LAUNCH("normalization_factor_kernel");
    return 0;
}

int project_grids_fwd(const delora_f4* pts_grid_pre, const delora_f4* nrm_grid_pre, int S, int Wp, const GridParams& g,
                      uint64_t* keys, float* image, int32_t* index_map, delora_f4* pts_grid, delora_f4* nrm_grid,
                      const float* factor, int fB, cudaStream_t st) {
    const int HWp = g.H * Wp, HW = g.H * g.W;
    const int per_block = kScatterThreads * kScatterPPT;
    const dim3 g1((HWp + per_block - 1) / per_block, S), g2((HW + 255) / 256, S);
    const float4* pp = (const float4*)pts_grid_pre;
    const float4* np_ = (const float4*)nrm_grid_pre;
    unsigned long long* k = (unsigned long long*)keys;
    if (factor)
        grids_scatter_kernel<true><<<g1, kScatterThreads, 0, st>>>(pp, HWp, g, k, factor, fB);
    else
        grids_scatter_kernel<false><<<g1, kScatterThreads, 0, st>>>(pp, HWp, g, k, nullptr, 0);
    DELORA_CHECK_LAUNCH("grids_scatter_kernel");
    if (factor)
        grids_resolve_kernel<true><<<g2, 256, 0, st>>>(pp, np_, HWp, HW, k, image, index_map, (float4*)pts_grid,
                                                       (float4*)nrm_grid, factor, fB);
    else
        grids_resolve_kernel<false><<<g2, 256, 0, st>>>(pp, np_, HWp, HW, k, image, index_map, (float4*)pts_grid,
                                                        (float4*)nrm_grid, nullptr, 0);
    DELORA_CHECK_LAUNCH("grids_resolve_kernel");
    return 0;
}

int launch_grid_normalization_factors(const delora_f4* grid, int B, int n_cells, float* factor, cudaStream_t st) {
    normalization_factor_kernel<true><<<2 * kFactorParts * B, kFactorThreads, 0, st>>>(
        nullptr, nullptr, (const float4*)grid, B, n_cells, factor);
    DELORA_CHECK_LAUNCH("normalization_factor_kernel");
    return 0;
}

}  // namespace delora

using namespace delora;

extern "C" int delora_normalization_factors(const float* points, const int32_t* n_points, int B, int n_stride,
                                            float* factor, void* stream) {
    const char* who = "delora_normalization_factors";
    DELORA_CHECK_ARG(points, "%s: null points", who);
    DELORA_CHECK_ARG(n_points, "%s: null n_points", who);
    DELORA_CHECK_ARG(factor, "%s: null factor", who);
    DELORA_CHECK_ARG(B >= 1 && B <= 65535, "%s: B=%d outside [1, 65535]", who, B);
    DELORA_CHECK_ARG(n_stride >= 1, "%s: n_stride=%d must be >= 1", who, n_stride);
    return launch_normalization_factors(points, n_points, B, n_stride, factor, (cudaStream_t)stream);
}

extern "C" int delora_project_fwd(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                                  int H, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                                  int div_mode, uint64_t* keys, float* image, int32_t* index_map,
                                  void* stream) {
    DELORA_CHECK_ARG(points && n_points && keys && image && index_map, "delora_project_fwd: null pointer");
    DELORA_CHECK_ARG(B > 0 && C >= 3 && n_stride > 0 && H > 0 && W > 0,
                     "delora_project_fwd: bad shape B=%d C=%d n_stride=%d H=%d W=%d", B, C, n_stride, H, W);
    DELORA_CHECK_ARG((long long)H * W < (1ll << 31) && B <= 65535, "delora_project_fwd: image or batch too large");
    const GridParams g = make_grid(H, W, hfov0, hfov1, vfov0, vfov1, div_mode);
    return project_fwd(points, n_points, B, C, n_stride, g, keys, image, index_map, nullptr, 0, (cudaStream_t)stream);
}

extern "C" int delora_project_grids_fwd(const delora_f4* pts_grid_pre, const delora_f4* nrm_grid_pre, int S, int H,
                                        int Wp, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                                        int div_mode, uint64_t* keys, float* image, int32_t* index_map,
                                        delora_f4* pts_grid, delora_f4* nrm_grid, void* stream) {
    DELORA_CHECK_ARG(pts_grid_pre && nrm_grid_pre && keys && image && pts_grid && nrm_grid,
                     "delora_project_grids_fwd: null pointer");
    DELORA_CHECK_ARG(S > 0 && S <= 65535 && H > 0 && Wp > 0 && W > 0,
                     "delora_project_grids_fwd: bad shape S=%d H=%d Wp=%d W=%d", S, H, Wp, W);
    DELORA_CHECK_ARG((long long)H * Wp < (1ll << 31) && (long long)H * W < (1ll << 31),
                     "delora_project_grids_fwd: image too large");
    const GridParams g = make_grid(H, W, hfov0, hfov1, vfov0, vfov1, div_mode);
    return project_grids_fwd(pts_grid_pre, nrm_grid_pre, S, Wp, g, keys, image, index_map, pts_grid, nrm_grid, nullptr, 0,
                             (cudaStream_t)stream);
}

extern "C" int delora_project_uv(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                                 int H, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                                 int div_mode, float* u, float* v, float* range, void* stream) {
    DELORA_CHECK_ARG(points && n_points && u && v, "delora_project_uv: null pointer");
    DELORA_CHECK_ARG(B > 0 && C >= 3 && n_stride > 0 && B <= 65535, "delora_project_uv: bad shape");
    const GridParams g = make_grid(H, W, hfov0, hfov1, vfov0, vfov1, div_mode);
    dim3 grid((n_stride + 255) / 256, B);
    project_uv_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(points, n_points, C, n_stride, g, u, v, range);
    DELORA_CHECK_LAUNCH("project_uv_kernel");
    return 0;
}
