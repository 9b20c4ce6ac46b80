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
//
// HBM/L2 traffic per scan: read 12 N (xyz) [+ 8 HW key RMW in L2] ; write 4 (C+1) HW + 4 HW.
#include "projection.cuh"

namespace delora {

constexpr int kScatterThreads = 256;
constexpr int kScatterPPT = 4;       // points per thread (independent loads in flight)

__global__ void __launch_bounds__(kScatterThreads)
project_scatter_kernel(const float* __restrict__ points, const int32_t* __restrict__ n_points,
                       int C, int n_stride, GridParams g, unsigned long long* __restrict__ keys) {
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

    float x[kScatterPPT], y[kScatterPPT], z[kScatterPPT];
#pragma unroll
    for (int i = 0; i < kScatterPPT; ++i) {
        const int idx = base + i * kScatterThreads;
        const bool ok = idx < n;
        x[i] = ok ? __ldg(px + idx) : 0.0f;
        y[i] = ok ? __ldg(py + idx) : 0.0f;
        z[i] = ok ? __ldg(pz + idx) : 0.0f;
    }
#pragma unroll
    for (int i = 0; i < kScatterPPT; ++i) {
        const int idx = base + i * kScatterThreads;
        float u, v;
        pixel_coords(g, x[i], y[i], z[i], u, v);
        const float ru = rintf(u), rv = rintf(v);            // torch.round: half to even (:74-77)
        const bool inside = (idx < n) && (ru <= g.wm1) && (ru >= 0.0f) && (rv <= g.hm1) && (rv >= 0.0f);
        if (inside) {
            const unsigned rbits = __float_as_uint(range3(x[i], y[i], z[i]));
            // One 64-bit atomicMin (a fire-and-forget RED at L2) per in-FOV point.  A match.any /
            // redux.min warp aggregation does not pay here: redux with per-group masks serialises
            // once per distinct pixel (~28 groups per warp at W = 2048), while 2 M atomics per step
            // are far below the L2 atomic rate.
            atomicMin(kb + (int)rv * g.W + (int)ru, ((unsigned long long)rbits << 32) | (unsigned)idx);
        }
    }
}

// One thread resolves 4 consecutive pixels: 2 x 16-byte key loads, float4 stores per channel.
// CT = compile-time channel count (3: xyz, 4: xyz + reflectance) so that all 4 x CT gathers are issued before
// the first store (the kernel is latency-bound on them); CT = 0: generic loop.
template <int CT>
__global__ void __launch_bounds__(256)
project_resolve_kernel(const float* __restrict__ points, int C, int n_stride, int HW,
                       unsigned long long* __restrict__ keys, float* __restrict__ image,
                       int32_t* __restrict__ index_map) {
    const int b = blockIdx.y;
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
            for (int j = 0; j < 4; ++j) val[c][j] = idx[j] >= 0 ? __ldg(pb + (size_t)c * n_stride + idx[j]) : 0.0f;
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
            for (int j = 0; j < 4; ++j) val[j] = idx[j] >= 0 ? __ldg(pb + (size_t)c * n_stride + idx[j]) : 0.0f;
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
                            const GridParams& g, unsigned long long* keys, cudaStream_t st) {
    const int per_block = kScatterThreads * kScatterPPT;
    dim3 grid((n_stride + per_block - 1) / per_block, B);
    project_scatter_kernel<<<grid, kScatterThreads, 0, st>>>(points, n_points, C, n_stride, g, keys);
}

}  // namespace delora

using namespace delora;

extern "C" int delora_project_fwd(const float* points, const int32_t* n_points, int B, int C, int n_stride,
                                  int H, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                                  int div_mode, uint64_t* keys, float* image, int32_t* index_map,
                                  void* stream) {
    DELORA_CHECK_ARG(points && n_points && keys && image && index_map, "delora_project_fwd: null pointer");
    DELORA_CHECK_ARG(B > 0 && C >= 3 && n_stride > 0 && H > 0 && W > 0,
                     "delora_project_fwd: bad shape B=%d C=%d n_stride=%d H=%d W=%d", B, C, n_stride, H, W);
    DELORA_CHECK_ARG((long long)H * W < (1ll << 31) && B <= 65535, "delora_project_fwd: image or batch too large");
    cudaStream_t st = (cudaStream_t)stream;
    const GridParams g = make_grid(H, W, hfov0, hfov1, vfov0, vfov1, div_mode);
    launch_project_scatter(points, n_points, B, C, n_stride, g, (unsigned long long*)keys, st);
    DELORA_CHECK_LAUNCH("project_scatter_kernel");
    const int HW = H * W;
    dim3 grid2((HW + 1023) / 1024, B);
    if (C == 3)
        project_resolve_kernel<3><<<grid2, 256, 0, st>>>(points, C, n_stride, HW, (unsigned long long*)keys, image, index_map);
    else if (C == 4)
        project_resolve_kernel<4><<<grid2, 256, 0, st>>>(points, C, n_stride, HW, (unsigned long long*)keys, image, index_map);
    else
        project_resolve_kernel<0><<<grid2, 256, 0, st>>>(points, C, n_stride, HW, (unsigned long long*)keys, image, index_map);
    DELORA_CHECK_LAUNCH("project_resolve_kernel");
    return 0;
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
