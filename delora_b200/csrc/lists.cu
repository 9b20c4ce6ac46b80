// Image -> point/normal lists and spherical cell index (CSR over pixels) (sm_90a).
//
// delora_lists_from_images: the reference's `get_image_coords` / list outputs
//   (src/preprocessing/normal_computation.py:30-41, :84-87): the valid pixels
//   (x!=0 & y!=0 & z!=0) in row-major order, with their normals.  The exclusive prefix sum of
//   the valid flags is at the same time the CSR `cell_start` of the NN search grid.
// delora_grid_build: counting sort of arbitrary [3,N] lists by spherical cell, the structure
//   that replaces `scipy.spatial.cKDTree(target)` (src/losses/icp_losses.py:34).
// Both are integer/byte work bounded by HBM/L2 bandwidth: read 12-24 B, write 32 B per point.
#include "common.cuh"

namespace delora {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 4;
constexpr int kScanTile = kScanThreads * kScanItems;   // cells per block

__device__ __forceinline__ int block_exclusive_scan(int val, int& total) {
    // exclusive scan of one int per thread over a 256-thread block
    __shared__ int warp_tot[kScanThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int inc = val;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_tot[w] = inc;
    __syncthreads();
    int base = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < kScanThreads / 32; ++i) {
        const int t = warp_tot[i];
        if (i < w) base += t;
        tot += t;
    }
    total = tot;
    __syncthreads();
    return base + inc - val;
}

__device__ __forceinline__ int block_sum(int val) {
    __shared__ int warp_tot2[kScanThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) val += __shfl_xor_sync(0xffffffffu, val, o);
    if (lane == 0) warp_tot2[w] = val;
    __syncthreads();
    int tot = 0;
#pragma unroll
    for (int i = 0; i < kScanThreads / 32; ++i) tot += warp_tot2[i];
    __syncthreads();
    return tot;
}

// sum of the block counts that precede this block (same scan segment)
__device__ __forceinline__ int preceding_blocks_sum(const int32_t* __restrict__ block_counts, int blk) {
    int s = 0;
    for (int j = threadIdx.x; j < blk; j += kScanThreads) s += block_counts[j];
    return block_sum(s);
}

// ---- image flags ------------------------------------------------------------------------
__device__ __forceinline__ bool valid_pixel(const float* __restrict__ img, size_t HW, int pix) {
    return __ldg(img + pix) != 0.0f && __ldg(img + HW + pix) != 0.0f && __ldg(img + 2 * HW + pix) != 0.0f;
}

__global__ void __launch_bounds__(kScanThreads)
image_count_kernel(const float* __restrict__ image, int C_img, int HW, int32_t* __restrict__ block_counts) {
    const int b = blockIdx.y;
    const float* __restrict__ img = image + (size_t)b * C_img * HW;
    const int p0 = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
    int c = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j)
        if (p0 + j < HW) c += valid_pixel(img, HW, p0 + j) ? 1 : 0;
    const int tot = block_sum(c);
    if (threadIdx.x == 0) block_counts[b * gridDim.x + blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kScanThreads)
image_emit_kernel(const float* __restrict__ image, const float* __restrict__ normals, int C_img, int HW,
                  const int32_t* __restrict__ block_counts, delora_f4* __restrict__ pts4,
                  delora_f4* __restrict__ nrm4, int32_t* __restrict__ cell_start, int32_t* __restrict__ counts) {
    const int b = blockIdx.y;
    const size_t sHW = (size_t)HW;
    const float* __restrict__ img = image + (size_t)b * C_img * sHW;
    const float* __restrict__ nrm = normals + (size_t)b * 3 * sHW;
    const int base = preceding_blocks_sum(block_counts + b * gridDim.x, blockIdx.x);
    const int p0 = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
    bool f[kScanItems];
    int c = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        f[j] = (p0 + j < HW) && valid_pixel(img, sHW, p0 + j);
        c += f[j] ? 1 : 0;
    }
    int total;
    int pos = base + block_exclusive_scan(c, total);
    float4* __restrict__ po = reinterpret_cast<float4*>(pts4) + (size_t)b * sHW;
    float4* __restrict__ no = reinterpret_cast<float4*>(nrm4) + (size_t)b * sHW;
    int32_t* __restrict__ cs = cell_start + (size_t)b * (sHW + 1);
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        const int pix = p0 + j;
        if (pix < HW) {
            cs[pix] = pos;
            if (f[j]) {
                po[pos] = make_float4(__ldg(img + pix), __ldg(img + sHW + pix), __ldg(img + 2 * sHW + pix),
                                      __int_as_float(pix));
                const float nx = __ldg(nrm + pix), ny = __ldg(nrm + sHW + pix), nz = __ldg(nrm + 2 * sHW + pix);
                const bool has = (nx != 0.0f) | (ny != 0.0f) | (nz != 0.0f);       // icp_losses.py:48-52
                no[pos] = make_float4(nx, ny, nz, has ? 1.0f : 0.0f);
                ++pos;
            }
        }
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == kScanThreads - 1) {
        // the last thread of the last block holds the inclusive total
        cs[HW] = pos;
        counts[b] = pos;
    }
}

// ---- generic lists: counting sort by cell -----------------------------------------------
// Points outside the field of view live in the border cells.  Rows clamp.  An azimuth in the horizontal gap (G =
// circ_px - wm1 pixels from the centre of column W-1 round to the centre of column 0) goes to the border column it is
// nearer to around the circle, not to the one on its side of atan2's +-pi wrap.  nn_search's column bounds take a
// target in column W-1 to lie at least 0.5 - seam_px pixels before column 0's centre (seam_px = max(0, 1 - G)), and
// one in column 0 as far past column W-1's centre.  Split at the gap's middle, the border columns keep their targets
// at least G/2 away from each other's centre, and G/2 >= 0.5 - max(0, 1 - G) for every G.  The plain clamp put an
// azimuth just short of column 0's centre into column W-1 (or the mirror image), which breaks the bound for G > 1/2.
__device__ __forceinline__ int cell_of(const GridParams& g, float x, float y, float z) {
    float u, v;
    pixel_coords(g, x, y, z, u, v);
    float ru = rintf(u);
    if (ru < 0.0f || ru > g.wm1) {                      // NaN fails both tests and is clamped to 0 below
        const float past = u > g.wm1 ? u - g.wm1 : (u + g.circ_px) - g.wm1;    // pixels past column W-1's centre
        ru = past <= 0.5f * (g.circ_px - g.wm1) ? g.wm1 : 0.0f;
    }
    const float cu = fminf(fmaxf(ru, 0.0f), g.wm1);
    const float rv = fminf(fmaxf(rintf(v), 0.0f), g.hm1);
    return (int)rv * g.W + (int)cu;
}

__global__ void __launch_bounds__(256)
bin_count_kernel(const float* __restrict__ pts, const int32_t* __restrict__ n, int n_stride, GridParams g,
                 int32_t* __restrict__ cursor) {
    const int b = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n[b]) return;
    const float* __restrict__ p = pts + (size_t)b * 3 * n_stride;
    const int cell = cell_of(g, __ldg(p + i), __ldg(p + n_stride + i), __ldg(p + 2 * (size_t)n_stride + i));
    atomicAdd(cursor + (size_t)b * g.H * g.W + cell, 1);
}

__global__ void __launch_bounds__(kScanThreads)
counts_block_kernel(const int32_t* __restrict__ cursor, int HW, int32_t* __restrict__ block_counts) {
    const int b = blockIdx.y;
    const int p0 = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
    int c = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j)
        if (p0 + j < HW) c += cursor[(size_t)b * HW + p0 + j];
    const int tot = block_sum(c);
    if (threadIdx.x == 0) block_counts[b * gridDim.x + blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kScanThreads)
counts_scan_kernel(int32_t* __restrict__ cursor, int HW, const int32_t* __restrict__ block_counts,
                   int32_t* __restrict__ cell_start) {
    const int b = blockIdx.y;
    const int base = preceding_blocks_sum(block_counts + b * gridDim.x, blockIdx.x);
    const int p0 = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
    int cnt[kScanItems];
    int c = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        cnt[j] = (p0 + j < HW) ? cursor[(size_t)b * HW + p0 + j] : 0;
        c += cnt[j];
    }
    int total;
    int pos = base + block_exclusive_scan(c, total);
    int32_t* __restrict__ cs = cell_start + (size_t)b * ((size_t)HW + 1);
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        if (p0 + j < HW) {
            cs[p0 + j] = pos;
            cursor[(size_t)b * HW + p0 + j] = 0;       // becomes the scatter cursor
            pos += cnt[j];
        }
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == kScanThreads - 1) cs[HW] = pos;
}

__global__ void __launch_bounds__(256)
bin_scatter_kernel(const float* __restrict__ pts, const float* __restrict__ nrm, const int32_t* __restrict__ n,
                   int n_stride, GridParams g, const int32_t* __restrict__ cell_start,
                   int32_t* __restrict__ cursor, delora_f4* __restrict__ pts4, delora_f4* __restrict__ nrm4) {
    const int b = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n[b]) return;
    const size_t HW = (size_t)g.H * g.W;
    const float* __restrict__ p = pts + (size_t)b * 3 * n_stride;
    const float x = __ldg(p + i), y = __ldg(p + n_stride + i), z = __ldg(p + 2 * (size_t)n_stride + i);
    const int cell = cell_of(g, x, y, z);
    const int pos = cell_start[(size_t)b * (HW + 1) + cell] + atomicAdd(cursor + (size_t)b * HW + cell, 1);
    reinterpret_cast<float4*>(pts4)[(size_t)b * n_stride + pos] = make_float4(x, y, z, __int_as_float(i));
    float nx = 0.f, ny = 0.f, nz = 0.f;
    if (nrm) {
        const float* __restrict__ q = nrm + (size_t)b * 3 * n_stride;
        nx = __ldg(q + i); ny = __ldg(q + n_stride + i); nz = __ldg(q + 2 * (size_t)n_stride + i);
    }
    const bool has = (nx != 0.0f) | (ny != 0.0f) | (nz != 0.0f);
    reinterpret_cast<float4*>(nrm4)[(size_t)b * n_stride + pos] = make_float4(nx, ny, nz, has ? 1.0f : 0.0f);
}

__global__ void __launch_bounds__(256)
pack_lists_kernel(const float* __restrict__ pts, const float* __restrict__ nrm, const int32_t* __restrict__ n,
                  int n_stride, delora_f4* __restrict__ pts4, delora_f4* __restrict__ nrm4) {
    const int b = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n[b]) return;
    const float* __restrict__ p = pts + (size_t)b * 3 * n_stride;
    reinterpret_cast<float4*>(pts4)[(size_t)b * n_stride + i] =
        make_float4(__ldg(p + i), __ldg(p + n_stride + i), __ldg(p + 2 * (size_t)n_stride + i), __int_as_float(i));
    if (nrm4) {
        float nx = 0.f, ny = 0.f, nz = 0.f;
        if (nrm) {
            const float* __restrict__ q = nrm + (size_t)b * 3 * n_stride;
            nx = __ldg(q + i); ny = __ldg(q + n_stride + i); nz = __ldg(q + 2 * (size_t)n_stride + i);
        }
        const bool has = (nx != 0.0f) | (ny != 0.0f) | (nz != 0.0f);
        reinterpret_cast<float4*>(nrm4)[(size_t)b * n_stride + i] = make_float4(nx, ny, nz, has ? 1.0f : 0.0f);
    }
}

// Training-step layout: the projection kept one point per pixel (index_map) out of a scan whose
// normals were precomputed per point (the reference sub-selects both lists with the projection's
// point indices: src/deploy/deployer.py:258-261).  Gather them into the dense float4 grids.
__global__ void __launch_bounds__(256)
grids_from_projection_kernel(const float* __restrict__ points, const float* __restrict__ normal_lists,
                             const int32_t* __restrict__ index_map, int C, int n_stride, int HW,
                             float4* __restrict__ pts_grid, float4* __restrict__ nrm_grid) {
    const int b = blockIdx.y, pix = blockIdx.x * 256 + threadIdx.x;
    if (pix >= HW) return;
    const int idx = index_map[(size_t)b * HW + pix];
    const float inf = __int_as_float(0x7f800000);
    float4 p = make_float4(inf, inf, inf, __int_as_float(-1)), q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (idx >= 0) {
        const float* __restrict__ pb = points + (size_t)b * C * n_stride;
        p = make_float4(__ldg(pb + idx), __ldg(pb + n_stride + idx), __ldg(pb + 2 * (size_t)n_stride + idx),
                        __int_as_float(pix));
        const float* __restrict__ nb = normal_lists + (size_t)b * 3 * n_stride;
        const float nx = __ldg(nb + idx), ny = __ldg(nb + n_stride + idx), nz = __ldg(nb + 2 * (size_t)n_stride + idx);
        const bool has = (nx != 0.0f) | (ny != 0.0f) | (nz != 0.0f);                     // icp_losses.py:48-52
        q = make_float4(nx, ny, nz, has ? 1.0f : 0.0f);
    }
    pts_grid[(size_t)b * HW + pix] = p;
    nrm_grid[(size_t)b * HW + pix] = q;
}

}  // namespace delora

using namespace delora;

extern "C" int delora_grids_from_projection(const float* points, const float* normal_lists,
                                            const int32_t* index_map, int B, int C, int n_stride, int H, int W,
                                            delora_f4* pts_grid, delora_f4* nrm_grid, void* stream) {
    DELORA_CHECK_ARG(points && normal_lists && index_map && pts_grid && nrm_grid,
                     "delora_grids_from_projection: null pointer");
    DELORA_CHECK_ARG(B > 0 && B <= 65535 && C >= 3 && n_stride > 0 && H > 0 && W > 0,
                     "delora_grids_from_projection: bad shape");
    const int HW = H * W;
    dim3 grid((HW + 255) / 256, B);
    grids_from_projection_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(points, normal_lists, index_map, C, n_stride,
                                                                         HW, (float4*)pts_grid, (float4*)nrm_grid);
    DELORA_CHECK_LAUNCH("grids_from_projection_kernel");
    return 0;
}


extern "C" int delora_scan_blocks(int n_cells) { return (n_cells + kScanTile - 1) / kScanTile; }

extern "C" int delora_lists_from_images(const float* image, const float* normals, int B, int C_img, int H, int W,
                                        delora_f4* pts4, delora_f4* nrm4, int32_t* cell_start, int32_t* counts,
                                        int32_t* scratch, void* stream) {
    DELORA_CHECK_ARG(image && normals && pts4 && nrm4 && cell_start && counts && scratch,
                     "delora_lists_from_images: null pointer");
    DELORA_CHECK_ARG(B > 0 && B <= 65535 && C_img >= 3 && H > 0 && W > 0, "delora_lists_from_images: bad shape");
    const int HW = H * W;
    dim3 grid(delora_scan_blocks(HW), B);
    cudaStream_t st = (cudaStream_t)stream;
    image_count_kernel<<<grid, kScanThreads, 0, st>>>(image, C_img, HW, scratch);
    DELORA_CHECK_LAUNCH("image_count_kernel");
    image_emit_kernel<<<grid, kScanThreads, 0, st>>>(image, normals, C_img, HW, scratch, pts4, nrm4, cell_start,
                                                     counts);
    DELORA_CHECK_LAUNCH("image_emit_kernel");
    return 0;
}

extern "C" int delora_grid_build(const float* pts, const float* nrm, const int32_t* n, int B, int n_stride,
                                 int H, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                                 delora_f4* pts4, delora_f4* nrm4, int32_t* cell_start, int32_t* cursor,
                                 int32_t* scratch, void* stream) {
    DELORA_CHECK_ARG(pts && n && pts4 && nrm4 && cell_start && cursor && scratch, "delora_grid_build: null pointer");
    DELORA_CHECK_ARG(B > 0 && B <= 65535 && n_stride > 0 && H > 0 && W > 0, "delora_grid_build: bad shape");
    const GridParams g = make_grid(H, W, hfov0, hfov1, vfov0, vfov1, 1);
    const int HW = H * W;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(cursor, 0, sizeof(int32_t) * (size_t)B * HW, st);
    DELORA_CHECK_ARG(e == cudaSuccess, "delora_grid_build: memset failed: %s", cudaGetErrorString(e));
    dim3 gp((n_stride + 255) / 256, B);
    bin_count_kernel<<<gp, 256, 0, st>>>(pts, n, n_stride, g, cursor);
    DELORA_CHECK_LAUNCH("bin_count_kernel");
    dim3 gs(delora_scan_blocks(HW), B);
    counts_block_kernel<<<gs, kScanThreads, 0, st>>>(cursor, HW, scratch);
    DELORA_CHECK_LAUNCH("counts_block_kernel");
    counts_scan_kernel<<<gs, kScanThreads, 0, st>>>(cursor, HW, scratch, cell_start);
    DELORA_CHECK_LAUNCH("counts_scan_kernel");
    bin_scatter_kernel<<<gp, 256, 0, st>>>(pts, nrm, n, n_stride, g, cell_start, cursor, pts4, nrm4);
    DELORA_CHECK_LAUNCH("bin_scatter_kernel");
    return 0;
}

extern "C" int delora_pack_lists(const float* pts, const float* nrm, const int32_t* n, int B, int n_stride,
                                 delora_f4* pts4, delora_f4* nrm4, void* stream) {
    DELORA_CHECK_ARG(pts && n && pts4, "delora_pack_lists: null pointer");
    DELORA_CHECK_ARG(B > 0 && B <= 65535 && n_stride > 0, "delora_pack_lists: bad shape");
    dim3 gp((n_stride + 255) / 256, B);
    pack_lists_kernel<<<gp, 256, 0, (cudaStream_t)stream>>>(pts, nrm, n, n_stride, pts4, nrm4);
    DELORA_CHECK_LAUNCH("pack_lists_kernel");
    return 0;
}
