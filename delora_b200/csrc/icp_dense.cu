// Fused SE(3) transform + exact NN + ICP losses fwd/bwd on DENSE range-image grids (sm_90a).
//
// Same contract as icp.cu (reference: src/deploy/deployer.py:181-189, src/losses/icp_losses.py:28-240),
// specialised for the case the training step actually has: source and target are the valid pixels
// of two projected H x W range images, i.e. at most one point per spherical cell.  Points and
// normals live as float4 per pixel ((x, y, z, pixel id) / (nx, ny, nz, has_normal); empty pixels
// are (+inf, +inf, +inf, -1)), written by the normals kernel, so no list compaction and no
// CSR index are needed and a window of cells is a fixed-stride walk over one array.
//
// One thread per SOURCE PIXEL; a warp = 32 adjacent pixels.  The search window is described by
// warp-uniform extents (rows down/up, columns left/right of every lane's own centre cell) and
// grows one strip at a time while ANY lane's exactness guard still fails, on the side the first
// failing lane needs.  Control flow is warp-uniform (no divergence), adjacent lanes read adjacent
// cells (coalesced, L1-resident), and the guard is the same proof as in icp.cu: all unsearched
// targets lie beyond a border half-plane (azimuth) or cone (elevation) of the lane's window.  Row (cone)
// borders also use the RANGE of the targets beyond them (row_border_bound).
//
// Four launches per call (DESIGN.md 4.3): target_extents_kernel ([min, max] range per 4 x 16-cell block and prefix /
// suffix range extents per pixel row of the target grids), icp_dense_kernel (its programmatic dependent: window
// search, bounded number of growing steps; lanes still open are appended to a work list), icp_dense_pending_kernel
// (one warp per open lane: range-pruned block search, float64 tie re-ranking, accumulation by the warp that completes
// an item) and icp_finalize_kernel (icp.cu: fixed-order fp64 column sums -> losses and the 3x4 transform gradient).
#include <stdlib.h>
#include <algorithm>
#include "icp_common.cuh"

namespace delora {

constexpr int kDenseThreads = 128;
constexpr float kInf = 3.0e38f;     // "no bound": the border does not exist, or nothing valid lies beyond it
constexpr float kSlack = 2e-3f;     // px subtracted from every border distance; covers the fp32 error of the cell binning

__device__ __forceinline__ int wrap_col(int c, int W) {
    c += (c < 0) ? W : 0;
    c -= (c >= W) ? W : 0;
    return c;
}

// lower bound of the distance from the source point to everything beyond a window border that is
// `dpx` pixels (of `rad_per_px` radians) away; `radius` is |p| (elevation cones) or |p_xy| (azimuth planes).
// __sinf (MUFU.SIN, absolute error ~2^-21.4 for |x| <= pi) inside an exactness proof is covered by the callers'
// margin: every bound is scaled by 0.9995 and shrunk by 2e-3 px before it is compared.  At one pixel of a
// W = 2250 image (2.8e-3 rad) the intrinsic's error is 1.3e-4 relative -- a quarter of the margin.  The limit
// of validity is a pixel pitch of ~7e-4 rad (W ~ 9000 columns): finer grids need sinf() here.
__device__ __forceinline__ float border_bound(float dpx, float rad_per_px, float radius) {
    const float d = fminf(fmaxf(dpx * rad_per_px, 0.0f), kHalfPiF);
    return radius * __sinf(d);
}

// Branch-free running (smallest, second smallest) fp32 squared distance + index of the smallest.
// The whole search runs on this; float64 is only consulted afterwards if the two smallest are
// within kNNBand of each other (nn_exact_rescan).
struct NN2 {
    float m1, m2;
    int j1;
};

__device__ __forceinline__ void nn2_eval(const float4 t, int j, float sx, float sy, float sz, NN2& s,
                                         bool ok = true) {
    const float dx = sx - t.x, dy = sy - t.y, dz = sz - t.z;
    const float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
    const float d2f = ok ? d2 : __int_as_float(0x7f800000);      // out-of-grid rows / idle lanes never win
    const bool lt = d2f < s.m1;
    s.m2 = lt ? s.m1 : fminf(s.m2, d2f);
    s.j1 = lt ? j : s.j1;
    s.m1 = lt ? d2f : s.m1;
}

__device__ __forceinline__ float4 inf4() {
    const float inf = __int_as_float(0x7f800000);
    return make_float4(inf, inf, inf, __int_as_float(-1));
}

// Rare path: two candidates within the fp32 ambiguity band.  Re-rank every candidate of the
// final window whose fp32 distance is inside the band in float64 (lowest pixel id on exact ties).
__device__ __noinline__ int nn_exact_rescan(const float4* __restrict__ tg, int H, int W, int rc, int cc, int e_dn,
                                            int e_up, int e_lf, int e_rt, float sx, float sy, float sz,
                                            float thresh) {
    double best = 1.0e300;
    int bj = -1;
    for (int dr = -e_dn; dr <= e_up; ++dr) {
        const int row = rc + dr;
        if (row < 0 || row >= H) continue;
        for (int dc = -e_lf; dc <= e_rt; ++dc) {
            const int j = row * W + wrap_col(cc + dc, W);
            const float4 t = __ldg(tg + j);
            const float dx = sx - t.x, dy = sy - t.y, dz = sz - t.z;
            const float d2f = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
            if (d2f <= thresh) {
                const double d2 = nn_d2_exact(sx, sy, sz, t.x, t.y, t.z);
                if (d2 < best || (d2 == best && j < bj)) { best = d2; bj = j; }
            }
        }
    }
    return bj;
}

// ---------------------------------------------------------------------------------------------
// Range pyramid for the far / misaligned case.  The strip search certifies its column borders with a
// purely ANGULAR bound, so a source point that is d away from the target surface has to scan every
// cell within the angle asin(d/r) -- thousands of cells when the predicted transform is still poor
// (d ~ 1 m), although almost all of them are provably farther than d once their RANGE is taken into
// account.  Blocks of 4 x 16 cells carry [min, max] of |t|; a block whose lower bound
//     min over rho in [rmin, rmax] of (r_s - rho)^2 + 4 r_s rho sin^2(theta/2),
//     sin^2(theta/2) >= max( sin^2(gap_el/2), cos(e_s) * min cos(e_blk) * sin^2(gap_az/2) )
// exceeds the current best distance cannot hold the nearest neighbour and is skipped.
constexpr int kBlkH = 4, kBlkW = 16;
// Search statistics, collected only when flags has DELORA_ICP_STATS (read with delora_icp_stats):
//  0 warps | 1 strips (warp level) | 2 cells per lane (warp level) | 3 warps entering the block search |
//  4 owners | 5 blocks tested | 6 blocks scanned | 7 max blocks scanned by one owner | 8 float64 re-rankings |
//  9 max blocks tested by one owner | 10 owners with > 256 blocks | 11 owners without any candidate so far |
//  16..23 warps by strip count {0, 1-2, 3-5, 6-10, 11-20, 21-40, 41-63, >= limit} | 24..31 cells per lane, same buckets
__device__ unsigned int g_dbg[32];
constexpr int kDefaultMaxStrips = 32; // window-growing steps before a lane is handed to the block-search kernel

constexpr int kExtThreads = 1024, kExtUnroll = 4;

// inclusive min / max scan of a[0..H) in place, forward (prefix) or backward (suffix); one warp.  min and max are
// exact, so the result does not depend on the order of the combination.
__device__ __forceinline__ void extent_scan(float2* __restrict__ a, int H, bool backward) {
    const int lane = threadIdx.x & 31;
    float2 carry = make_float2(3.0e38f, -3.0e38f);
    for (int r0 = 0; r0 < H; r0 += 32) {
        const int k = r0 + lane, r = backward ? H - 1 - k : k;
        float2 v = (k < H) ? __ldcg(a + r) : make_float2(3.0e38f, -3.0e38f);
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float ux = __shfl_up_sync(0xffffffffu, v.x, o), uy = __shfl_up_sync(0xffffffffu, v.y, o);
            if (lane >= o) { v.x = fminf(v.x, ux); v.y = fmaxf(v.y, uy); }
        }
        v.x = fminf(v.x, carry.x); v.y = fmaxf(v.y, carry.y);
        if (k < H) a[r] = v;
        carry.x = __shfl_sync(0xffffffffu, v.x, 31); carry.y = __shfl_sync(0xffffffffu, v.y, 31);
    }
}

// Pre-pass over the target grids: one CTA per (block row of kBlkH pixel rows, pair), each of the 32 warps takes every
// 32nd block of the row, kExtUnroll blocks at a time (8 independent 16-byte loads per lane): at W = 2048 a CTA issues
// all of its 128 KB at once.  The kernel is latency-bound, so it needs that many loads in flight.  The CTA writes its blocks and its
// rows' extents; the last CTA of a pair turns the row extents into the prefix / suffix extents and re-arms the counter.
// The window search is launched as this kernel's programmatic dependent: it may start once every CTA here has begun.
__global__ void __launch_bounds__(kExtThreads)
target_extents_kernel(const float4* __restrict__ grid, int H, int W, int nbh, int nbw, TargetExtents ext) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    constexpr int kWarps = kExtThreads / 32;
    __shared__ float s_lo[kWarps][kBlkH], s_hi[kWarps][kBlkH];
    __shared__ int is_last;
    const int br = blockIdx.x, b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float4* __restrict__ tg = grid + (size_t)b * H * W;
    float2* __restrict__ blk = ext.blk + (size_t)b * nbh * nbw;
    // lane's cells of a block: (row (lane >> 4) + 2 h, column lane & 15), h = 0, 1
    float rlo[2] = {3.0e38f, 3.0e38f}, rhi[2] = {-1.0f, -1.0f};
    for (int bc0 = warp; bc0 < nbw; bc0 += kWarps * kExtUnroll) {
        // all loads first (unconditional, at a clamped address), so that none waits behind a branch on another
        float4 t[kExtUnroll][2];
        bool in[kExtUnroll][2];
#pragma unroll
        for (int u = 0; u < kExtUnroll; ++u) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = lane + 32 * h;
                const int row = br * kBlkH + (c >> 4), col = (bc0 + u * kWarps) * kBlkW + (c & 15);
                in[u][h] = row < H && col < W;
                t[u][h] = __ldg(tg + (size_t)min(row, H - 1) * W + min(col, W - 1));
            }
        }
        float rr[kExtUnroll][2];                                   // |t|, or -1 for an empty / outside cell
#pragma unroll
        for (int u = 0; u < kExtUnroll; ++u) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float4 q = t[u][h];
                rr[u][h] = (in[u][h] && __float_as_int(q.w) >= 0) ? sqrtf(fmaf(q.z, q.z, fmaf(q.y, q.y, q.x * q.x)))
                                                                  : -1.0f;
            }
        }
#pragma unroll
        for (int u = 0; u < kExtUnroll; ++u) {
            const int bc = bc0 + u * kWarps;
            float lo = 3.0e38f, hi = -1.0f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (rr[u][h] >= 0.0f) {
                    lo = fminf(lo, rr[u][h]); hi = fmaxf(hi, rr[u][h]);
                    rlo[h] = fminf(rlo[h], rr[u][h]); rhi[h] = fmaxf(rhi[h], rr[u][h]);
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
                hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
            }
            if (lane == 0 && bc < nbw) blk[br * nbw + bc] = make_float2(lo * (1.0f - 1e-6f), hi * (1.0f + 1e-6f));
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
            rlo[h] = fminf(rlo[h], __shfl_xor_sync(0xffffffffu, rlo[h], o));
            rhi[h] = fmaxf(rhi[h], __shfl_xor_sync(0xffffffffu, rhi[h], o));
        }
        if ((lane & 15) == 0) { s_lo[warp][(lane >> 4) + 2 * h] = rlo[h]; s_hi[warp][(lane >> 4) + 2 * h] = rhi[h]; }
    }
    __syncthreads();
    if (threadIdx.x < kBlkH && br * kBlkH + (int)threadIdx.x < H) {
        float lo = s_lo[0][threadIdx.x], hi = s_hi[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < kWarps; ++w) { lo = fminf(lo, s_lo[w][threadIdx.x]); hi = fmaxf(hi, s_hi[w][threadIdx.x]); }
        const float2 e = make_float2(lo * (1.0f - 1e-6f), hi * (1.0f + 1e-6f));
        const size_t r = (size_t)b * H + br * kBlkH + threadIdx.x;
        ext.row_pre[r] = e;
        ext.row_suf[r] = e;
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(ext.counter + b, 1) == nbh - 1);
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    if (warp == 0) extent_scan(ext.row_pre + (size_t)b * H, H, false);
    if (warp == 1) extent_scan(ext.row_suf + (size_t)b * H, H, true);
    if (threadIdx.x == 0) ext.counter[b] = 0;
}

// Lower bound of |s - t|^2 (times 0.999, the fp32 / __sinf margin) over targets t whose range |t| lies in
// [rho.x, rho.y] and whose direction is at an angle theta from the source direction with sin^2(theta / 2) >= S:
//     |s - t|^2 = (r - rho)^2 + 4 r rho sin^2(theta / 2)
// is convex in rho with its minimum at rho = r (1 - 2 S), so the bound is its value there, clamped to the extent.
// Over all rho >= 0 the minimum is r^2 sin^2(theta): never weaker than the purely angular bound.
__device__ __forceinline__ float range_lb2(float r, float S, float2 rho) {
    const float rh = fminf(fmaxf(r * (1.0f - 2.0f * S), rho.x), rho.y);
    const float dr = r - rh;
    return fmaf(dr, dr, 4.0f * r * rh * S) * 0.999f;
}

// Lower bound of the distance from the source point (range r) to every target beyond a ROW border that is `dpx`
// pixels (of `rad_per_px` radians) of elevation away, when the rows beyond it have the range extent `rho`.
// Exactness: a target in those rows differs from the source direction by at least the elevation gap, so
// theta >= gap and sin^2(theta / 2) >= sin^2(gap / 2); the angular bound r sin(gap) is kept as a floor (the two are
// equal at rho = r, and taking the larger is safe against the rounding of either).  No valid target beyond: no bound.
// __sinf of the HALF angle: its absolute error (~2^-21.4) changes sin^2 by at most 2^-20.4 / (half angle) relative,
// which the 0.999 margin on the squared bound covers for half angles >= 7.2e-4 rad.  A row border is at least
// 1 - 2e-3 rows from the source direction, so this holds for row pitches down to 1.45e-3 rad (0.083 deg).
__device__ __forceinline__ float row_border_bound(float dpx, float rad_per_px, float r, float2 rho) {
    if (!(rho.y >= 0.0f)) return kInf;
    const float d = fminf(fmaxf(dpx * rad_per_px, 0.0f), kHalfPiF);
    const float sh = __sinf(0.5f * d);
    return fmaxf(r * __sinf(d), sqrtf(range_lb2(r, sh * sh, rho)));
}

// first / last pixel column of the (unwrapped) block column bc; bc in [-nbw, 2 nbw)
__device__ __forceinline__ int blk_u_lo(int bc, int nbw, int W) {
    const int k = (bc < 0) ? -1 : (bc >= nbw) ? 1 : 0;
    return (bc - k * nbw) * kBlkW + k * W;
}
__device__ __forceinline__ int blk_u_hi(int bc, int nbw, int W) {
    const int k = (bc < 0) ? -1 : (bc >= nbw) ? 1 : 0;
    return min((bc - k * nbw) * kBlkW + kBlkW - 1, W - 1) + k * W;
}

__device__ __forceinline__ void nn2_merge(NN2& a, float bm1, float bm2, int bj) {
    if (bj >= 0 && bj == a.j1) { a.m2 = fminf(a.m2, bm2); return; }     // the same cell seen twice is not a tie
    const bool take = (bm1 < a.m1) || (bm1 == a.m1 && bj >= 0 && (a.j1 < 0 || bj < a.j1));
    const float lose = take ? a.m1 : bm1;                   // the larger of the two minima
    a.m2 = fminf(fminf(a.m2, bm2), (bj >= 0 && a.j1 >= 0) ? lose : kInf);
    if (take) { a.m1 = bm1; a.j1 = bj; }
}

// Per-lane source state shared by the two kernels: the transformed source point, its re-projection and
// the centre cell of its search window.
struct SrcLane {
    float4 p, m;                       // source point / normal before the transform
    float sx, sy, sz, nsx, nsy, nsz;   // after the transform
    float us, vs, r, rxy;
    int rc, cc;
    bool active;
};

__device__ __forceinline__ SrcLane load_src_lane(const float4* __restrict__ src_grid, const float4* __restrict__ src_ngrid,
                                                 const float* __restrict__ T, int b, int i, int HW, const GridParams& g) {
    SrcLane s;
    s.p = make_float4(0.f, 0.f, 0.f, 0.f);
    s.m = s.p;
    s.active = false;
    if (i < HW) {
        s.p = __ldg(src_grid + (size_t)b * HW + i);
        s.active = __float_as_int(s.p.w) >= 0;
        if (s.active) s.m = __ldg(src_ngrid + (size_t)b * HW + i);
    }
    s.sx = s.sy = s.sz = s.nsx = s.nsy = s.nsz = 0.f;
    if (s.active) {
        const Rigid rt = load_rigid(T + (size_t)b * 12);
        apply_rigid(rt, s.p, s.m, s.sx, s.sy, s.sz, s.nsx, s.nsy, s.nsz);
    }
    s.us = 0.f; s.vs = 0.f;
    pixel_coords(g, s.sx, s.sy, s.sz, s.us, s.vs);
    if (!(s.us == s.us)) s.us = 0.0f;
    if (!(s.vs == s.vs)) s.vs = 0.0f;
    s.rxy = sqrtf(fmaf(s.sx, s.sx, s.sy * s.sy));
    s.r = sqrtf(fmaf(s.sz, s.sz, fmaf(s.sx, s.sx, s.sy * s.sy)));
    s.cc = (int)fminf(fmaxf(rintf(s.us), 0.0f), g.wm1);
    s.rc = (int)fminf(fmaxf(rintf(s.vs), 0.0f), g.hm1);
    return s;
}

// Exactness bound of the window's lower (DOWN) or upper row border, `e` rows from the lane's centre row rc; `f` is the
// distance (px) from the source direction to that border of the centre cell.  Angular + range bound over the rows
// beyond (row_border_bound; prefix extents below, suffix extents above); no row beyond: no bound.
template <bool DOWN>
__device__ __forceinline__ float window_row_bound(int e, int rc, int H, float f, float dv_rad, float r,
                                                  const float2* __restrict__ row_pre,
                                                  const float2* __restrict__ row_suf) {
    const bool open = DOWN ? rc - e > 0 : rc + e < H - 1;
    return open ? row_border_bound(f + (float)e, dv_rad, r, __ldg(DOWN ? row_pre + rc - e - 1 : row_suf + rc + e + 1))
                : kInf;
}

// Exactness bounds of the window's left and right column borders, e_lf / e_rt columns from the lane's centre column
// cc (f_lf, f_rt as for window_row_bound); angular only.  A window as wide as the grid has no column border, and a
// border at or beyond the +-180 deg seam is seam_px closer than its unwrapped pixel distance.
__device__ __forceinline__ void window_col_bounds(int e_lf, int e_rt, int cc, int W, float f_lf, float f_rt, float rxy,
                                                  const GridParams& g, float& b_lf, float& b_rt) {
    const bool full_w = e_lf + e_rt + 1 >= W;
    b_lf = full_w ? kInf : border_bound(f_lf + (float)e_lf - (cc - e_lf <= 0 ? g.seam_px : 0.0f), g.du_rad, rxy);
    b_rt = full_w ? kInf : border_bound(f_rt + (float)e_rt - (cc + e_rt >= W - 1 ? g.seam_px : 0.0f), g.du_rad, rxy);
}

// ---------------------------------------------------------------------------------------------
// Kernel 1: window search for everybody; the (few) lanes whose exactness guard still fails after
// `max_strips` steps are handed to kernel 2 and contribute nothing to their warp's partial row here.
// Why two kernels: those lanes are the far-ground points lying between two LiDAR rings of the other
// scan (NN distance ~ half the ring spacing, metres) and depth discontinuities; ~2-5 % of the warps,
// but each needs thousands of cells or a serial per-lane block search, and as stragglers inside this
// kernel they would set its duration.
// IDS (delora_icp_dense_information): every source pixel also writes its kept NN to nn_ids [B, H*W] (kept_nn); the
// lanes handed to kernel 2 write -1 here and their NN there.  Without IDS, nn_ids is not read.
template <bool PO2PO, bool STATS, bool IDS = false>
__global__ void __launch_bounds__(kDenseThreads, 8)
icp_dense_kernel(const float4* __restrict__ src_grid, const float4* __restrict__ src_ngrid,
                 const float* __restrict__ T, const float4* __restrict__ tgt_grid,
                 const float4* __restrict__ tgt_ngrid, int max_strips, GridParams g, uint32_t flags,
                 float* __restrict__ partial_rows, int rows_per_pair, PendingList pend, TargetExtents ext,
                 int* __restrict__ nn_ids) {
    const int b = blockIdx.y;
    const int H = g.H, W = g.W, HW = H * W;
    const float4* __restrict__ tg = tgt_grid + (size_t)b * HW;
    const float4* __restrict__ tn = tgt_ngrid + (size_t)b * HW;
    const int i = blockIdx.x * kDenseThreads + threadIdx.x;
    const int warp_in_pair = i >> 5;
    const int lane = threadIdx.x & 31;

    const SrcLane s = load_src_lane(src_grid, src_ngrid, T, b, i, HW, g);
    const bool active = s.active;
    const bool any_active = __ballot_sync(0xffffffffu, active) != 0u;
    const float sx = s.sx, sy = s.sy, sz = s.sz;
    const float us = s.us, vs = s.vs, r = s.r, rxy = s.rxy;
    const int rc = s.rc, cc = s.cc;
    NN2 nn;
    nn.m1 = kInf; nn.m2 = kInf; nn.j1 = -1;
    // warp-uniform window extents around every lane's own (rc, cc); the 3 x 5 start window is
    // fully unrolled: 15 independent loads in flight
    int e_dn = 1, e_up = 1, e_lf = 2, e_rt = 2;
    if (any_active) {
        if (H >= 3 && W >= 5) {
            int col[5];
#pragma unroll
            for (int dc = -2; dc <= 2; ++dc) col[dc + 2] = wrap_col(cc + dc, W);
#pragma unroll
            for (int dr = -1; dr <= 1; ++dr) {
                const int row = rc + dr;
                const bool rok = active && row >= 0 && row < H;
                const int rbase = min(max(row, 0), H - 1) * W;          // always a valid address
#pragma unroll
                for (int dc = 0; dc < 5; ++dc)   // unsigned index: one IMAD.WIDE.U32 instead of a 4-instruction sign-extending LEA chain
                    nn2_eval(__ldg(tg + (unsigned)(rbase + col[dc])), rbase + col[dc], sx, sy, sz, nn, rok);
            }
        } else {
            e_dn = e_up = e_lf = e_rt = 0;
            nn2_eval(__ldg(tg + rc * W + cc), rc * W + cc, sx, sy, sz, nn, active);
        }
    }
    // Everything above reads only the source and target grids.  This kernel is the programmatic dependent of the
    // target-extents pre-pass: wait for that grid (and its writes) before the first bound.  Every thread waits, so
    // this grid never completes before the pre-pass has.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    int best_j = -1;
    if (any_active) {
        // distance (px) from the source direction to the four borders of its own centre cell
        const float f_dn = (vs - (float)rc) + 0.5f - kSlack, f_up = ((float)rc - vs) + 0.5f - kSlack;
        const float f_lf = (us - (float)cc) + 0.5f - kSlack, f_rt = ((float)cc - us) + 0.5f - kSlack;
        const float2* __restrict__ row_pre = ext.row_pre + (size_t)b * H;
        const float2* __restrict__ row_suf = ext.row_suf + (size_t)b * H;
        float b_dn = window_row_bound<true>(e_dn, rc, H, f_dn, g.dv_rad, r, row_pre, row_suf);
        float b_up = window_row_bound<false>(e_up, rc, H, f_up, g.dv_rad, r, row_pre, row_suf);
        float b_lf, b_rt;
        window_col_bounds(e_lf, e_rt, cc, W, f_lf, f_rt, rxy, g, b_lf, b_rt);
        unsigned pending = 0u;                                   // lanes that still fail after max_strips steps
        int n_strips = 0, n_cells = 15;
        for (int strip = 0;; ++strip) {
            const float bmin = fminf(fminf(b_dn, b_up), fminf(b_lf, b_rt));
            const bool done = !active || bmin >= kInf ||
                              (nn.j1 >= 0 && sqrtf(nn.m1) * 1.00001f <= bmin * 0.9995f);
            const unsigned failing = __ballot_sync(0xffffffffu, !done);
            if (failing == 0u) break;
            if (strip >= max_strips) { pending = failing; break; }
            if (STATS) n_strips = strip + 1;
            const int my_side = (bmin == b_dn) ? 0 : (bmin == b_up) ? 1 : (bmin == b_lf) ? 2 : 3;
            const int side = __shfl_sync(0xffffffffu, my_side, __ffs(failing) - 1);
            if (side < 2) {
                const int row = (side == 0) ? rc - (++e_dn) : rc + (++e_up);
                const bool rok = active && row >= 0 && row < H;
                const int rbase = min(max(row, 0), H - 1) * W;
                const int n = e_lf + e_rt + 1;
                if (STATS) n_cells += n;
                int col = wrap_col(cc - e_lf, W);
                // n is odd and >= 5 on grids at least 5 wide (the window starts 5 wide and grows by 2): a first batch
                // of 5 independent loads, then batches of 4 and at most one of 2 -- no generic remainder loop
                int k = 0;
                if (n >= 5) {
                    int cols[5];
#pragma unroll
                    for (int j = 0; j < 5; ++j) { cols[j] = col; ++col; col = (col == W) ? 0 : col; }
#pragma unroll
                    for (int j = 0; j < 5; ++j)
                        nn2_eval(__ldg(tg + (unsigned)(rbase + cols[j])), rbase + cols[j], sx, sy, sz, nn, rok);
                    k = 5;
                }
                for (; k + 4 <= n; k += 4) {
                    int cols[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) { cols[j] = col; ++col; col = (col == W) ? 0 : col; }
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        nn2_eval(__ldg(tg + (unsigned)(rbase + cols[j])), rbase + cols[j], sx, sy, sz, nn, rok);
                }
                for (; k < n; ++k) {
                    nn2_eval(__ldg(tg + (unsigned)(rbase + col)), rbase + col, sx, sy, sz, nn, rok);
                    ++col;
                    col = (col == W) ? 0 : col;
                }
                if (side == 0)
                    b_dn = window_row_bound<true>(e_dn, rc, H, f_dn, g.dv_rad, r, row_pre, row_suf);
                else
                    b_up = window_row_bound<false>(e_up, rc, H, f_up, g.dv_rad, r, row_pre, row_suf);
            } else {
                const int step = min(2, W - (e_lf + e_rt + 1));
                const int c0 = wrap_col((side == 2) ? cc - e_lf - 1 : cc + e_rt + 1, W);
                const int c1 = wrap_col((side == 2) ? cc - e_lf - 2 : cc + e_rt + 2, W);
                const int n = e_dn + e_up + 1;
                if (STATS) n_cells += 2 * n;
                const bool two = (step == 2);
#pragma unroll 2
                for (int k = 0; k < n; ++k) {
                    const int row = rc - e_dn + k;
                    const bool rok = active && row >= 0 && row < H;
                    const int rbase = min(max(row, 0), H - 1) * W;
                    nn2_eval(__ldg(tg + (unsigned)(rbase + c0)), rbase + c0, sx, sy, sz, nn, rok);
                    nn2_eval(__ldg(tg + (unsigned)(rbase + c1)), rbase + c1, sx, sy, sz, nn, rok && two);
                }
                if (side == 2) e_lf += step; else e_rt += step;
                window_col_bounds(e_lf, e_rt, cc, W, f_lf, f_rt, rxy, g, b_lf, b_rt);
            }
        }
        if (STATS && lane == 0) {
            const int bucket = pending ? 7 : n_strips == 0 ? 0 : n_strips <= 2 ? 1 : n_strips <= 5 ? 2 : n_strips <= 10 ? 3
                             : n_strips <= 20 ? 4 : n_strips <= 40 ? 5 : 6;
            atomicAdd(&g_dbg[0], 1u); atomicAdd(&g_dbg[1], (unsigned)n_strips); atomicAdd(&g_dbg[2], (unsigned)n_cells);
            atomicAdd(&g_dbg[16 + bucket], 1u); atomicAdd(&g_dbg[24 + bucket], (unsigned)n_cells);
            if (pending) atomicAdd(&g_dbg[3], 1u);
        }
        if (pending) {
            // hand the unfinished lanes to kernel 2 (items and entries land in arbitrary order, but every item
            // owns its warp's partial row and adds to it in lane order, so the sums stay deterministic)
            int item = 0, first = 0;
            if (lane == 0) {
                item = atomicAdd(pend.counters, 1);
                first = atomicAdd(pend.counters + 2, __popc(pending));
                pend.items[item] = make_int4(b, warp_in_pair, (int)pending, first);
            }
            item = __shfl_sync(0xffffffffu, item, 0);
            first = __shfl_sync(0xffffffffu, first, 0);
            if ((pending >> lane) & 1u)
                pend.entries[first + __popc(pending & ((1u << lane) - 1u))] =
                    make_float4(nn.m1, nn.m2, __int_as_float(nn.j1), __int_as_float(item * 32 + lane));
        }
        best_j = ((pending >> lane) & 1u) ? -1 : nn.j1;
        if (active && best_j >= 0 && nn.m2 <= nn.m1 * (1.0f + kNNBand)) {
            if (STATS) atomicAdd(&g_dbg[8], 1u);
            best_j = nn_exact_rescan(tg, H, W, rc, cc, e_dn, e_up, e_lf, e_rt, sx, sy, sz, nn.m1 * (1.0f + kNNBand));
        }
    }
    if (IDS && i < HW)
        nn_ids[(size_t)b * HW + i] = kept_nn(active && best_j >= 0, PO2PO, s.nsx, s.nsy, s.nsz, tn, best_j);
    accumulate_warp_row<(PO2PO ? kIcpAcc : kColPo2po), false>(active && best_j >= 0, flags, s.p, s.m, sx, sy, sz, s.nsx,
                                                              s.nsy, s.nsz, tg, tn, best_j, nullptr, nullptr,
                                                              partial_rows, b, rows_per_pair, warp_in_pair);
}

struct OwnerGeom { float sx, sy, sz, us, vs, r, cos_es; };
struct BlockRect { int br_lo, bc_lo, nbc, nblk; };       // bc_lo unwrapped; nbc columns x (nblk / nbc) rows of blocks

// One pass of a warp over the blocks of `rect` for one source point: 32 blocks are bounded at a time (one per
// lane), the blocks whose lower bound does not exceed `bound` are scanned, 2 cells per lane.
//   EXACT = false: fp32 (smallest, second smallest) tracking in `loc`; `bound` tightens as candidates are found.
//   EXACT = true : `bound` is the fixed tie threshold; candidates inside it are ranked in float64 (ebest, ej).
// Returns the number of blocks scanned.
template <bool EXACT>
__device__ __forceinline__ int block_pass(const float4* __restrict__ tg, const float2* __restrict__ blk,
                                          const GridParams& g, int nbw, const OwnerGeom& o, const BlockRect& rect,
                                          float& bound, NN2& loc, double& ebest, int& ej) {
    const int H = g.H, W = g.W;
    const int lane = threadIdx.x & 31;
    int scanned = 0;
    for (int base = 0; base < rect.nblk; base += 32) {
        const int idx = base + lane;
        const bool in = idx < rect.nblk;
        const int br = rect.br_lo + (in ? idx / rect.nbc : 0);
        int bc = rect.bc_lo + (in ? idx % rect.nbc : 0);
        bc += (bc < 0) ? nbw : 0;
        bc -= (bc >= nbw) ? nbw : 0;
        bool ok = in;
        float lb2 = kInf;
        if (ok) {
            const float2 rg = __ldg(blk + br * nbw + bc);
            if (rg.y >= 0.0f) {
                const float v_lo = (float)(br * kBlkH) - 0.5f, v_hi = (float)min(br * kBlkH + kBlkH - 1, H - 1) + 0.5f;
                const float u_lo = (float)(bc * kBlkW) - 0.5f, u_hi = (float)min(bc * kBlkW + kBlkW - 1, W - 1) + 0.5f;
                const float gv = fmaxf(fmaxf(v_lo - o.vs, o.vs - v_hi) - kSlack, 0.0f) * g.dv_rad;
                // azimuth gap ON THE CIRCLE: the direct way, or the other way round through the seam
                const float d1 = u_lo - o.us, d2 = o.us - u_hi;
                const float gpx = fminf(fmaxf(fmaxf(d1, d2), 0.0f), g.circ_px + fminf(d1, d2));
                const float gu = fmaxf(gpx - kSlack, 0.0f) * g.du_rad;
                const float sv = __sinf(fminf(0.5f * gv, kHalfPiF)), su = __sinf(fminf(0.5f * gu, kHalfPiF));
                const float e_lo = g.vf0 + v_lo * g.dv_rad, e_hi = g.vf0 + v_hi * g.dv_rad;
                const float c_blk = fmaxf(fminf(__cosf(e_lo), __cosf(e_hi)), 0.0f);
                lb2 = range_lb2(o.r, fmaxf(sv * sv, o.cos_es * c_blk * su * su), rg);
            } else {
                ok = false;                                       // empty block
            }
        }
        unsigned need = __ballot_sync(0xffffffffu, ok && lb2 <= bound * 1.001f);
        scanned += __popc(need);
        while (need) {
            const int sel = __ffs(need) - 1;
            need &= need - 1;
            const int sbr = __shfl_sync(0xffffffffu, br, sel), sbc = __shfl_sync(0xffffffffu, bc, sel);
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2) {
                const int c = lane + 32 * h2;
                const int row = sbr * kBlkH + (c >> 4), col = sbc * kBlkW + (c & 15);
                const bool cok = row < H && col < W;
                const int j = min(row, H - 1) * W + min(col, W - 1);
                const float4 t = __ldg(tg + j);
                if (!EXACT) {
                    nn2_eval(t, j, o.sx, o.sy, o.sz, loc, cok);
                } else {
                    const float dx = o.sx - t.x, dy = o.sy - t.y, dz = o.sz - t.z;
                    const float d2f = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
                    if (cok && d2f <= bound) {
                        const double d2e = nn_d2_exact(o.sx, o.sy, o.sz, t.x, t.y, t.z);
                        if (d2e < ebest || (d2e == ebest && j < ej)) { ebest = d2e; ej = j; }
                    }
                }
            }
        }
        if (!EXACT) {   // tighten the running best with what this chunk found (prunes the following chunks harder)
            float wm = loc.m1;
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) wm = fminf(wm, __shfl_xor_sync(0xffffffffu, wm, s));
            bound = fminf(bound, wm);
        }
    }
    return scanned;
}

// rare path, kept out of line so that its float64 registers do not count against the search loop
__device__ __noinline__ int exact_rerank_warp(const float4* __restrict__ tg, const float2* __restrict__ blk,
                                              const GridParams& g, int nbw, const OwnerGeom& o, const BlockRect& rect,
                                              float thresh) {
    double ebest = 1.0e300;
    int ej = 0x7fffffff;
    NN2 unused;
    unused.m1 = unused.m2 = kInf; unused.j1 = -1;
    block_pass<true>(tg, blk, g, nbw, o, rect, thresh, unused, ebest, ej);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, ebest, s);
        const int oj = __shfl_xor_sync(0xffffffffu, ej, s);
        if (ob < ebest || (ob == ebest && oj < ej)) { ebest = ob; ej = oj; }
    }
    return ej;
}

// ---------------------------------------------------------------------------------------------
// Kernel 2: range-pruned block search for the lanes kernel 1 gave up on.  One WARP per entry (= one source
// point), no coupling between the warps of a CTA: the 32 lanes bound 32 blocks of the certifying rectangle at a
// time and scan the blocks that survive, 2 cells per lane.  The warp that finishes the LAST entry of an item
// (atomic count) adds the loss / gradient terms of all the item's entries to the partial row kernel 1 wrote
// for that warp, in lane order (whichever warp does it, the arithmetic is the same: deterministic).
// Persistent grid-stride over the entries; the last CTA re-arms the work list.
constexpr int kPendThreads = 256;

template <bool PO2PO, bool STATS, bool IDS = false>
__global__ void __launch_bounds__(kPendThreads, 4)
icp_dense_pending_kernel(const float4* __restrict__ src_grid, const float4* __restrict__ src_ngrid,
                         const float* __restrict__ T, const float4* __restrict__ tgt_grid,
                         const float4* __restrict__ tgt_ngrid, TargetExtents ext, int nbh, int nbw,
                         GridParams g, uint32_t flags, float* __restrict__ partial_rows, int rows_per_pair,
                         PendingList pend, int* __restrict__ nn_ids) {
    const int H = g.H, W = g.W, HW = H * W;
    const int lane = threadIdx.x & 31;
    const int warps_per_cta = (int)blockDim.x >> 5;
    const int gwarp = blockIdx.x * warps_per_cta + ((int)threadIdx.x >> 5), n_warps = gridDim.x * warps_per_cta;
    const int n_entries = *reinterpret_cast<volatile int*>(pend.counters + 2);
    for (int e = gwarp; e < n_entries; e += n_warps) {
        const float4 ent = __ldg(pend.entries + e);
        const int code = __float_as_int(ent.w), item = code >> 5, owner = code & 31;
        const int4 it = __ldg(pend.items + item);
        const int b = it.x, warp_in_pair = it.y;
        const unsigned pending = (unsigned)it.z;
        const float4* __restrict__ tg = tgt_grid + (size_t)b * HW;
        const float2* __restrict__ blk = ext.blk + (size_t)b * nbh * nbw;
        // every lane rebuilds the SAME source point (uniform addresses: broadcast loads)
        const SrcLane o = load_src_lane(src_grid, src_ngrid, T, b, warp_in_pair * 32 + owner, HW, g);
        const float osx = o.sx, osy = o.sy, osz = o.sz, orr = o.r, ous = o.us, ovs = o.vs, orxy = o.rxy;
        NN2 nn;                                                          // the window-search result so far
        nn.m1 = ent.x; nn.m2 = ent.y; nn.j1 = __float_as_int(ent.z);
        float obest = nn.m1;                                             // running best d^2 (fp32), warp-uniform
        const int obr = o.rc / kBlkH, obc = o.cc / kBlkW;
        const float cos_es = orr > 0.0f ? orxy / orr : 1.0f;
        NN2 loc;
        loc.m1 = kInf; loc.m2 = kInf; loc.j1 = -1;
        // Block rectangle that certifies the CURRENT best: grow it (warp-uniform scalar loops) until all
        // four borders are at least d0 away; the best can only shrink while the rectangle is scanned, so
        // one pass over its blocks is enough (no ring-by-ring dependency chain).
        const float obest0 = obest;
        const float d0 = (obest < kInf) ? sqrtf(obest) * (1.00001f / 0.9995f) : kInf;
        int br_lo = obr, br_hi = obr, bc_lo = obc, bc_hi = obc;            // bc_* unwrapped
        const float2* __restrict__ row_pre = ext.row_pre + (size_t)b * H;
        const float2* __restrict__ row_suf = ext.row_suf + (size_t)b * H;
        while (br_lo > 0 && row_border_bound(ovs - ((float)(br_lo * kBlkH) - 0.5f) - kSlack, g.dv_rad, orr,
                                             __ldg(row_pre + br_lo * kBlkH - 1)) < d0)
            --br_lo;
        while (br_hi < nbh - 1 && row_border_bound(((float)(br_hi * kBlkH + kBlkH - 1) + 0.5f) - ovs - kSlack, g.dv_rad,
                                                   orr, __ldg(row_suf + br_hi * kBlkH + kBlkH)) < d0)
            ++br_hi;
        // (unwrapped block columns: W need not be a multiple of kBlkW, so the pixel span of block column
        //  bc outside [0, nbw) is that of its wrapped twin shifted by +-W, not bc * kBlkW)
        while (bc_hi - bc_lo + 1 < nbw &&
               border_bound(ous - ((float)blk_u_lo(bc_lo, nbw, W) - 0.5f) - kSlack - (bc_lo <= 0 ? g.seam_px : 0.0f),
                            g.du_rad, orxy) < d0) --bc_lo;
        while (bc_hi - bc_lo + 1 < nbw &&
               border_bound(((float)blk_u_hi(bc_hi, nbw, W) + 0.5f) - ous - kSlack - (bc_hi >= nbw - 1 ? g.seam_px : 0.0f),
                            g.du_rad, orxy) < d0) ++bc_hi;
        const int nbc = bc_hi - bc_lo + 1, nblk = (br_hi - br_lo + 1) * nbc;
        const OwnerGeom og = {osx, osy, osz, ous, ovs, orr, cos_es};
        const BlockRect rect = {br_lo, bc_lo, nbc, nblk};
        double unused_d = 0.0;
        int unused_j = 0;
        const int dbg_scanned = block_pass<false>(tg, blk, g, nbw, og, rect, obest, loc, unused_d, unused_j);
        if (STATS && lane == 0) {
            atomicAdd(&g_dbg[4], 1u); atomicAdd(&g_dbg[5], (unsigned)nblk); atomicAdd(&g_dbg[6], (unsigned)dbg_scanned);
            atomicMax(&g_dbg[7], (unsigned)dbg_scanned);
            atomicMax(&g_dbg[9], (unsigned)nblk);
            if (nblk > 256) atomicAdd(&g_dbg[10], 1u);
            if (!(obest0 < kInf)) atomicAdd(&g_dbg[11], 1u);
        }
        // merge the 32 partial results, then into the window-search result
#pragma unroll
        for (int s2 = 16; s2 > 0; s2 >>= 1) {
            const float bm1 = __shfl_xor_sync(0xffffffffu, loc.m1, s2), bm2 = __shfl_xor_sync(0xffffffffu, loc.m2, s2);
            const int bj = __shfl_xor_sync(0xffffffffu, loc.j1, s2);
            nn2_merge(loc, bm1, bm2, bj);
        }
        NN2 fin = nn;
        nn2_merge(fin, loc.m1, loc.m2, loc.j1);
        const float fm1 = __shfl_sync(0xffffffffu, fin.m1, 0), fm2 = __shfl_sync(0xffffffffu, fin.m2, 0);
        int fj = __shfl_sync(0xffffffffu, fin.j1, 0);
        if (fj >= 0 && fm2 <= fm1 * (1.0f + kNNBand)) {
            // Two candidates inside the fp32 ambiguity band: float64 re-ranking (cKDTree's order) by the whole
            // warp, over the blocks of the certified rectangle whose lower bound reaches into the band (every
            // candidate of the band lies inside that rectangle: all cells outside it are farther than d0).
            if (STATS && lane == 0) atomicAdd(&g_dbg[8], 1u);
            const float thresh = fm1 * (1.0f + kNNBand);
            const int ej = exact_rerank_warp(tg, blk, g, nbw, og, rect, thresh);
            fj = (ej == 0x7fffffff) ? fj : ej;
        }
        // publish the result; the warp that completes the item does the item's accumulation
        int finisher = 0;
        if (lane == 0) {
            pend.result[e] = fj;
            __threadfence();
            finisher = (atomicAdd(pend.item_done + item, 1) == __popc(pending) - 1) ? 1 : 0;
        }
        finisher = __shfl_sync(0xffffffffu, finisher, 0);
        if (finisher) {
            __threadfence();
            const float4* __restrict__ tn = tgt_ngrid + (size_t)b * HW;
            const SrcLane s = load_src_lane(src_grid, src_ngrid, T, b, warp_in_pair * 32 + lane, HW, g);
            const bool mine = ((pending >> lane) & 1u) != 0u && s.active;
            const int best_j = mine ? __ldcg(pend.result + it.w + __popc(pending & ((1u << lane) - 1u))) : -1;
            if (IDS && ((pending >> lane) & 1u))
                nn_ids[(size_t)b * HW + warp_in_pair * 32 + lane] =
                    kept_nn(mine && best_j >= 0, PO2PO, s.nsx, s.nsy, s.nsz, tn, best_j);
            accumulate_warp_row<(PO2PO ? kIcpAcc : kColPo2po), true>(mine && best_j >= 0, flags, s.p, s.m, s.sx, s.sy,
                                                                     s.sz, s.nsx, s.nsy, s.nsz, tg, tn, best_j, nullptr,
                                                                     nullptr, partial_rows, b, rows_per_pair,
                                                                     warp_in_pair);
            if (lane == 0) pend.item_done[item] = 0;                    // re-arm
        }
    }
    // re-arm the work list: the last CTA to get here has seen every other CTA finish
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(pend.counters + 1, 1) == (int)gridDim.x - 1) {
            pend.counters[0] = 0;
            pend.counters[1] = 0;
            pend.counters[2] = 0;
            __threadfence();
        }
    }
}

// The window search of one (PO2PO, STATS, IDS) instantiation, as the programmatic dependent of target_extents_kernel
// (see griddepcontrol.wait in the kernel: its CTAs load their source lanes and start windows while the pre-pass is still
// running), then the block search of the lanes it hands over.
template <bool PO2PO, bool STATS, bool IDS = false>
int launch_dense_search(const float4* src_grid, const float4* src_ngrid, const float* T, const float4* tgt_grid,
                        const float4* tgt_ngrid, int B, int rows, int nbh, int nbw, int max_strips, const GridParams& g,
                        uint32_t flags, const IcpScratch& sc, int* nn_ids, cudaStream_t st) {
    const dim3 grid((g.H * g.W + kDenseThreads - 1) / kDenseThreads, B);
    const cudaError_t e = launch_pdl(icp_dense_kernel<PO2PO, STATS, IDS>, grid, dim3(kDenseThreads), st, src_grid,
                                     src_ngrid, T, tgt_grid, tgt_ngrid, max_strips, g, flags, sc.rows, rows, sc.pend,
                                     sc.ext, nn_ids);
    DELORA_CHECK_LAUNCH_RESULT(e, "icp_dense_kernel");
    // persistent block search: enough CTAs for one wave (up to 4 per SM), never more than there can be items
    const int pend_grid = (int)std::min<long long>(((long long)B * rows * 32 + 7) / 8, 4ll * num_sms());
    icp_dense_pending_kernel<PO2PO, STATS, IDS><<<pend_grid, kPendThreads, 0, st>>>(
        src_grid, src_ngrid, T, tgt_grid, tgt_ngrid, sc.ext, nbh, nbw, g, flags, sc.rows, rows, sc.pend, nn_ids);
    DELORA_CHECK_LAUNCH("icp_dense_pending_kernel");
    return 0;
}

}  // namespace delora

using namespace delora;

extern "C" int delora_icp_stats(uint32_t* out32, int reset) {
    if (out32) {
        const cudaError_t e = cudaMemcpyFromSymbol(out32, delora::g_dbg, 32 * sizeof(unsigned int));
        DELORA_CHECK_ARG(e == cudaSuccess, "delora_icp_stats: %s", cudaGetErrorString(e));
    }
    if (reset) {
        const unsigned int z[32] = {0};
        const cudaError_t e = cudaMemcpyToSymbol(delora::g_dbg, z, sizeof(z));
        DELORA_CHECK_ARG(e == cudaSuccess, "delora_icp_stats: %s", cudaGetErrorString(e));
    }
    return 0;
}

// delora_icp_dense_fwd_bwd (nn_ids NULL) and the search + finalize of delora_icp_dense_information (nn_ids [B, H*W]:
// the IDS instantiations, which the DELORA_ICP_STATS ones never are)
static int dense_icp(const delora_f4* src_grid, const delora_f4* src_ngrid, const float* T, const delora_f4* tgt_grid,
                     const delora_f4* tgt_ngrid, int B, int H, int W, double hfov0, double hfov1, double vfov0,
                     double vfov1, float lambda_po2pl, uint32_t flags, float* losses, float* grad_T, float* scratch,
                     int* nn_ids, cudaStream_t st, const char* who) {
    DELORA_CHECK_ARG(src_grid && src_ngrid && T && tgt_grid && tgt_ngrid && losses && grad_T && scratch,
                     "%s: null pointer", who);
    DELORA_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && W > 0 && (long long)H * W < (1ll << 31), "%s: bad shape", who);
    const IcpLayout L = icp_layout(B, H * W);
    const int nbh = (H + kBlkH - 1) / kBlkH, nbw = (W + kBlkW - 1) / kBlkW;
    DELORA_CHECK_ARG((int64_t)nbh * nbw <= L.blk_per_pair,
                     "%s: H=%d W=%d needs %lld range-pyramid blocks per pair, the scratch holds %lld",
                     who, H, W, (long long)nbh * nbw, (long long)L.blk_per_pair);
    const GridParams g = make_grid(H, W, hfov0, hfov1, vfov0, vfov1, 1);
    const IcpScratch sc = icp_scratch(scratch, L);
    int max_strips = kDefaultMaxStrips;
    if (const char* e = getenv("DELORA_ICP_MAX_STRIPS")) max_strips = atoi(e);      // tuning knob (tests / profiling)
    target_extents_kernel<<<dim3(nbh, B), kExtThreads, 0, st>>>((const float4*)tgt_grid, H, W, nbh, nbw, sc.ext);
    DELORA_CHECK_LAUNCH("target_extents_kernel");
    using DenseSearch = decltype(&launch_dense_search<false, false>);
    constexpr DenseSearch kSearch[2][3] = {
        {launch_dense_search<false, false>, launch_dense_search<false, true>, launch_dense_search<false, false, true>},
        {launch_dense_search<true, false>, launch_dense_search<true, true>, launch_dense_search<true, false, true>}};
    const int variant = nn_ids ? 2 : (flags & DELORA_ICP_STATS) != 0u ? 1 : 0;
    const int rc = kSearch[(flags & DELORA_LOSS_PO2PO) != 0u][variant](
        (const float4*)src_grid, (const float4*)src_ngrid, T, (const float4*)tgt_grid, (const float4*)tgt_ngrid, B,
        L.rows, nbh, nbw, max_strips, g, flags, sc, nn_ids, st);
    if (rc != 0) return rc;
    return launch_icp_finalize(sc, B, L.rows, lambda_po2pl, losses, grad_T, st);
}

extern "C" int delora_icp_dense_fwd_bwd(const delora_f4* src_grid, const delora_f4* src_ngrid, const float* T,
                                        const delora_f4* tgt_grid, const delora_f4* tgt_ngrid, int B, int H, int W,
                                        double hfov0, double hfov1, double vfov0, double vfov1, float lambda_po2pl,
                                        uint32_t flags, float* losses, float* grad_T, float* scratch, void* stream) {
    return dense_icp(src_grid, src_ngrid, T, tgt_grid, tgt_ngrid, B, H, W, hfov0, hfov1, vfov0, vfov1, lambda_po2pl,
                     flags, losses, grad_T, scratch, nullptr, (cudaStream_t)stream, "delora_icp_dense_fwd_bwd");
}

extern "C" int64_t delora_icp_information_scratch_floats(int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0 || (long long)H * W >= (1ll << 31)) return -1;
    return icp_info_layout(B, H * W).total;
}

// delora_icp_dense_information (factor NULL) and delora_icp_dense_information_scaled
static int dense_information(const delora_f4* src_grid, const delora_f4* src_ngrid, const float* T,
                             const delora_f4* tgt_grid, const delora_f4* tgt_ngrid, int B, int H, int W, double hfov0,
                             double hfov1, double vfov0, double vfov1, float lambda_po2pl, uint32_t flags, float* losses,
                             float* grad_T, float* scratch, float* info, float* info_scratch, const float* factor,
                             cudaStream_t st, const char* who) {
    DELORA_CHECK_ARG(info && info_scratch, "%s: null pointer", who);
    DELORA_CHECK_ARG((flags & DELORA_ICP_STATS) == 0u, "%s: DELORA_ICP_STATS is not counted here", who);
    int* nn_ids = reinterpret_cast<int*>(info_scratch);
    const int rc = dense_icp(src_grid, src_ngrid, T, tgt_grid, tgt_ngrid, B, H, W, hfov0, hfov1, vfov0, vfov1,
                             lambda_po2pl, flags, losses, grad_T, scratch, nn_ids, st, who);
    if (rc != 0) return rc;
    return launch_icp_information((const float4*)src_grid, (const float4*)src_ngrid, T, (const float4*)tgt_ngrid, B, H * W, lambda_po2pl, flags, losses, info_scratch, info,
                                  factor, st);
}

extern "C" int delora_icp_dense_information(const delora_f4* src_grid, const delora_f4* src_ngrid, const float* T,
                                            const delora_f4* tgt_grid, const delora_f4* tgt_ngrid, int B, int H, int W,
                                            double hfov0, double hfov1, double vfov0, double vfov1, float lambda_po2pl,
                                            uint32_t flags, float* losses, float* grad_T, float* scratch, float* info,
                                            float* info_scratch, void* stream) {
    return dense_information(src_grid, src_ngrid, T, tgt_grid, tgt_ngrid, B, H, W, hfov0, hfov1, vfov0, vfov1,
                             lambda_po2pl, flags, losses, grad_T, scratch, info, info_scratch, nullptr,
                             (cudaStream_t)stream, "delora_icp_dense_information");
}

extern "C" int delora_icp_dense_information_scaled(const delora_f4* src_grid, const delora_f4* src_ngrid,
                                                   const float* T, const delora_f4* tgt_grid,
                                                   const delora_f4* tgt_ngrid, int B, int H, int W, double hfov0,
                                                   double hfov1, double vfov0, double vfov1, float lambda_po2pl,
                                                   uint32_t flags, float* losses, float* grad_T, float* scratch,
                                                   float* info, float* info_scratch, const float* factor,
                                                   void* stream) {
    const char* who = "delora_icp_dense_information_scaled";
    DELORA_CHECK_ARG(factor, "%s: null factor", who);
    return dense_information(src_grid, src_ngrid, T, tgt_grid, tgt_ngrid, B, H, W, hfov0, hfov1, vfov0, vfov1,
                             lambda_po2pl, flags, losses, grad_T, scratch, info, info_scratch, factor,
                             (cudaStream_t)stream, who);
}
