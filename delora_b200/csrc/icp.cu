// Fused SE(3) transform + exact nearest neighbour + ICP losses, forward and backward (sm_90a).
//
// Replaces, per scan pair (reference paths relative to its root):
//   Deployer.transform/rotate_point_cloud_transformation_matrix   src/deploy/deployer.py:181-189
//   ICPLosses.forward (cKDTree build + 2 queries + masking)        src/losses/icp_losses.py:28-158
//   KDPointToPlaneLoss :196-206, KDPlaneToPlaneLoss :224-240, KDPointToPointLoss :168-179
//   and the autograd backward of all of it down to the 3x4 transform (SURVEY.md §3.4).
//
// Nearest neighbour: the reference asks scipy's cKDTree for the exact Euclidean NN in float64.
// Here the target list is indexed by its spherical cell (CSR over the H x W range-image grid);
// a source point searches a window of cells around its own re-projection and the result is
// PROVEN exact by a geometric guard: every unsearched target lies beyond one of the window's
// four borders (two half-planes of constant azimuth, two cones of constant elevation), so it is
// at least  min(r_xy*sin(d_az), r*sin(d_el))  away; if the best distance found is below that
// bound the window result is the global NN, otherwise the window grows strip by strip on its weakest side (up to the whole grid).
// Candidates are pre-filtered in fp32 and ranked in fp64 (ties: lowest tag), like cKDTree.
#include "icp_common.cuh"

namespace delora {

constexpr int kIcpThreads = 256;

__device__ __forceinline__ void nn_scan_range(const float4* __restrict__ tp, int j0, int j1, float sx, float sy,
                                              float sz, NNBest& best) {
    for (int j = j0; j < j1; ++j) nn_eval(__ldg(tp + j), j, sx, sy, sz, best);
}

// scan the cells [c0, c1] (unwrapped column indices, c1 - c0 + 1 <= W) of one grid row
__device__ __forceinline__ void nn_scan_cols(const float4* __restrict__ tp, const int32_t* __restrict__ crow, int W,
                                             int c0, int c1, float sx, float sy, float sz, NNBest& best) {
    // bring c0 into [0, W); the span may then run past W (wraps around the seam)
    if (c0 < 0) { c0 += W; c1 += W; }
    else if (c0 >= W) { c0 -= W; c1 -= W; }
    if (c1 < W) {
        nn_scan_range(tp, crow[c0], crow[c1 + 1], sx, sy, sz, best);
    } else {
        nn_scan_range(tp, crow[c0], crow[W], sx, sy, sz, best);
        nn_scan_range(tp, crow[0], crow[c1 - W + 1], sx, sy, sz, best);
    }
}

// Exact NN of (sx,sy,sz) among the cell-sorted targets of one scan.
//
// The window [r_lo, r_hi] x [c_lo, c_hi] grows one strip at a time on the side whose exactness
// bound is currently the smallest, scanning only the new strip, until the best distance found is
// below all four bounds (or the window is the whole grid).  Every cell is visited at most once.
__device__ __forceinline__ NNBest nn_search(const GridParams& g, const float4* __restrict__ tp,
                                            const int32_t* __restrict__ cs, float sx, float sy, float sz) {
    NNBest best;
    nn_init(best);
    const int H = g.H, W = g.W;
    if (cs[(size_t)H * W] == 0) return best;
    float us, vs;
    pixel_coords(g, sx, sy, sz, us, vs);
    if (!(us == us)) us = 0.0f;                       // NaN input: degenerate, ends in the exhaustive search
    if (!(vs == vs)) vs = 0.0f;
    const float rxy = sqrtf(fmaf(sx, sx, sy * sy));
    const float r = sqrtf(fmaf(sz, sz, fmaf(sx, sx, sy * sy)));
    const int cc = (int)fminf(fmaxf(rintf(us), 0.0f), g.wm1);
    const int rc = (int)fminf(fmaxf(rintf(vs), 0.0f), g.hm1);
    constexpr int kColStep = 2;
    int r_lo = max(rc - 1, 0), r_hi = min(rc + 1, H - 1);
    int c_lo = cc - min(2, (W - 1) / 2), c_hi = cc + min(2, (W - 1) / 2);     // unwrapped; width <= W
    for (int row = r_lo; row <= r_hi; ++row) nn_scan_cols(tp, cs + (size_t)row * W, W, c_lo, c_hi, sx, sy, sz, best);
    while (true) {
        // exactness bounds of the four borders (pixel units -> radians; 2e-3 px of slack covers the
        // fp32 error of the binning): unsearched targets beyond a border are at least this far away
        const float kInf = 3.0e38f;
        float b_dn = kInf, b_up = kInf, b_lf = kInf, b_rt = kInf;
        if (r_lo > 0) {
            const float d = (vs - ((float)r_lo - 0.5f) - 2e-3f) * g.dv_rad;
            b_dn = d <= 0.0f ? 0.0f : r * __sinf(fminf(d, kHalfPiF));
        }
        if (r_hi < H - 1) {
            const float d = (((float)r_hi + 0.5f) - vs - 2e-3f) * g.dv_rad;
            b_up = d <= 0.0f ? 0.0f : r * __sinf(fminf(d, kHalfPiF));
        }
        const int width = c_hi - c_lo + 1;
        if (width < W) {
            // a border at or beyond the seam: see GridParams::seam_px
            const float dl = (us - ((float)c_lo - 0.5f) - 2e-3f - (c_lo <= 0 ? g.seam_px : 0.0f)) * g.du_rad;
            const float dr = (((float)c_hi + 0.5f) - us - 2e-3f - (c_hi >= W - 1 ? g.seam_px : 0.0f)) * g.du_rad;
            b_lf = dl <= 0.0f ? 0.0f : rxy * __sinf(fminf(dl, kHalfPiF));
            b_rt = dr <= 0.0f ? 0.0f : rxy * __sinf(fminf(dr, kHalfPiF));
        }
        const float bmin = fminf(fminf(b_dn, b_up), fminf(b_lf, b_rt));
        if (bmin >= kInf) break;                                           // the window is the whole grid
        if (best.pos >= 0 && nn_best_dist_ub(best) <= bmin * 0.9995f) break;
        if (bmin == b_dn) {
            --r_lo;
            nn_scan_cols(tp, cs + (size_t)r_lo * W, W, c_lo, c_hi, sx, sy, sz, best);
        } else if (bmin == b_up) {
            ++r_hi;
            nn_scan_cols(tp, cs + (size_t)r_hi * W, W, c_lo, c_hi, sx, sy, sz, best);
        } else if (bmin == b_lf) {
            const int step = min(kColStep, W - width);
            for (int row = r_lo; row <= r_hi; ++row)
                nn_scan_cols(tp, cs + (size_t)row * W, W, c_lo - step, c_lo - 1, sx, sy, sz, best);
            c_lo -= step;
        } else {
            const int step = min(kColStep, W - width);
            for (int row = r_lo; row <= r_hi; ++row)
                nn_scan_cols(tp, cs + (size_t)row * W, W, c_hi + 1, c_hi + step, sx, sy, sz, best);
            c_hi += step;
        }
    }
    return best;
}

template <bool HAS_T>
__global__ void __launch_bounds__(kIcpThreads)
icp_kernel(const float4* __restrict__ src_pts4, const float4* __restrict__ src_nrm4, const int32_t* __restrict__ n_src,
           int src_stride, const float* __restrict__ T, const float4* __restrict__ tgt_pts4,
           const float4* __restrict__ tgt_nrm4, const int32_t* __restrict__ cell_start, int tgt_stride, GridParams g,
           uint32_t flags, int32_t* __restrict__ nn_index, float4* __restrict__ point_dir,
           float4* __restrict__ normal_dir, float* __restrict__ partial_rows, int rows_per_pair) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * kIcpThreads + threadIdx.x;
    const bool active = i < n_src[b];
    const float4* __restrict__ tp = tgt_pts4 + (size_t)b * tgt_stride;
    const float4* __restrict__ tn = tgt_nrm4 + (size_t)b * tgt_stride;
    const int32_t* __restrict__ cs = cell_start + (size_t)b * ((size_t)g.H * g.W + 1);

    float4 p = make_float4(0.f, 0.f, 0.f, 0.f), m = p;
    float sx = 0.f, sy = 0.f, sz = 0.f, nsx = 0.f, nsy = 0.f, nsz = 0.f;
    int pos = -1;
    if (active) {
        p = __ldg(src_pts4 + (size_t)b * src_stride + i);
        m = __ldg(src_nrm4 + (size_t)b * src_stride + i);
        if (HAS_T) {
            const Rigid rt = load_rigid(T + (size_t)b * 12);
            apply_rigid(rt, p, m, sx, sy, sz, nsx, nsy, nsz);
        } else {
            sx = p.x; sy = p.y; sz = p.z; nsx = m.x; nsy = m.y; nsz = m.z;
        }
        const NNBest best = nn_search(g, tp, cs, sx, sy, sz);
        if (nn_index) nn_index[(size_t)b * src_stride + i] = best.pos >= 0 ? best.tag : -1;
        pos = best.pos;
    }
    // the accumulators only come alive after the search (keeps the search loop's register set small)
    const size_t k = (size_t)b * src_stride + i;
    accumulate_warp_row<kIcpAcc, false>(pos >= 0, flags, p, m, sx, sy, sz, nsx, nsy, nsz, tp, tn, pos,
                                        active && point_dir ? point_dir + k : nullptr,
                                        active && normal_dir ? normal_dir + k : nullptr,
                                        partial_rows, b, rows_per_pair, (blockIdx.x * kIcpThreads + threadIdx.x) >> 5);
}

// Column sums of the per-warp partial rows: one block per (group of 8 columns, pair).  Thread t reads the group's
// 32 contiguous bytes of rows t, t + 256, ... (every sector fetched once, by one block) and keeps 8 fp64 sums; each
// column is then reduced by the same fixed-order tree (deterministic).  The last block of a pair to finish turns the
// 40 sums into the means and the 3x4 gradient and re-arms the pair's counter.
constexpr int kFinCols = 8, kFinGroups = DELORA_ICP_PARTIAL / kFinCols;
static_assert(DELORA_ICP_PARTIAL % kFinCols == 0, "partial rows are whole column groups");

__global__ void __launch_bounds__(256)
icp_finalize_kernel(const float* __restrict__ rows, int rows_per_pair, float* __restrict__ colsum,
                    int* __restrict__ counter, float lambda_po2pl, float* __restrict__ losses,
                    float* __restrict__ grad_T) {
    __shared__ double red[kFinCols][256];
    __shared__ float s[DELORA_ICP_PARTIAL];
    __shared__ int is_last;
    const int c0 = blockIdx.x * kFinCols, b = blockIdx.y;
    const float* __restrict__ p = rows + (size_t)b * rows_per_pair * DELORA_ICP_PARTIAL + c0;
    double a[kFinCols];
#pragma unroll
    for (int k = 0; k < kFinCols; ++k) a[k] = 0.0;
    for (int r = threadIdx.x; r < rows_per_pair; r += 256) {
        const float* __restrict__ q = p + (size_t)r * DELORA_ICP_PARTIAL;
#pragma unroll
        for (int k = 0; k < kFinCols; ++k) a[k] += (double)q[k];
    }
#pragma unroll
    for (int k = 0; k < kFinCols; ++k) red[k][threadIdx.x] = a[k];
    __syncthreads();
#pragma unroll
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
#pragma unroll
            for (int k = 0; k < kFinCols; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x < kFinCols) {
        colsum[(size_t)b * DELORA_ICP_PARTIAL + c0 + threadIdx.x] = (float)red[threadIdx.x][0];
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int prev = atomicAdd(counter + b, 1);
        is_last = (prev == kFinGroups - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    if (threadIdx.x < DELORA_ICP_PARTIAL) s[threadIdx.x] = __ldcg(colsum + (size_t)b * DELORA_ICP_PARTIAL + threadIdx.x);
    if (threadIdx.x == 0) counter[b] = 0;
    __syncthreads();
    const float M = s[kColM], Mp = s[kColMp];
    const float inv_m = M > 0.0f ? 1.0f / M : 0.0f;              // torch's mean over an empty set is NaN; we return 0
    const float inv_mp = Mp > 0.0f ? 1.0f / (3.0f * Mp) : 0.0f;  // MSE over 3*M' coordinates (icp_losses.py:169)
    if (threadIdx.x == 0) {
        float* __restrict__ o = losses + (size_t)b * DELORA_LOSS_ROW;
        o[kLossPo2po] = s[kColD2] * inv_mp;
        o[kLossPo2pl] = s[kColR2] * inv_m;
        o[kLossPl2pl] = s[kColPl2pl] * inv_m;
        o[kLossM] = M;
        o[kLossMp] = Mp;
        for (int k = kLossMp + 1; k < DELORA_LOSS_ROW; ++k) o[k] = 0.f;
    }
    if (threadIdx.x < 12) {
        const int row = threadIdx.x / 4, col = threadIdx.x % 4;
        float gval;
        const float k_pl = 2.0f * lambda_po2pl * inv_m, k_nn = 2.0f * inv_m, k_pp = 2.0f * inv_mp;
        if (col < 3) {
            gval = k_pl * s[kColRnP + row * 3 + col] + k_nn * s[kColGnM + row * 3 + col] +
                   k_pp * s[kColDP + row * 3 + col];
        } else {
            gval = k_pl * s[kColRn + row] + k_pp * s[kColD + row];
        }
        grad_T[(size_t)b * 12 + threadIdx.x] = gval;
    }
}

int launch_icp_finalize(const IcpScratch& sc, int B, int rows, float lambda_po2pl, float* losses, float* grad_T,
                        cudaStream_t st) {
    dim3 grid(kFinGroups, B);
    icp_finalize_kernel<<<grid, 256, 0, st>>>(sc.rows, rows, sc.colsum, sc.counter, lambda_po2pl, losses, grad_T);
    DELORA_CHECK_LAUNCH("icp_finalize_kernel");
    return 0;
}

// Per-point gradients for the drop-in autograd path (ICPLosses.forward takes already-transformed
// clouds and PyTorch back-propagates into them):  grad_pts = g_po2pl * 2/M * r n_t (+ po2po),
// grad_nrm = g_pl2pl * 2/M * g_n.   Outputs channels-first [B,3,stride] like the reference tensors.
__global__ void __launch_bounds__(256)
icp_point_grads_kernel(const float4* __restrict__ point_dir, const float4* __restrict__ normal_dir,
                       const int32_t* __restrict__ n_src, int src_stride, const float* __restrict__ losses,
                       const float* __restrict__ upstream, float* __restrict__ grad_pts,
                       float* __restrict__ grad_nrm) {
    const int b = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
    if (i >= src_stride) return;
    float gx = 0.f, gy = 0.f, gz = 0.f, hx = 0.f, hy = 0.f, hz = 0.f;
    if (i < n_src[b]) {
        const float M = losses[(size_t)b * DELORA_LOSS_ROW + kLossM], Mp = losses[(size_t)b * DELORA_LOSS_ROW + kLossMp];
        const float g_po2po = upstream[b * 3 + 0], g_po2pl = upstream[b * 3 + 1], g_pl2pl = upstream[b * 3 + 2];
        const float4 pd = point_dir[(size_t)b * src_stride + i];
        const float4 nd = normal_dir[(size_t)b * src_stride + i];
        if (pd.w == 1.0f) {
            const float k = M > 0.f ? 2.0f * g_po2pl / M : 0.f;
            gx = k * pd.x; gy = k * pd.y; gz = k * pd.z;
            const float kn = M > 0.f ? 2.0f * g_pl2pl / M : 0.f;
            hx = kn * nd.x; hy = kn * nd.y; hz = kn * nd.z;
        } else if (pd.w == 2.0f) {
            const float k = Mp > 0.f ? 2.0f * g_po2po / (3.0f * Mp) : 0.f;
            gx = k * pd.x; gy = k * pd.y; gz = k * pd.z;
        }
    }
    float* __restrict__ gp = grad_pts + (size_t)b * 3 * src_stride + i;
    float* __restrict__ gn = grad_nrm + (size_t)b * 3 * src_stride + i;
    gp[0] = gx; gp[src_stride] = gy; gp[2 * (size_t)src_stride] = gz;
    gn[0] = hx; gn[src_stride] = hy; gn[2 * (size_t)src_stride] = hz;
}

// quaternion + translation -> 4x4 (quat_to_T_row, common.cuh); one thread per batch element.
__global__ void quat_to_T_kernel(const float* __restrict__ quat, const float* __restrict__ trans, int B,
                                 float* __restrict__ T) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    quat_to_T_row(quat[b * 4 + 0], quat[b * 4 + 1], quat[b * 4 + 2], quat[b * 4 + 3], trans[b * 3 + 0],
                  trans[b * 3 + 1], trans[b * 3 + 2], T + (size_t)b * 16);
}

__global__ void quat_to_T_bwd_kernel(const float* __restrict__ quat, const float* __restrict__ gT, int B,
                                     float* __restrict__ gq, float* __restrict__ gt) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    quat_to_T_bwd_row(quat[b * 4 + 0], quat[b * 4 + 1], quat[b * 4 + 2], quat[b * 4 + 3], gT + (size_t)b * 16,
                      gq + b * 4, gt + b * 3);
}

}  // namespace delora

using namespace delora;

extern "C" int delora_icp_partial_rows(int src_stride) { return icp_layout(1, src_stride).rows; }

extern "C" int64_t delora_icp_scratch_floats(int B, int src_stride) { return icp_layout(B, src_stride).total; }

extern "C" int delora_icp_fwd_bwd(const delora_f4* src_pts4, const delora_f4* src_nrm4, const int32_t* n_src,
                                  int src_stride, const float* T, const delora_f4* tgt_pts4,
                                  const delora_f4* tgt_nrm4, const int32_t* cell_start, int tgt_stride, int B,
                                  int H, int W, double hfov0, double hfov1, double vfov0, double vfov1,
                                  float lambda_po2pl, uint32_t flags, float* losses, float* grad_T,
                                  int32_t* nn_index, delora_f4* point_dir, delora_f4* normal_dir, float* partials,
                                  void* stream) {
    DELORA_CHECK_ARG(src_pts4 && src_nrm4 && n_src && tgt_pts4 && tgt_nrm4 && cell_start && losses && grad_T &&
                         partials, "delora_icp_fwd_bwd: null pointer");
    DELORA_CHECK_ARG(B > 0 && B <= 65535 && src_stride > 0 && tgt_stride > 0 && H > 0 && W > 0,
                     "delora_icp_fwd_bwd: bad shape");
    const GridParams g = make_grid(H, W, hfov0, hfov1, vfov0, vfov1, 1);
    const IcpLayout L = icp_layout(B, src_stride);
    const int rows = L.rows;
    const IcpScratch sc = icp_scratch(partials, L);
    dim3 grid((src_stride + kIcpThreads - 1) / kIcpThreads, B);
    cudaStream_t st = (cudaStream_t)stream;
    if (T) {
        icp_kernel<true><<<grid, kIcpThreads, 0, st>>>(
            (const float4*)src_pts4, (const float4*)src_nrm4, n_src, src_stride, T, (const float4*)tgt_pts4,
            (const float4*)tgt_nrm4, cell_start, tgt_stride, g, flags, nn_index, (float4*)point_dir,
            (float4*)normal_dir, sc.rows, rows);
    } else {
        icp_kernel<false><<<grid, kIcpThreads, 0, st>>>(
            (const float4*)src_pts4, (const float4*)src_nrm4, n_src, src_stride, T, (const float4*)tgt_pts4,
            (const float4*)tgt_nrm4, cell_start, tgt_stride, g, flags, nn_index, (float4*)point_dir,
            (float4*)normal_dir, sc.rows, rows);
    }
    DELORA_CHECK_LAUNCH("icp_kernel");
    return launch_icp_finalize(sc, B, rows, lambda_po2pl, losses, grad_T, st);
}

extern "C" int delora_icp_point_grads(const delora_f4* point_dir, const delora_f4* normal_dir,
                                      const int32_t* n_src, int src_stride, int B, const float* losses,
                                      const float* upstream, float* grad_pts, float* grad_nrm, void* stream) {
    DELORA_CHECK_ARG(point_dir && normal_dir && n_src && losses && upstream && grad_pts && grad_nrm,
                     "delora_icp_point_grads: null pointer");
    DELORA_CHECK_ARG(B > 0 && B <= 65535 && src_stride > 0, "delora_icp_point_grads: bad shape");
    dim3 grid((src_stride + 255) / 256, B);
    icp_point_grads_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float4*)point_dir,
                                                                   (const float4*)normal_dir, n_src, src_stride,
                                                                   losses, upstream, grad_pts, grad_nrm);
    DELORA_CHECK_LAUNCH("icp_point_grads_kernel");
    return 0;
}

extern "C" int delora_quat_to_T(const float* quaternion, const float* translation, int B, float* T, void* stream) {
    DELORA_CHECK_ARG(quaternion && translation && T && B > 0, "delora_quat_to_T: bad argument");
    quat_to_T_kernel<<<(B + 63) / 64, 64, 0, (cudaStream_t)stream>>>(quaternion, translation, B, T);
    DELORA_CHECK_LAUNCH("quat_to_T_kernel");
    return 0;
}

extern "C" int delora_quat_to_T_bwd(const float* quaternion, const float* grad_T, int B, float* grad_quaternion,
                                    float* grad_translation, void* stream) {
    DELORA_CHECK_ARG(quaternion && grad_T && grad_quaternion && grad_translation && B > 0,
                     "delora_quat_to_T_bwd: bad argument");
    quat_to_T_bwd_kernel<<<(B + 63) / 64, 64, 0, (cudaStream_t)stream>>>(quaternion, grad_T, B, grad_quaternion,
                                                                         grad_translation);
    DELORA_CHECK_LAUNCH("quat_to_T_bwd_kernel");
    return 0;
}
