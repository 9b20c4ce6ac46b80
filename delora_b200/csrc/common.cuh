// Shared device/host helpers for the delora_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/delora_b200.h"

namespace delora {

void set_error(const char* fmt, ...);

#define DELORA_CHECK_ARG(cond, ...)                        \
    do {                                                   \
        if (!(cond)) {                                     \
            ::delora::set_error(__VA_ARGS__);              \
            return 1;                                      \
        }                                                  \
    } while (0)

// `err`: the result of a launch call that returns it (launch_pdl).  A failed launch is also the runtime's last error,
// which is cleared here so that it is not reported again by a later check.
#define DELORA_CHECK_LAUNCH_RESULT(err, name)                                       \
    do {                                                                            \
        const cudaError_t e__ = (err);                                              \
        if (e__ != cudaSuccess) {                                                   \
            cudaGetLastError();                                                     \
            ::delora::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
            return 2;                                                               \
        }                                                                           \
    } while (0)

// after a <<<...>>> launch
#define DELORA_CHECK_LAUNCH(name) DELORA_CHECK_LAUNCH_RESULT(cudaGetLastError(), name)

// Launches `kernel` as the programmatic dependent of the kernel before it on `st`: its CTAs may start once every CTA of
// that kernel has executed griddepcontrol.launch_dependents (or exited), and must execute griddepcontrol.wait before
// they read what that kernel writes.  Returns the launch error.
template <typename... Params, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(Params...), dim3 grid, dim3 block, cudaStream_t st, Args... args) {
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, args...);
}

// SMs of the current device: persistent grids and split-K factors are sized to it (132 on an H100 SXM, 114 on an
// H100 PCIe).  Cached per device; 132 when no device answers (host-side size queries without a GPU).
inline int num_sms() {
    static int cache[64] = {};
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) { cudaGetLastError(); return 132; }
    if (dev < 64 && cache[dev] > 0) return cache[dev];
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { cudaGetLastError(); return 132; }
    if (dev < 64) cache[dev] = n;
    return n;
}

// Spherical grid parameters shared by the projection, the cell binning and the NN search.
// The float constants are produced exactly as torch produces them from the reference's Python
// doubles: the scalar operand of `tensor - float` / `tensor / float` is rounded to fp32 once.
struct GridParams {
    int H, W;
    float hf0, hspan, hinv, wm1;   // u = (atan2(y,x) - hf0) / hspan * wm1
    float vf0, vspan, vinv, hm1;   // v = (atan2(z,|xy|) - vf0) / vspan * hm1
    float du_rad, dv_rad;          // radians per pixel step (hspan/wm1, vspan/hm1)
    // The column index continues across the +-180 deg seam as if column W followed column W-1 at one pixel
    // pitch, but the real gap between the centres of columns W-1 and 0 is 2 pi - hspan.  When a pixel is
    // WIDER than that gap (W = 720: 0.50 deg vs 0.2 deg) an "unwrapped" pixel distance across the seam
    // overstates the angle by seam_px pixels; every exactness bound that looks across the seam subtracts it.
    float seam_px;                 // max(0, 1 - (2 pi - hspan) / du_rad)
    float circ_px;                 // 2 pi / du_rad: pixels once around
    int div_mode;
};

inline GridParams make_grid(int H, int W, double hf0, double hf1, double vf0, double vf1, int div_mode) {
    GridParams g;
    g.H = H; g.W = W;
    g.hf0 = (float)hf0; g.hspan = (float)(hf1 - hf0); g.hinv = 1.0f / g.hspan; g.wm1 = (float)(W - 1);
    g.vf0 = (float)vf0; g.vspan = (float)(vf1 - vf0); g.vinv = 1.0f / g.vspan; g.hm1 = (float)(H - 1);
    g.du_rad = (W > 1) ? (float)((hf1 - hf0) / (double)(W - 1)) : 1.0f;
    g.dv_rad = (H > 1) ? (float)((vf1 - vf0) / (double)(H - 1)) : 1.0f;
    g.seam_px = fmaxf(0.0f, 1.0f - (float)((6.283185307179586 - (hf1 - hf0)) / (double)g.du_rad));
    g.circ_px = (float)(6.283185307179586 / (double)g.du_rad);
    g.div_mode = div_mode;
    return g;
}

// range = torch.norm(xyz, dim=1) on CPU == sqrt((x*x + y*y) + z*z), no FMA contraction
// (probed bit-exact against torch 2.11 CPU on 2e5 random points; DESIGN.md §projection).
__device__ __forceinline__ float range3(float x, float y, float z) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}
__device__ __forceinline__ float range2(float x, float y) {
    return __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
}

// ---------------------------------------------------------------------------------------------
// atan2f with the bits of torch's CPU path.  torch.atan2 on float32 CPU tensors is SLEEF's
// `Sleef_atan2f{8,16}_u10` (FMA builds); CUDA's libdevice atan2f differs from it by 1-2 ulp in a few
// percent of the inputs, enough to move a point across a pixel-rounding boundary now and then.
// This is the same algorithm operation by operation (double-float arithmetic with fma; restated
// from SLEEF's published source and verified against this image's libtorch: see
// oracle/sleef_atan2f.c, its scalar twin, bit-identical to Sleef_atan2f8_u10avx2 on 8e6 pairs).
// Every operation is an IEEE round-to-nearest intrinsic so nvcc can neither fuse nor reorder.
struct F2 { float x, y; };
__device__ __forceinline__ F2 df_div(F2 n, F2 d) {
    const float t = __fdiv_rn(1.0f, d.x);
    const float s = __fmul_rn(n.x, t);
    const float u = __fmaf_rn(t, n.x, -s);
    const float v = __fmaf_rn(-d.y, t, __fmaf_rn(-d.x, t, 1.0f));
    return {s, __fmaf_rn(s, v, __fmaf_rn(n.y, t, u))};
}
__device__ __forceinline__ F2 df_squ(F2 x) {
    const float s = __fmul_rn(x.x, x.x);
    return {s, __fmaf_rn(__fadd_rn(x.x, x.x), x.y, __fmaf_rn(x.x, x.x, -s))};
}
__device__ __forceinline__ F2 df_norm(F2 t) {
    const float s = __fadd_rn(t.x, t.y);
    return {s, __fadd_rn(__fsub_rn(t.x, s), t.y)};
}
__device__ __forceinline__ F2 df_mul(F2 x, F2 y) {
    const float s = __fmul_rn(x.x, y.x);
    return {s, __fmaf_rn(x.x, y.y, __fmaf_rn(x.y, y.x, __fmaf_rn(x.x, y.x, -s)))};
}
__device__ __forceinline__ F2 df_mul_f(F2 x, float y) {
    const float s = __fmul_rn(x.x, y);
    return {s, __fmaf_rn(x.y, y, __fmaf_rn(x.x, y, -s))};
}
__device__ __forceinline__ float mulsign(float x, float y) {
    return __uint_as_float(__float_as_uint(x) ^ (__float_as_uint(y) & 0x80000000u));
}
__device__ __forceinline__ float sleef_atan2f_u10(float y0, float x0) {
    float x = x0, y = y0;
    if (fabsf(x) < 2.9387372783541830947e-39f) { x = __fmul_rn(x, 16777216.0f); y = __fmul_rn(y, 16777216.0f); }
    F2 yy = {fabsf(y), 0.0f}, xx = {x, 0.0f};
    int q = (xx.x < 0.0f) ? -2 : 0;
    if (xx.x < 0.0f) { xx.x = -xx.x; xx.y = -xx.y; }
    const bool p = xx.x < yy.x;
    if (p) q += 1;
    F2 s = p ? F2{-xx.x, -xx.y} : yy;
    F2 t = p ? yy : xx;
    s = df_div(s, t);
    t = df_norm(df_squ(s));
    float u = -0.00176397908944636583328247f;
    u = __fmaf_rn(u, t.x, 0.0107900900766253471374512f);
    u = __fmaf_rn(u, t.x, -0.0309564601629972457885742f);
    u = __fmaf_rn(u, t.x, 0.0577365085482597351074219f);
    u = __fmaf_rn(u, t.x, -0.0838950723409652709960938f);
    u = __fmaf_rn(u, t.x, 0.109463557600975036621094f);
    u = __fmaf_rn(u, t.x, -0.142626821994781494140625f);
    u = __fmaf_rn(u, t.x, 0.199983194470405578613281f);
    {   // t = t * (c + u*t.x)
        const float c = -0.333332866430282592773438f, w = __fmul_rn(u, t.x);
        const float ax = __fadd_rn(c, w);
        t = df_mul(t, F2{ax, __fadd_rn(__fsub_rn(c, ax), w)});
    }
    {   // t = s * (1 + t)
        const float bx = __fadd_rn(1.0f, t.x);
        t = df_mul(s, F2{bx, __fadd_rn(__fadd_rn(__fsub_rn(1.0f, bx), t.x), t.y)});
    }
    {   // t = q * (pi/2 as hi+lo) + t
        const F2 pq = df_mul_f(F2{1.5707963705062866211f, -4.3711388286737928865e-08f}, (float)q);
        const float sx = __fadd_rn(pq.x, t.x);
        t = F2{sx, __fadd_rn(__fadd_rn(__fadd_rn(__fsub_rn(pq.x, sx), t.x), pq.y), t.y)};
    }
    float r = __fadd_rn(t.x, t.y);
    r = mulsign(r, x);
    const float pio2 = 1.5707963267948966f, pio4 = 0.78539816339744831f, pi = 3.14159265358979323846f;
    if (isinf(x) || x == 0.0f) r = __fsub_rn(pio2, isinf(x) ? mulsign(pio2, x) : 0.0f);
    if (isinf(y)) r = __fsub_rn(pio2, isinf(x) ? mulsign(pio4, x) : 0.0f);
    if (y == 0.0f) r = signbit(x) ? pi : 0.0f;
    if (isnan(x) || isnan(y)) return __int_as_float(0x7fc00000);
    return mulsign(r, y);
}

// (u, v) with the reference's op order: src/utility/projection.py:21-31.
// div_mode 0: torch-CPU arithmetic (SLEEF atan2, true division) -- bit-identical to the reference's
//             CPU tensors; div_mode 1: libdevice atan2f and a*(1/b), what torch-CUDA would compute.
__device__ __forceinline__ void pixel_coords(const GridParams& g, float x, float y, float z,
                                             float& u, float& v) {
    const float a_h = (g.div_mode == 0) ? sleef_atan2f_u10(y, x) : atan2f(y, x);
    const float a_v = (g.div_mode == 0) ? sleef_atan2f_u10(z, range2(x, y)) : atan2f(z, range2(x, y));
    float au = __fsub_rn(a_h, g.hf0);
    float av = __fsub_rn(a_v, g.vf0);
    if (g.div_mode == 0) {
        u = __fmul_rn(__fdiv_rn(au, g.hspan), g.wm1);
        v = __fmul_rn(__fdiv_rn(av, g.vspan), g.hm1);
    } else {
        u = __fmul_rn(__fmul_rn(au, g.hinv), g.wm1);
        v = __fmul_rn(__fmul_rn(av, g.vinv), g.hm1);
    }
}

// kornia 0.3.0 quaternion_to_rotation_matrix ((x,y,z,w), L2-normalised with eps 1e-12) and the
// [R|t; 0 0 0 1] assembly of src/models/model_parts.py:37-44, for one batch element: q[4], t[3] -> o[16].
__device__ __forceinline__ void quat_to_T_row(float qx, float qy, float qz, float qw, float t0, float t1, float t2,
                                              float* __restrict__ o) {
    const float nrm = fmaxf(sqrtf(qx * qx + qy * qy + qz * qz + qw * qw), 1e-12f);
    const float x = qx / nrm, y = qy / nrm, z = qz / nrm, w = qw / nrm;
    const float tx = 2.f * x, ty = 2.f * y, tz = 2.f * z;
    const float twx = tx * w, twy = ty * w, twz = tz * w;
    const float txx = tx * x, txy = ty * x, txz = tz * x;
    const float tyy = ty * y, tyz = tz * y, tzz = tz * z;
    o[0] = 1.f - (tyy + tzz); o[1] = txy - twz;         o[2] = txz + twy;         o[3] = t0;
    o[4] = txy + twz;         o[5] = 1.f - (txx + tzz); o[6] = tyz - twx;         o[7] = t1;
    o[8] = txz - twy;         o[9] = tyz + twx;         o[10] = 1.f - (txx + tyy); o[11] = t2;
    o[12] = 0.f; o[13] = 0.f; o[14] = 0.f; o[15] = 1.f;
}

// Backward of quat_to_T_row for one batch element: g = dL/dT in the row-major layout of its first 12 entries (a 4x4 or
// a 3x4 row: the indices coincide) -> dL/dq (q as passed in, before the per-row normalisation) and dL/dt.
__device__ __forceinline__ void quat_to_T_bwd_row(float qx, float qy, float qz, float qw, const float* __restrict__ g,
                                                  float* __restrict__ gq, float* __restrict__ gt) {
    const float nrm_raw = sqrtf(qx * qx + qy * qy + qz * qz + qw * qw);
    const float nrm = fmaxf(nrm_raw, 1e-12f);
    const float x = qx / nrm, y = qy / nrm, z = qz / nrm, w = qw / nrm;
    const float g00 = g[0], g01 = g[1], g02 = g[2], g10 = g[4], g11 = g[5], g12 = g[6], g20 = g[8], g21 = g[9],
                g22 = g[10];
    // dL/d(unit quaternion): R = I + 2*[[-(yy+zz), xy-wz, xz+wy],[xy+wz, -(xx+zz), yz-wx],[xz-wy, yz+wx, -(xx+yy)]]
    const float dx = 2.f * (y * (g01 + g10) + z * (g02 + g20) - 2.f * x * (g11 + g22) + w * (g21 - g12));
    const float dy = 2.f * (x * (g01 + g10) + z * (g12 + g21) - 2.f * y * (g00 + g22) + w * (g02 - g20));
    const float dz = 2.f * (x * (g02 + g20) + y * (g12 + g21) - 2.f * z * (g00 + g11) + w * (g10 - g01));
    const float dw = 2.f * (x * (g21 - g12) + y * (g02 - g20) + z * (g10 - g01));
    // back through q / max(|q|, eps)
    float ox = dx / nrm, oy = dy / nrm, oz = dz / nrm, ow = dw / nrm;
    if (nrm_raw > 1e-12f) {
        const float dot = (dx * x + dy * y + dz * z + dw * w) / nrm;
        ox -= dot * x; oy -= dot * y; oz -= dot * z; ow -= dot * w;
    }
    gq[0] = ox; gq[1] = oy; gq[2] = oz; gq[3] = ow;
    gt[0] = g[3]; gt[1] = g[7]; gt[2] = g[11];
}

// The peer-memory gradient all-reduce (grad_allreduce.cu): its limits, and its launcher for the entry points that
// validated their arguments.  seq_step non-NULL: the device-seq variant, seq = *seq_step * seq_stride + seq.
constexpr int kArMaxThreads = 128;
constexpr int kArMaxWorld = 16;
constexpr int kArMaxCtas = 160;
int grad_allreduce_launch(const uint64_t* peer_bufs, const uint64_t* peer_flags, uint64_t multicast_ptr, int rank,
                          int world, long long offset, long long count, float scale, unsigned seq,
                          const long long* seq_step, unsigned seq_stride, int n_ctas, int n_threads, int32_t* status,
                          cudaStream_t st);
// The valid-count exchange of the adapting streams' group tick: *tick += 1, then *n_out = the sum over the ranks of
// their *n_local, through int32 [2][kArMaxWorld] slots at peer_slots[q] and flag word (phase 0, CTA 0) with
// seq = *tick * seq_stride.
int count_allreduce_launch(const uint64_t* peer_slots, const uint64_t* peer_flags, int rank, int world,
                           unsigned seq_stride, long long* tick, const int32_t* n_local, int32_t* n_out, int32_t* status,
                           cudaStream_t st);
// Loads count_allreduce_kernel and the device-seq all-reduce kernels on the current device (see grad_allreduce.cu)
int collective_kernels_preload(const char* who);

// The dense ICP operator (icp_dense.cu) behind delora_icp_dense_fwd_bwd (info NULL) and
// delora_icp_dense_information[_scaled] (info and info_scratch non-NULL; factor NULL: H unscaled), its refusals
// naming `who`.  The callers check info, info_scratch and factor.
int icp_dense_launch(const delora_f4* src_grid, const delora_f4* src_ngrid, const float* T, const delora_f4* tgt_grid,
                     const delora_f4* tgt_ngrid, int B, int H, int W, double hfov0, double hfov1, double vfov0,
                     double vfov1, float lambda_po2pl, uint32_t flags, float* losses, float* grad_T, float* scratch,
                     float* info, float* info_scratch, const float* factor, cudaStream_t st, const char* who);

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace delora
