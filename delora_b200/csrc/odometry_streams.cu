// The streams workspaces (sm_90a): S = max_batch independent LiDAR streams in one workspace, one call per tick.
//
// delora_odometry_streams_push: per tick, the masked count clamp, the projection of the S new frames (inactive streams
// project 0 points), the fused input conversion + cache update, the trunk and the fc / hidden layers at B = S (the
// launches of _pairs), and the per-row output kernel.  A stream's row goes through the same instructions as _push's
// batch-1 call: the trunk's kernels and the tail's row_dot4 sum a row in an order that does not depend on B, and the
// output kernel divides each quaternion by its own norm, which at B = 1 is the block norm of odometry_out_kernel.
// Every launch is unconditional; activity and per-stream state are read on the device only.
//
// The kinds.  Each one is the layout of the kind it extends with its own sections appended, so no offset of that
// layout moves and _streams_load_weights and _streams_reset work on every kind.
//   plain (delora_odometry_streams_push): S = max_batch streams, this tick's S frames, each stream's previous frame and
//     whether it has one; the trunk and tail then run at B = S.
//   residual (_push_residual): plain, then the sections of the per-frame ICP residual.
//   info (_push_info): residual, then the information rows and the information operator's scratch.
//   normalized (_push_normalized): plain, then the staged point rows and the pair factors.  Its prev_image section
//     holds this tick's projection of each previous frame; nothing reads it across ticks.
//   pre (_push_pre): residual (its H x W grids and ICP sections serve the recipe's ICP), then the H x w_pre sections.
//     The plain layout's key buffers serve both H x W projections of a tick, its images hold this tick's projection
//     of both frames of each pair.
//   pre_info (_push_pre_info): pre, then info's information rows and scratch.
//
// The grid clear, reset, pre and masked-row kernels also serve the adapting streams (odometry_adapt.cu) through the
// host functions declared in odometry.cuh.
#include <cuda_bf16.h>
#include <string.h>

#include "odometry.cuh"
#include "projection.cuh"

namespace delora {

enum class Streams { plain, residual, normalized, pre, info, pre_info };

// The inference plan of S = max_batch streams (see plan_inference), with the sections of its kind appended
struct StreamsPlan : InferPlan {
    // residual only (delora_odometry_streams_push_residual), after every other section: the dense grids of the S new
    // frames and of each stream's previous frame, the 3x4 transforms the ICP reads, its outputs and its scratch
    size_t pts_grid, nrm_grid, prev_pts_grid, prev_nrm_grid, T12, losses, grad_T, icp;
    // information streams only (delora_odometry_streams_push_info), after every residual section: the information rows
    // of the S pairs and the operator's info_scratch
    size_t info, info_scratch;
    // normalised streams only (delora_odometry_streams_push_normalized), after every streams section: the point rows
    // [2S, 3, n_stride] (each stream's previous frame, then its last frame), their counts [2S] followed by the count
    // of each stream's last frame [S], and the factor of each pair [S]
    size_t stage, stage_counts, factor;
    // recipe streams only (delora_odometry_streams_push_pre), after every residual section: the H x w_pre stage of the
    // S new frames (depth keys, image, index map), the H x w_pre grids [2S] (each stream's previous frame, then this
    // tick's frames), the model's T in the units it saw [S, 16]; factor (above) holds the pair factors
    size_t pre_keys, pre_image, pre_index_map, pre_pts, pre_nrm, T16;
};

static void make_streams_plan(const delora_odometry_desc* d, Streams kind, StreamsPlan* p) {
    memset(p, 0, sizeof(StreamsPlan));
    const int MB = d->max_batch;
    plan_inference(d, MB, MB, true, p);
    const size_t S = (size_t)MB, HW = (size_t)d->H * d->W, HWp = (size_t)d->H * d->w_pre;
    size_t off = p->total;
    const bool pre = kind == Streams::pre || kind == Streams::pre_info;
    if (kind == Streams::residual || pre || kind == Streams::info) {
        p->pts_grid = take(off, S * HW * 16);
        p->nrm_grid = take(off, S * HW * 16);
        p->prev_pts_grid = take(off, S * HW * 16);
        p->prev_nrm_grid = take(off, S * HW * 16);
        p->T12 = take(off, S * 12 * 4);
        p->losses = take(off, S * DELORA_LOSS_ROW * 4);
        p->grad_T = take(off, S * 12 * 4);
        p->icp = take(off, (size_t)delora_icp_scratch_floats(MB, (int)HW) * 4);
    }
    if (kind == Streams::normalized) {
        p->stage = take(off, 2 * S * 3 * (size_t)d->n_stride * 4);
        p->stage_counts = take(off, 3 * S * 4);
        p->factor = take(off, S * 4);
    }
    if (pre) {
        p->pre_keys = take(off, S * HWp * 8);
        p->pre_image = take(off, S * 4 * HWp * 4);
        p->pre_index_map = take(off, S * HWp * 4);
        p->pre_pts = take(off, 2 * S * HWp * 16);
        p->pre_nrm = take(off, 2 * S * HWp * 16);
        p->T16 = take(off, S * 16 * 4);
        p->factor = take(off, S * 4);
    }
    if (kind == Streams::info || kind == Streams::pre_info) {
        p->info = take(off, S * DELORA_INFO_ROW * 4);
        p->info_scratch = take(off, (size_t)delora_icp_information_scratch_floats(MB, d->H, d->W) * 4);
    }
    p->total = off;
}

// (prev [S,4,H,W], cur [S,4,H,W]) fp32 -> the trunk input [S, H+2, W+2, C] bf16 with the bits of images_to_nhwc16_kernel
// (C = 16) / images_to_nhwc_kernel (C = 64, Cpad 64), and cur -> prev for every active stream.
// One thread per (stream, padded row, image column w, 8-channel group; C = 16 has one group of 16).  The thread of
// column w writes padded column w + 1, and also the circular halo column 0 when w = W - 1 and column W + 1 when w = 0.
// So every prev pixel has exactly one reader, the thread that then overwrites it: no pixel is overwritten before it is
// read, without a barrier.  prev is read with plain loads (it is written in this kernel).
template <int C>
__global__ void __launch_bounds__(256)
odometry_streams_input_kernel(const float* __restrict__ cur, float* prev, const int32_t* __restrict__ active, int S,
                              int H, int W, __nv_bfloat16* __restrict__ x) {
    constexpr int G = C == 16 ? 1 : C / 8;
    const int Hp = H + 2, Wp = W + 2;
    const size_t total = (size_t)S * Hp * W * G;
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const int grp = (int)(i % G);
    const size_t pix = i / G;
    const int w = (int)(pix % W), hp = (int)((pix / W) % Hp), s = (int)(pix / ((size_t)W * Hp));
    uint4 v0 = make_uint4(0u, 0u, 0u, 0u), v1 = make_uint4(0u, 0u, 0u, 0u);
    const bool interior = hp != 0 && hp != Hp - 1;
    if (grp == 0 && interior) {
        const size_t plane = (size_t)H * W, base = (size_t)s * 4 * plane + (size_t)(hp - 1) * W + w;
        float f[8];
#pragma unroll
        for (int c = 0; c < 4; ++c) { f[c] = prev[base + c * plane]; f[4 + c] = __ldg(cur + base + c * plane); }
        if (C == 16) {
            __nv_bfloat16 hv[8], lv[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                hv[c] = __float2bfloat16_rn(f[c]);
                lv[c] = __float2bfloat16_rn(f[c] - __bfloat162float(hv[c]));
            }
            v0 = *reinterpret_cast<uint4*>(hv);
            v1 = *reinterpret_cast<uint4*>(lv);
        } else {
            __nv_bfloat162 v[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) v[c] = __floats2bfloat162_rn(f[2 * c], f[2 * c + 1]);
            v0 = *reinterpret_cast<uint4*>(v);
        }
        if (stream_active(active, s)) {
#pragma unroll
            for (int c = 0; c < 4; ++c) prev[base + c * plane] = f[4 + c];
        }
    }
    auto store = [&](int wp) {
        __nv_bfloat16* dst = x + (((size_t)s * Hp + hp) * Wp + wp) * C + grp * 8;
        reinterpret_cast<uint4*>(dst)[0] = v0;
        if (C == 16) reinterpret_cast<uint4*>(dst)[1] = v1;
    };
    store(w + 1);
    if (w == W - 1) store(0);
    if (w == 0) store(W + 1);
}

// delora_odometry_streams_push_normalized's masked count clamp fused with the staging of the point rows.
// stage [2S, 3, n_stride]: row s holds stream s's previous frame, row S + s its last frame; counts [3S]: this tick's
// counts of the 2S rows, then the count of each stream's last frame.  For every active stream: row S + s moves to row s
// (the counts[2S + s] points of its last frame, if it has a previous frame; none otherwise), then the caller's frame
// (its clamped count of points) goes to row S + s.  This tick's counts: row s = the moved count, row S + s = the
// clamped count for an active stream, 0 for an inactive one, whose rows are not touched.  One thread per (point index, stream)
// moves and copies the three coordinates of its point: the thread that reads an old value of row S + s is the one that
// then overwrites it, so no value is overwritten before it is read, without a barrier.  counts[2S + s], which every
// CTA of the stream reads here, is updated by the output kernel.
__global__ void __launch_bounds__(256)
odometry_streams_stage_kernel(const float* __restrict__ points, const int32_t* __restrict__ n_points,
                              const int32_t* __restrict__ active, const int32_t* __restrict__ has_prev, int S,
                              int n_stride, float* stage, int32_t* counts) {
    const int s = blockIdx.y;
    const int i = blockIdx.x * 256 + threadIdx.x;
    const bool act = stream_active(active, s);
    const int n_prev = act && has_prev[s] != 0 ? counts[2 * S + s] : 0;
    const int n_cur = act ? min(max(n_points[s], 0), n_stride) : 0;
    if (i == 0) {
        counts[s] = n_prev;
        counts[S + s] = n_cur;
    }
    if (i >= max(n_prev, n_cur)) return;
    float* prev = stage + (size_t)s * 3 * n_stride;
    float* last = stage + (size_t)(S + s) * 3 * n_stride;
    const float* src = points + (size_t)s * 3 * n_stride;
    float old[3], cur[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        old[c] = i < n_prev ? last[(size_t)c * n_stride + i] : 0.0f;       // plain loads: row S + s is written here
        cur[c] = i < n_cur ? __ldg(src + (size_t)c * n_stride + i) : 0.0f;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        if (i < n_prev) prev[(size_t)c * n_stride + i] = old[c];
        if (i < n_cur) last[(size_t)c * n_stride + i] = cur[c];
    }
}

__global__ void odometry_streams_reset_kernel(const int32_t* __restrict__ mask, int S, int32_t* __restrict__ has_prev) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < S && mask[s] != 0) has_prev[s] = 0;
}

// ---- the per-frame ICP residual (delora_odometry_streams_push_residual)
__device__ __forceinline__ float4 empty_grid_cell() {       // what the normals kernel writes for a pixel without a point
    return make_float4(__int_as_float(0x7f800000), __int_as_float(0x7f800000), __int_as_float(0x7f800000),
                       __int_as_float(-1));
}

// every cached grid starts empty: the target of a stream that has not had a frame yet
__global__ void __launch_bounds__(256)
odometry_streams_grid_clear_kernel(float4* __restrict__ pts, float4* __restrict__ nrm, size_t n) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    pts[i] = empty_grid_cell();
    nrm[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

// The grids of the S new frames (cur) and of each stream's previous frame (prev) around the ICP, which runs at B = S
// with source = cur, target = prev.  One thread per cell, a float4 of the point grid and one of the normal grid.
// kPhase 0, before the ICP: a stream that is active without a transform this tick (its first frame since the start
//   or a reset) caches its grids now and its cur grids become empty, so the ICP finds no source pixel for it and never
//   searches its stale target; streams without a frame have empty cur grids from the projection already.  Also
//   T12 [S, 12] = the 3x4 part of T of the valid streams, the identity for the others (whose T row is not written).
// kPhase 1, after the ICP has read the targets: the valid streams cache their grids; losses [S, DELORA_LOSS_ROW] =
//   the ICP's row of the valid streams, zeros for the others.
// Every stream's grids are copied at most once per tick, and only if it has a frame.
template <int kPhase>
__global__ void __launch_bounds__(256)
odometry_streams_grids_kernel(float4* __restrict__ cur_pts, float4* __restrict__ cur_nrm, float4* __restrict__ prev_pts,
                              float4* __restrict__ prev_nrm, const int32_t* __restrict__ active,
                              const int32_t* __restrict__ valid, int S, int HW, const float* __restrict__ T16,
                              float* __restrict__ T12, const float* __restrict__ icp_losses,
                              float* __restrict__ losses) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (kPhase == 0 && i < (size_t)S * 12) {
        const int s = (int)i / 12, e = (int)i % 12;
        T12[i] = valid[s] != 0 ? T16[s * 16 + e] : (e % 5 == 0 ? 1.0f : 0.0f);
    }
    if (kPhase == 1 && i < (size_t)S * DELORA_LOSS_ROW)
        losses[i] = valid[i / DELORA_LOSS_ROW] != 0 ? icp_losses[i] : 0.0f;
    if (i >= (size_t)S * HW) return;
    const int s = (int)(i / HW);
    const bool ok = valid[s] != 0;
    if (kPhase == 0 ? (ok || !stream_active(active, s)) : !ok) return;
    prev_pts[i] = cur_pts[i];
    prev_nrm[i] = cur_nrm[i];
    if (kPhase == 0) {
        cur_pts[i] = empty_grid_cell();
        cur_nrm[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
}

// ---- the recipe streams (delora_odometry_streams_push_pre) and the adapting streams (_streams_push_adapt)
// Between the output kernel (which wrote T16 and valid) and the ICP; one thread per element of the largest of T16
// [S, 16], the H x W grids [S, HW] and the cached grids [S, HWp].
//   T16: for a valid stream T[s] = T16[s] (factor non-NULL: T[:3, 3] multiplied by factor[s] with the instructions of
//     odometry_out_kernel<true>) and factor_out[s] = factor[s] (factor_out non-NULL); factor_out[s] = 0 for the others,
//     whose T row is not written.  T12 = the 3x4 of T16 (the model's units, the ICP's) for valid streams, the identity
//     for the others.
//   The masked cache write: every active stream's new grids (pre_cur, HWp cells each) become its cached previous frame
//     (pre_prev); inactive streams' slots stay.  cur_image non-NULL: so does its image, [S, 4, H, W] read as HW float4
//     per stream (HWp = HW then).  The cache was last read by stages that precede this kernel.
//   H x W: then a stream without a transform has its source grids (cur) emptied, so the ICP finds no source pixel for
//     it (a stream without a frame has empty grids already; one on its first frame has points).  pre_cur may be cur
//     (the adapting streams at w_pre = 0 cache their H x W grids): the thread that caches a cell is the one that then
//     empties it.
__global__ void __launch_bounds__(256)
odometry_streams_pre_kernel(const float* __restrict__ T16, const float* __restrict__ factor,
                            const int32_t* __restrict__ active, const int32_t* __restrict__ valid, int S, int HW,
                            int HWp, float* __restrict__ T, float* __restrict__ T12, float* __restrict__ factor_out,
                            float4* cur_pts, float4* cur_nrm, const float4* pre_cur_pts, const float4* pre_cur_nrm,
                            float4* __restrict__ pre_prev_pts, float4* __restrict__ pre_prev_nrm,
                            const float4* __restrict__ cur_image = nullptr, float4* __restrict__ cache_image = nullptr) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i < (size_t)S * 16) {
        const int s = (int)i / 16, e = (int)i % 16;
        const bool ok = valid[s] != 0;
        const float t = T16[i];
        if (ok) T[i] = (factor && (e == 3 || e == 7 || e == 11)) ? __fmul_rn(t, factor[s]) : t;
        if (e < 12) T12[s * 12 + e] = ok ? t : (e % 5 == 0 ? 1.0f : 0.0f);
        if (e == 0 && factor_out) factor_out[s] = ok ? factor[s] : 0.0f;
    }
    if (i < (size_t)S * HWp && stream_active(active, (int)(i / HWp))) {
        pre_prev_pts[i] = pre_cur_pts[i];
        pre_prev_nrm[i] = pre_cur_nrm[i];
        if (cur_image) cache_image[i] = cur_image[i];
    }
    if (i < (size_t)S * HW && valid[i / HW] == 0) {
        cur_pts[i] = empty_grid_cell();
        cur_nrm[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
}

// out [S, kRow] = the rows [S, kRow] of the valid streams, zeros for the others: the ICP's loss rows
// (DELORA_LOSS_ROW) or the information operator's rows (DELORA_INFO_ROW)
template <int kRow>
__global__ void odometry_streams_rows_kernel(const int32_t* __restrict__ valid, int S, const float* __restrict__ rows,
                                             float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < S * kRow) out[i] = valid[i / kRow] != 0 ? rows[i] : 0.0f;
}

// check_desc plus the preprocessing width the recipe streams read (the training rule, but w_pre = 0 is refused)
static int check_pre_desc(const delora_odometry_desc* d, const char* who) {
    if (check_desc(d, who)) return 1;
    DELORA_CHECK_ARG(d->w_pre >= 2 && (long long)d->H * d->w_pre < (1ll << 27),
                     "%s: w_pre=%d must be >= 2 with H * w_pre < 2^27 (H=%d): the recipe streams estimate the normals "
                     "at H x w_pre", who, d->w_pre, d->H);
    return 0;
}

static int check_streams_desc(const delora_odometry_desc* d, Streams kind, const char* who) {
    return kind == Streams::pre || kind == Streams::pre_info ? check_pre_desc(d, who) : check_desc(d, who);
}

static int64_t streams_workspace_bytes(const delora_odometry_desc* d, Streams kind, const char* who) {
    if (check_streams_desc(d, kind, who)) return -1;
    StreamsPlan p;
    make_streams_plan(d, kind, &p);
    return (int64_t)p.total;
}

// The sections the streams entry points of one kind dereference.  Offsets of a section the kind does not have stay 0
// in its plan (run_streams_push forms the grid pointers of a plain workspace at ws + 0, the keys, and reads them only
// with rp, i.e. on the residual and information kinds); those are not listed.  Nor are the normalised kind's counts
// (its count clamp writes stage_counts) and the recipe kinds' index map (their H x W projections pass none).
int map_streams(SectionMap& s, const delora_odometry_desc* d, int kind, const char* who) {
    static const Streams kinds[] = {Streams::plain, Streams::residual, Streams::info, Streams::normalized, Streams::pre,
                                    Streams::pre_info};
    const Streams k = kinds[kind - DELORA_WS_STREAMS];
    if (check_streams_desc(d, k, who)) return 1;
    StreamsPlan p;
    make_streams_plan(d, k, &p);
    const bool pre = k == Streams::pre || k == Streams::pre_info;
    // the recipe and normalised kinds project both frames of every pair each tick: their prev_image holds no state
    const bool cached = !pre && k != Streams::normalized;
    map_frames(s, p.f, !pre, k != Streams::normalized, cached ? DELORA_WS_STATE : DELORA_WS_SCRATCH);
    map_inference(s, p, DELORA_WS_SCRATCH);
    if (p.pts_grid) {
        s.field("pts_grid", p.pts_grid, DELORA_WS_SCRATCH);
        s.field("nrm_grid", p.nrm_grid, DELORA_WS_SCRATCH);
        // the residual kinds cache each stream's grids here; the recipe re-projects them from pre_pts every tick
        s.field("prev_pts_grid", p.prev_pts_grid, pre ? DELORA_WS_SCRATCH : DELORA_WS_STATE);
        s.field("prev_nrm_grid", p.prev_nrm_grid, pre ? DELORA_WS_SCRATCH : DELORA_WS_STATE);
        s.field("T12", p.T12, DELORA_WS_SCRATCH);
        s.field("losses", p.losses, DELORA_WS_OUTPUT);
        s.field("grad_T", p.grad_T, DELORA_WS_SCRATCH);
        s.field("icp", p.icp, DELORA_WS_SCRATCH);
    }
    if (p.stage) {
        s.field("stage", p.stage, DELORA_WS_STATE);                  // row S + s: each stream's last frame
        s.field("stage_counts", p.stage_counts, DELORA_WS_STATE);    // [2S + s]: its count
    }
    if (pre) {
        s.field("pre_keys", p.pre_keys, DELORA_WS_SCRATCH);
        s.field("pre_image", p.pre_image, DELORA_WS_SCRATCH);
        s.field("pre_index_map", p.pre_index_map, DELORA_WS_SCRATCH);
        s.field("pre_pts", p.pre_pts, DELORA_WS_STATE);               // [0, S): each stream's cached grids
        s.field("pre_nrm", p.pre_nrm, DELORA_WS_STATE);
        s.field("T16", p.T16, DELORA_WS_SCRATCH);
    }
    if (p.factor) s.field("factor", p.factor, DELORA_WS_SCRATCH);
    if (p.info) {
        s.field("info", p.info, DELORA_WS_OUTPUT);
        s.field("info_scratch", p.info_scratch, DELORA_WS_SCRATCH);
    }
    return 0;
}

// The n cells of the cached grids at offsets pts / nrm start empty: the target of a stream that has not had a frame yet
int clear_grids(char* ws, size_t pts, size_t nrm, size_t n, cudaStream_t st) {
    odometry_streams_grid_clear_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        reinterpret_cast<float4*>(ws + pts), reinterpret_cast<float4*>(ws + nrm), n);
    DELORA_CHECK_LAUNCH("odometry_streams_grid_clear_kernel");
    return 0;
}

// The residual, information and recipe kinds' ICP scratch is zeroed here, once, and their cached grids start empty
static int streams_init(const delora_odometry_desc* d, Streams kind, void* workspace, cudaStream_t st, const char* who) {
    if (check_streams_desc(d, kind, who)) return 1;
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    StreamsPlan p;
    make_streams_plan(d, kind, &p);
    char* ws = (char*)workspace;
    const int rc = init_workspace(p.f, p.total, workspace, st, who);
    if (rc) return rc;
    const size_t S = (size_t)d->max_batch;
    if (kind == Streams::residual || kind == Streams::info) return clear_grids(ws, p.prev_pts_grid, p.prev_nrm_grid, S * d->H * d->W, st);
    if (kind == Streams::pre || kind == Streams::pre_info) {
        const size_t n = S * d->H * d->w_pre;
        const cudaError_t e = cudaMemsetAsync(ws + p.pre_keys, 0xFF, n * 8, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
        return clear_grids(ws, p.pre_pts, p.pre_nrm, n, st);
    }
    return 0;
}

// The caller's buffers of a streams tick, refused in this order; extra is the kind's own output named extra_name
// (losses or factor), or nothing with extra_name NULL
int check_tick(const void* points, const void* n_points, const void* workspace, const float* T, const int32_t* valid,
               const float* extra, const char* extra_name, const char* who) {
    DELORA_CHECK_ARG(points, "%s: null points", who);
    DELORA_CHECK_ARG(n_points, "%s: null n_points", who);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    DELORA_CHECK_ARG(T, "%s: null T", who);
    DELORA_CHECK_ARG(valid, "%s: null valid", who);
    DELORA_CHECK_ARG(!extra_name || extra, "%s: null %s", who, extra_name);
    return 0;
}

// The residual's settings: loss_flags may have the ICP losses, DELORA_NORMAL_LINEAR, DELORA_LOSS_PO2PO_ALONE and, with
// scaling (the recipe streams), DELORA_TRAIN_NORMALIZATION_SCALING
static int check_residual_params(const delora_odometry_residual_params* rp, bool scaling, const char* who) {
    DELORA_CHECK_ARG(rp, "%s: null residual_params", who);
    if (check_icp_params(rp->lambda_po2pl, rp->loss_flags, rp->nb_h, rp->nb_w, rp->epsilon_range, rp->min_neighbors, who))
        return 1;
    const uint32_t bits = DELORA_LOSS_PO2PO | DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL | DELORA_NORMAL_LINEAR |
                          DELORA_LOSS_PO2PO_ALONE | (scaling ? DELORA_TRAIN_NORMALIZATION_SCALING : 0u);
    DELORA_CHECK_ARG((rp->loss_flags & ~bits) == 0u, "%s: loss_flags=0x%x has a bit other than %s", who, rp->loss_flags,
                     scaling ? "the ICP losses, DELORA_NORMAL_LINEAR, DELORA_LOSS_PO2PO_ALONE and "
                               "DELORA_TRAIN_NORMALIZATION_SCALING"
                             : "the ICP losses, DELORA_NORMAL_LINEAR and DELORA_LOSS_PO2PO_ALONE");
    return 0;
}

// The ICP entry point whose work icp_dense_launch does with these info and factor pointers: the name its refusals give
const char* icp_entry(const float* info, const float* factor) {
    return !info ? "delora_icp_dense_fwd_bwd" : factor ? "delora_icp_dense_information_scaled"
                                                       : "delora_icp_dense_information";
}

// The ICP at B = S on a residual or recipe plan's H x W grids: source pts_grid moved by T12, target prev_pts_grid,
// into its losses and grad_T; on an information plan (p.info set) also into its information rows, in metres with the
// pair factors of a normalised recipe (factor non-NULL).  The recipe's DELORA_TRAIN_NORMALIZATION_SCALING is not an
// ICP bit; DELORA_LOSS_PO2PO_ALONE is DELORA_LOSS_PO2PO on the zero normal grids of the points-only front end.
static int streams_icp(const delora_odometry_desc* d, const delora_odometry_residual_params* rp, const StreamsPlan& p,
                       char* ws, const float* factor, cudaStream_t st) {
    auto f = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
    auto f4 = [&](size_t o) { return reinterpret_cast<delora_f4*>(ws + o); };
    const uint32_t flags = rp->loss_flags & ~(DELORA_TRAIN_NORMALIZATION_SCALING | DELORA_LOSS_PO2PO_ALONE);
    float* info = p.info ? f(p.info) : nullptr;
    if (!info) factor = nullptr;
    return icp_dense_launch(f4(p.pts_grid), f4(p.nrm_grid), f(p.T12), f4(p.prev_pts_grid), f4(p.prev_nrm_grid),
                            d->max_batch, d->H, d->W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, rp->lambda_po2pl, flags,
                            f(p.losses), f(p.grad_T), f(p.icp), info, info ? f(p.info_scratch) : nullptr, factor, st,
                            icp_entry(info, factor));
}

// out [S, row] = the rows [S, row] at `rows` of the valid streams, zeros for the others; row is DELORA_LOSS_ROW or
// DELORA_INFO_ROW
int streams_rows_out(int row, const int32_t* valid, int S, const float* rows, float* out, cudaStream_t st) {
    const unsigned blocks = (S * row + 255) / 256;
    if (row == DELORA_INFO_ROW)
        odometry_streams_rows_kernel<DELORA_INFO_ROW><<<blocks, 256, 0, st>>>(valid, S, rows, out);
    else
        odometry_streams_rows_kernel<DELORA_LOSS_ROW><<<blocks, 256, 0, st>>>(valid, S, rows, out);
    DELORA_CHECK_LAUNCH(row == DELORA_INFO_ROW ? "odometry_streams_rows_kernel<DELORA_INFO_ROW>"
                                               : "odometry_streams_rows_kernel<DELORA_LOSS_ROW>");
    return 0;
}

// odometry_streams_pre_kernel (see there for the arguments), one thread per element of the largest of T16 [S, 16], the
// H x W grids [S, HW] and the cached grids [S, HWp]
int streams_pre(const float* T16, const float* factor, const int32_t* active, const int32_t* valid, int S, int HW,
                int HWp, float* T, float* T12, float* factor_out, float4* cur_pts, float4* cur_nrm,
                const float4* pre_cur_pts, const float4* pre_cur_nrm, float4* pre_prev_pts, float4* pre_prev_nrm,
                const float4* cur_image, float4* cache_image, cudaStream_t st) {
    int per_stream = HWp > HW ? HWp : HW;
    if (per_stream < 16) per_stream = 16;
    const size_t cells = (size_t)S * per_stream;
    odometry_streams_pre_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, st>>>(
        T16, factor, active, valid, S, HW, HWp, T, T12, factor_out, cur_pts, cur_nrm, pre_cur_pts, pre_cur_nrm,
        pre_prev_pts, pre_prev_nrm, cur_image, cache_image);
    DELORA_CHECK_LAUNCH("odometry_streams_pre_kernel");
    return 0;
}

// delora_odometry_streams_reset and _streams_adapt_reset, on the has_prev flags at that offset
int reset_streams(const delora_odometry_desc* d, const int32_t* mask, void* workspace, size_t has_prev,
                  void* stream, const char* who) {
    DELORA_CHECK_ARG(mask, "%s: null mask", who);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    const int S = d->max_batch;
    odometry_streams_reset_kernel<<<(S + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
        mask, S, reinterpret_cast<int32_t*>((char*)workspace + has_prev));
    DELORA_CHECK_LAUNCH("odometry_streams_reset_kernel");
    return 0;
}

}  // namespace delora

using namespace delora;

extern "C" int64_t delora_odometry_streams_workspace_bytes(const delora_odometry_desc* d) {
    return streams_workspace_bytes(d, Streams::plain, "delora_odometry_streams_workspace_bytes");
}

extern "C" int delora_odometry_streams_init(const delora_odometry_desc* d, void* workspace, void* stream) {
    return streams_init(d, Streams::plain, workspace, (cudaStream_t)stream, "delora_odometry_streams_init");
}

extern "C" int delora_odometry_streams_load_weights(const delora_odometry_desc* d, const float* weights, void* workspace,
                                                    void* stream) {
    const char* who = "delora_odometry_streams_load_weights";
    if (check_desc(d, who)) return 1;
    DELORA_CHECK_ARG(weights, "%s: null weights", who);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    StreamsPlan p;
    make_streams_plan(d, Streams::plain, &p);
    return load_weights(p, weights, workspace, (cudaStream_t)stream, who);
}

// delora_odometry_streams_push (rp NULL), delora_odometry_streams_push_residual and, with info, _streams_push_info
// (arguments checked by the callers)
static int run_streams_push(const delora_odometry_desc* d, const delora_odometry_residual_params* rp, const float* points,
                            const int32_t* n_points, const int32_t* active, void* workspace, float* T, int32_t* valid,
                            float* losses, float* info, cudaStream_t st) {
    StreamsPlan p;
    make_streams_plan(d, info ? Streams::info : rp ? Streams::residual : Streams::plain, &p);
    char* ws = (char*)workspace;
    const int S = d->max_batch, H = d->H, W = d->W;
    float* cur = reinterpret_cast<float*>(ws + p.f.images);
    float* prev = reinterpret_cast<float*>(ws + p.f.prev_image);
    int32_t* has_prev = reinterpret_cast<int32_t*>(ws + p.f.has_prev);
    float4* pts_grid = reinterpret_cast<float4*>(ws + p.pts_grid);
    float4* nrm_grid = reinterpret_cast<float4*>(ws + p.nrm_grid);
    int rc;
    if (rp) {
        // the image of delora_project_fwd, bit for bit, plus the grids of the S frames with their normals
        if ((rc = clamp_counts(p.f, ws, n_points, active, S, d->n_stride, st))) return rc;
        if ((rc = project_scan_grids(d, W, rp->loss_flags, rp->nb_h, rp->nb_w, rp->epsilon_range, rp->min_neighbors,
                                     points, reinterpret_cast<int32_t*>(ws + p.f.counts), S,
                                     reinterpret_cast<uint64_t*>(ws + p.f.keys), cur,
                                     reinterpret_cast<int32_t*>(ws + p.f.index_map),
                                     reinterpret_cast<delora_f4*>(pts_grid), reinterpret_cast<delora_f4*>(nrm_grid), st)))
            return rc;
    } else if ((rc = project(p.f, d, ws, points, n_points, active, S, st))) {
        return rc;
    }
    __nv_bfloat16* x_in = reinterpret_cast<__nv_bfloat16*>(ws + p.t.x_in);
    if (p.m.t.stem_fast) {
        const size_t n = (size_t)S * (H + 2) * W;
        odometry_streams_input_kernel<16><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(cur, prev, active, S, H, W, x_in);
    } else {
        const size_t n = (size_t)S * (H + 2) * W * 8;
        odometry_streams_input_kernel<64><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(cur, prev, active, S, H, W, x_in);
    }
    DELORA_CHECK_LAUNCH("odometry_streams_input_kernel");
    if ((rc = streams_forward(p.m, inference_tail_io(p, ws), p.t, p.w, ws, d->act,
                                     reinterpret_cast<float*>(ws + p.pooled), S, active, has_prev, T, valid, nullptr,
                                     nullptr, nullptr, nullptr, st))) return rc;
    if (!rp) return 0;
    // the residual: this frame moved by T against the stream's previous frame (the training step's orientation,
    // scan_2 -> scan_1), for all S streams in one ICP call whose sources are empty where there is no T
    const int HW = H * W;
    float4* prev_pts = reinterpret_cast<float4*>(ws + p.prev_pts_grid);
    float4* prev_nrm = reinterpret_cast<float4*>(ws + p.prev_nrm_grid);
    float* T12 = reinterpret_cast<float*>(ws + p.T12);
    float* icp_losses = reinterpret_cast<float*>(ws + p.losses);
    const size_t cells = (size_t)S * HW > (size_t)S * 12 ? (size_t)S * HW : (size_t)S * 12;
    const unsigned blocks = (unsigned)((cells + 255) / 256);
    odometry_streams_grids_kernel<0><<<blocks, 256, 0, st>>>(pts_grid, nrm_grid, prev_pts, prev_nrm, active, valid, S, HW,
                                                             T, T12, icp_losses, losses);
    DELORA_CHECK_LAUNCH("odometry_streams_grids_kernel<0>");
    if ((rc = streams_icp(d, rp, p, ws, nullptr, st))) return rc;
    odometry_streams_grids_kernel<1><<<blocks, 256, 0, st>>>(pts_grid, nrm_grid, prev_pts, prev_nrm, active, valid, S, HW,
                                                             T, T12, icp_losses, losses);
    DELORA_CHECK_LAUNCH("odometry_streams_grids_kernel<1>");
    return info ? streams_rows_out(DELORA_INFO_ROW, valid, S, reinterpret_cast<float*>(ws + p.info), info, st) : 0;
}

extern "C" int delora_odometry_streams_push(const delora_odometry_desc* d, const float* points, const int32_t* n_points,
                                            const int32_t* active, void* workspace, float* T, int32_t* valid,
                                            void* stream) {
    const char* who = "delora_odometry_streams_push";
    if (check_desc(d, who)) return 1;
    if (check_tick(points, n_points, workspace, T, valid, nullptr, nullptr, who)) return 1;
    return run_streams_push(d, nullptr, points, n_points, active, workspace, T, valid, nullptr, nullptr,
                            (cudaStream_t)stream);
}

extern "C" int64_t delora_odometry_streams_residual_workspace_bytes(const delora_odometry_desc* d) {
    return streams_workspace_bytes(d, Streams::residual, "delora_odometry_streams_residual_workspace_bytes");
}

extern "C" int delora_odometry_streams_residual_init(const delora_odometry_desc* d, void* workspace, void* stream) {
    return streams_init(d, Streams::residual, workspace, (cudaStream_t)stream, "delora_odometry_streams_residual_init");
}

extern "C" int delora_odometry_streams_push_residual(const delora_odometry_desc* d,
                                                     const delora_odometry_residual_params* rp, const float* points,
                                                     const int32_t* n_points, const int32_t* active, void* workspace,
                                                     float* T, int32_t* valid, float* losses, void* stream) {
    const char* who = "delora_odometry_streams_push_residual";
    if (check_desc(d, who)) return 1;
    if (check_residual_params(rp, false, who)) return 1;
    if (check_tick(points, n_points, workspace, T, valid, losses, "losses", who)) return 1;
    return run_streams_push(d, rp, points, n_points, active, workspace, T, valid, losses, nullptr, (cudaStream_t)stream);
}

extern "C" int64_t delora_odometry_streams_info_workspace_bytes(const delora_odometry_desc* d) {
    return streams_workspace_bytes(d, Streams::info, "delora_odometry_streams_info_workspace_bytes");
}

extern "C" int delora_odometry_streams_info_init(const delora_odometry_desc* d, void* workspace, void* stream) {
    return streams_init(d, Streams::info, workspace, (cudaStream_t)stream, "delora_odometry_streams_info_init");
}

extern "C" int delora_odometry_streams_push_info(const delora_odometry_desc* d, const delora_odometry_residual_params* rp,
                                                 const float* points, const int32_t* n_points, const int32_t* active,
                                                 void* workspace, float* T, int32_t* valid, float* losses, float* info,
                                                 void* stream) {
    const char* who = "delora_odometry_streams_push_info";
    if (check_desc(d, who)) return 1;
    if (check_residual_params(rp, false, who)) return 1;
    if (check_tick(points, n_points, workspace, T, valid, losses, "losses", who)) return 1;
    DELORA_CHECK_ARG(info, "%s: null info", who);
    return run_streams_push(d, rp, points, n_points, active, workspace, T, valid, losses, info, (cudaStream_t)stream);
}

extern "C" int64_t delora_odometry_streams_normalized_workspace_bytes(const delora_odometry_desc* d) {
    return streams_workspace_bytes(d, Streams::normalized, "delora_odometry_streams_normalized_workspace_bytes");
}

extern "C" int delora_odometry_streams_normalized_init(const delora_odometry_desc* d, void* workspace, void* stream) {
    return streams_init(d, Streams::normalized, workspace, (cudaStream_t)stream,
                        "delora_odometry_streams_normalized_init");
}

// One tick of a normalised model: the staging of the point rows, the factor of the S pairs (side 0 = rows 0..S-1, the
// previous frames; side 1 = rows S..2S-1, this tick's), the scaled projection of each half (the previous frames into
// prev_image, this tick's into images; each resolve re-arms the shared keys), the pairs' trunk-input conversion, the
// trunk and the tail at B = S, and the rescaling output kernel.  A stream without a pair this tick has a row-s count of
// 0, so its factor is 0 / 0 = NaN and its scaled coordinates project to no pixel; its outputs are not written.
extern "C" int delora_odometry_streams_push_normalized(const delora_odometry_desc* d, const float* points,
                                                       const int32_t* n_points, const int32_t* active, void* workspace,
                                                       float* T, int32_t* valid, float* factor_out, void* stream) {
    const char* who = "delora_odometry_streams_push_normalized";
    if (check_desc(d, who)) return 1;
    if (check_tick(points, n_points, workspace, T, valid, factor_out, "factor", who)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    StreamsPlan p;
    make_streams_plan(d, Streams::normalized, &p);
    char* ws = (char*)workspace;
    const int S = d->max_batch, ns = d->n_stride;
    float* stage = reinterpret_cast<float*>(ws + p.stage);
    int32_t* counts = reinterpret_cast<int32_t*>(ws + p.stage_counts);
    float* factor = reinterpret_cast<float*>(ws + p.factor);
    int32_t* has_prev = reinterpret_cast<int32_t*>(ws + p.f.has_prev);
    float* prev = reinterpret_cast<float*>(ws + p.f.prev_image);
    float* cur = reinterpret_cast<float*>(ws + p.f.images);
    uint64_t* keys = reinterpret_cast<uint64_t*>(ws + p.f.keys);
    int32_t* index_map = reinterpret_cast<int32_t*>(ws + p.f.index_map);
    odometry_streams_stage_kernel<<<dim3((unsigned)((ns + 255) / 256), (unsigned)S), 256, 0, st>>>(
        points, n_points, active, has_prev, S, ns, stage, counts);
    DELORA_CHECK_LAUNCH("odometry_streams_stage_kernel");
    int rc;
    if ((rc = launch_normalization_factors(stage, counts, S, ns, factor, st))) return rc;
    const GridParams g = make_grid(d->H, d->W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0);
    if ((rc = project_fwd(stage, counts, S, 3, ns, g, keys, prev, index_map, factor, S, st))) return rc;
    if ((rc = project_fwd(stage + (size_t)S * 3 * ns, counts + S, S, 3, ns, g, keys, cur, index_map, factor, S, st)))
        return rc;
    if ((rc = trunk_input(p.m.t, p.t, ws, prev, cur, S, st))) return rc;
    return streams_forward(p.m, inference_tail_io(p, ws), p.t, p.w, ws, d->act,
                                 reinterpret_cast<float*>(ws + p.pooled), S, active, has_prev, T, valid, factor,
                                 factor_out, counts, nullptr, st);
}

extern "C" int64_t delora_odometry_streams_pre_workspace_bytes(const delora_odometry_desc* d) {
    return streams_workspace_bytes(d, Streams::pre, "delora_odometry_streams_pre_workspace_bytes");
}

extern "C" int delora_odometry_streams_pre_init(const delora_odometry_desc* d, void* workspace, void* stream) {
    return streams_init(d, Streams::pre, workspace, (cudaStream_t)stream, "delora_odometry_streams_pre_init");
}

// One tick of the recipe (the training step's stages 1-3 at B = S, each pair's first frame from the cache): the masked
// count clamp, projection + normals of the S new frames at H x w_pre, the pair factors over the valid H x w_pre cells
// (flagged models; cached frames are side 0, new ones side 1), both frames of every pair projected to H x W (scaled by
// the pair's factor when flagged), the trunk input, trunk and tail at B = S, the output kernel into T16, the
// bookkeeping kernel (T, T12, factor, emptied sources, cache write), the ICP at B = S and the masked loss rows; with
// info (delora_odometry_streams_push_pre_info) the ICP is the information operator and the masked rows follow.
static int check_push_pre(const delora_odometry_desc* d, const delora_odometry_residual_params* rp, const float* points,
                          const int32_t* n_points, void* workspace, float* T, int32_t* valid, float* losses,
                          float* factor_out, const char* who) {
    if (check_pre_desc(d, who)) return 1;
    if (check_residual_params(rp, true, who)) return 1;
    if (check_tick(points, n_points, workspace, T, valid, losses, "losses", who)) return 1;
    const bool normalized = (rp->loss_flags & DELORA_TRAIN_NORMALIZATION_SCALING) != 0u;
    DELORA_CHECK_ARG(!normalized || factor_out, "%s: null factor with DELORA_TRAIN_NORMALIZATION_SCALING in loss_flags",
                     who);
    DELORA_CHECK_ARG(normalized || !factor_out, "%s: factor must be NULL without DELORA_TRAIN_NORMALIZATION_SCALING in "
                     "loss_flags", who);
    return 0;
}

static int run_push_pre(const delora_odometry_desc* d, const delora_odometry_residual_params* rp, const float* points,
                        const int32_t* n_points, const int32_t* active, void* workspace, float* T, int32_t* valid,
                        float* losses, float* factor_out, float* info, cudaStream_t st) {
    StreamsPlan p;
    make_streams_plan(d, info ? Streams::pre_info : Streams::pre, &p);
    char* ws = (char*)workspace;
    const int S = d->max_batch, H = d->H, W = d->W, Wp = d->w_pre, HW = H * W, HWp = H * Wp;
    auto f = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
    auto f4 = [&](size_t o) { return reinterpret_cast<delora_f4*>(ws + o); };
    delora_f4* pre_prev_pts = f4(p.pre_pts);
    delora_f4* pre_prev_nrm = f4(p.pre_nrm);
    delora_f4* pre_cur_pts = pre_prev_pts + (size_t)S * HWp;
    delora_f4* pre_cur_nrm = pre_prev_nrm + (size_t)S * HWp;
    float* prev = f(p.f.prev_image);
    float* cur = f(p.f.images);
    uint64_t* keys = reinterpret_cast<uint64_t*>(ws + p.f.keys);
    int rc;
    if ((rc = clamp_counts(p.f, ws, n_points, active, S, d->n_stride, st))) return rc;
    if ((rc = project_scan_grids(d, Wp, rp->loss_flags, rp->nb_h, rp->nb_w, rp->epsilon_range, rp->min_neighbors,
                                 points, reinterpret_cast<int32_t*>(ws + p.f.counts), S,
                                 reinterpret_cast<uint64_t*>(ws + p.pre_keys), f(p.pre_image),
                                 reinterpret_cast<int32_t*>(ws + p.pre_index_map), pre_cur_pts, pre_cur_nrm, st)))
        return rc;
    float* factor = factor_out ? f(p.factor) : nullptr;
    if (factor && (rc = launch_grid_normalization_factors(pre_prev_pts, S, HWp, factor, st))) return rc;
    const GridParams g = make_grid(H, W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0);
    if ((rc = project_grids_fwd(pre_prev_pts, pre_prev_nrm, S, Wp, g, keys, prev, nullptr, f4(p.prev_pts_grid),
                                f4(p.prev_nrm_grid), factor, S, st))) return rc;
    if ((rc = project_grids_fwd(pre_cur_pts, pre_cur_nrm, S, Wp, g, keys, cur, nullptr, f4(p.pts_grid), f4(p.nrm_grid),
                                factor, S, st))) return rc;
    if ((rc = trunk_input(p.m.t, p.t, ws, prev, cur, S, st))) return rc;
    int32_t* has_prev = reinterpret_cast<int32_t*>(ws + p.f.has_prev);
    if ((rc = streams_forward(p.m, inference_tail_io(p, ws), p.t, p.w, ws, d->act, f(p.pooled), S, active,
                                     has_prev, f(p.T16), valid, nullptr, nullptr, nullptr, nullptr, st))) return rc;
    if ((rc = streams_pre(f(p.T16), factor, active, valid, S, HW, HWp, T, f(p.T12), factor_out,
                          reinterpret_cast<float4*>(ws + p.pts_grid), reinterpret_cast<float4*>(ws + p.nrm_grid),
                          reinterpret_cast<const float4*>(pre_cur_pts), reinterpret_cast<const float4*>(pre_cur_nrm),
                          reinterpret_cast<float4*>(pre_prev_pts), reinterpret_cast<float4*>(pre_prev_nrm), nullptr,
                          nullptr, st))) return rc;
    if ((rc = streams_icp(d, rp, p, ws, factor, st))) return rc;
    if ((rc = streams_rows_out(DELORA_LOSS_ROW, valid, S, f(p.losses), losses, st))) return rc;
    return info ? streams_rows_out(DELORA_INFO_ROW, valid, S, f(p.info), info, st) : 0;
}

extern "C" int delora_odometry_streams_push_pre(const delora_odometry_desc* d, const delora_odometry_residual_params* rp,
                                                const float* points, const int32_t* n_points, const int32_t* active,
                                                void* workspace, float* T, int32_t* valid, float* losses,
                                                float* factor_out, void* stream) {
    const char* who = "delora_odometry_streams_push_pre";
    if (check_push_pre(d, rp, points, n_points, workspace, T, valid, losses, factor_out, who)) return 1;
    return run_push_pre(d, rp, points, n_points, active, workspace, T, valid, losses, factor_out, nullptr,
                        (cudaStream_t)stream);
}

extern "C" int64_t delora_odometry_streams_pre_info_workspace_bytes(const delora_odometry_desc* d) {
    return streams_workspace_bytes(d, Streams::pre_info, "delora_odometry_streams_pre_info_workspace_bytes");
}

extern "C" int delora_odometry_streams_pre_info_init(const delora_odometry_desc* d, void* workspace, void* stream) {
    return streams_init(d, Streams::pre_info, workspace, (cudaStream_t)stream, "delora_odometry_streams_pre_info_init");
}

extern "C" int delora_odometry_streams_push_pre_info(const delora_odometry_desc* d,
                                                     const delora_odometry_residual_params* rp, const float* points,
                                                     const int32_t* n_points, const int32_t* active, void* workspace,
                                                     float* T, int32_t* valid, float* losses, float* factor_out,
                                                     float* info, void* stream) {
    const char* who = "delora_odometry_streams_push_pre_info";
    if (check_push_pre(d, rp, points, n_points, workspace, T, valid, losses, factor_out, who)) return 1;
    DELORA_CHECK_ARG(info, "%s: null info", who);
    return run_push_pre(d, rp, points, n_points, active, workspace, T, valid, losses, factor_out, info,
                        (cudaStream_t)stream);
}



extern "C" int delora_odometry_streams_reset(const delora_odometry_desc* d, const int32_t* mask, void* workspace,
                                             void* stream) {
    const char* who = "delora_odometry_streams_reset";
    if (check_desc(d, who)) return 1;
    StreamsPlan p;
    make_streams_plan(d, Streams::plain, &p);
    return reset_streams(d, mask, workspace, p.f.has_prev, stream, who);
}
