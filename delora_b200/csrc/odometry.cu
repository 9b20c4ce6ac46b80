// Odometry inference through the C ABI (sm_90a): raw scans -> relative transforms in one call.
//
// Projection, then the encoder trunk of trunk.cuh (the one the Python encoder runs too), then the tail.
//
// New here: the fully connected tail (reference: src/models/model.py:58-84, :103-116) in fp32.
//   odometry_linear_kernel: y = act(W x + b) for all B rows; one warp per output neuron, a float4 per lane per step.
//     The weight row is read from HBM once per call (batch rows after the first four hit L1), which is what bounds the
//     tail at small B: fc 512 x 1000 (2.05 MB) + heads (0.8 MB two heads / 1.7 MB single MLP).
//   odometry_out_kernel: the last Linear of each head (7 outputs per row), the division of the quaternion by the norm
//     of the WHOLE [B, 4] block (a quirk of the reference, :114) and quaternion -> T, in one CTA.
// Every sum has a fixed order (lane partials in k order, then an xor butterfly; the norm is one thread's loop), there
// are no atomics, so results are bit-identical from run to run and do not depend on B except through the norm.
#include <cuda_bf16.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <memory>

#include "common.cuh"
#include "dropout.cuh"
#include "projection.cuh"
#include "trunk.cuh"

namespace delora {

constexpr int kTailWarps = 8;
constexpr int kMaxLinear = 5;
constexpr int kMaxBatch = 1024;
constexpr int kHeadHidden = 100;

struct TailLinear {
    const float* w;        // [N, K] row-major
    const float* bias;     // [N]
    const float* x;        // [B, ldx]
    float* y;              // [B, ldy]
    int K, N, ldx, ldy;
};

__device__ __forceinline__ float tail_act(float v, int act) {
    if (act == 2) return tanhf(v);                          // torch.tanh on CUDA floats
    if (act == 1) return (v != v) ? v : (v < 0.0f ? 0.0f : v);   // torch.relu (clamp_min 0, NaN propagates)
    return v;
}

// Dot products of one weight row with nb <= 4 input rows; on return every lane holds the four sums.  Lane l adds
// k = 4l .. 4l+3, then 4l+128 ..., in order (vec) or k = l, l+32, ... (scalar), then the xor butterfly.
__device__ __forceinline__ void row_dot4(const float* __restrict__ w, const float* __restrict__ x, int ldx, int K, int nb,
                                         int lane, int vec, float acc[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = 0.0f;
    if (vec) {
#pragma unroll 4
        for (int k = lane * 4; k < K; k += 128) {
            const float4 wv = __ldg(reinterpret_cast<const float4*>(w + k));
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j < nb) {
                    const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (size_t)j * ldx + k));
                    acc[j] = fmaf(wv.x, xv.x, acc[j]);
                    acc[j] = fmaf(wv.y, xv.y, acc[j]);
                    acc[j] = fmaf(wv.z, xv.z, acc[j]);
                    acc[j] = fmaf(wv.w, xv.w, acc[j]);
                }
            }
        }
    } else {
        for (int k = lane; k < K; k += 32) {
            const float wv = __ldg(w + k);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (j < nb) acc[j] = fmaf(wv, __ldg(x + (size_t)j * ldx + k), acc[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
}

// y = act(W x + b) for two independent problems in one launch (the hidden layers of the two heads share one):
// warps [0, p0.N) compute p0's outputs, the next p1.N warps p1's.  kDrop (resnet.fc in a dropout training step, p1
// empty): y = act(keep * 1.25f * (W x + b)), element b * N + n of the fc mask.
template <bool kDrop>
__device__ __forceinline__ void linear_body(const TailLinear& p0, const TailLinear& p1, int B, int act_out, int vec,
                                            const DropoutCtr& drop) {
    const int lane = threadIdx.x & 31;
    int n = blockIdx.x * kTailWarps + (threadIdx.x >> 5);
    const bool second = n >= p0.N;
    const TailLinear p = second ? p1 : p0;
    if (second) n -= p0.N;
    if (n >= p.N) return;
    const float* __restrict__ w = p.w + (size_t)n * p.K;
    const float bn = __ldg(p.bias + n);
    for (int b0 = 0; b0 < B; b0 += 4) {
        const int nb = min(4, B - b0);
        float acc[4];
        row_dot4(w, p.x + (size_t)b0 * p.ldx, p.ldx, p.K, nb, lane, vec, acc);
        const float v = lane == 0 ? acc[0] : lane == 1 ? acc[1] : lane == 2 ? acc[2] : acc[3];
        if (lane < nb) {
            float z = v + bn;
            if (kDrop) {
                uint64_t seed, step;
                dropout_seed_step(drop, seed, step);
                z = dropout_keep(seed, step, kDropFc, (uint64_t)(b0 + lane) * p.N + n) ? z * kDropScale : 0.0f;
            }
            p.y[(size_t)(b0 + lane) * p.ldy + n] = tail_act(z, act_out);
        }
    }
}

__global__ void __launch_bounds__(kTailWarps * 32)
odometry_linear_kernel(TailLinear p0, TailLinear p1, int B, int act_out, int vec) {
    linear_body<false>(p0, p1, B, act_out, vec, DropoutCtr{nullptr, 0});
}

__global__ void __launch_bounds__(kTailWarps * 32)
odometry_linear_dropout_kernel(TailLinear p0, TailLinear p1, int B, int act_out, int vec, DropoutCtr drop) {
    linear_body<true>(p0, p1, B, act_out, vec, drop);
}

// The last layer of the heads (rot: 4 outputs, trans: 3) for every row b < B with want(b) (warp-uniform):
// s_out[b * 7 + o] = the quaternion (x, y, z, w), then the translation.  One warp per output, row_dot4 with nb = 1.
template <class Want>
__device__ __forceinline__ void head_outputs(const TailLinear& rot, const TailLinear& trans, int B, int vec, Want want,
                                             float* s_out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = warp; i < B * 7; i += kTailWarps) {
        const int b = i / 7, o = i - b * 7;
        if (!want(b)) continue;
        const TailLinear p = o < 4 ? rot : trans;
        const int n = o < 4 ? o : o - 4;
        float acc[4];
        row_dot4(p.w + (size_t)n * p.K, p.x + (size_t)b * p.ldx, p.ldx, p.K, 1, lane, vec, acc);
        if (lane == 0) s_out[i] = acc[0] + __ldg(p.bias + n);
    }
}

// Last layer of the heads, quaternion / ||quaternion block||_F, quaternion -> T.
// raw [B, 7] or NULL: the head outputs before the normalisation (quaternion, translation), which training keeps.
// kRescale (normalised models, src/deploy/deployer.py:344-346): T[:3, 3] of row b is then multiplied by factor[b].
template <bool kRescale>
__global__ void __launch_bounds__(kTailWarps * 32)
odometry_out_kernel(TailLinear rot, TailLinear trans, int B, int vec, float* __restrict__ T, float* __restrict__ raw,
                    const float* __restrict__ factor) {
    extern __shared__ float s_out[];                        // [B, 7]: quaternion (x, y, z, w), translation
    __shared__ float s_norm;
    head_outputs(rot, trans, B, vec, [](int) { return true; }, s_out);
    __syncthreads();
    if (raw)
        for (int i = threadIdx.x; i < B * 7; i += blockDim.x) raw[i] = s_out[i];
    if (threadIdx.x == 0) {                                 // torch.norm of the [B, 4] block: one ordered sum
        float ss = 0.0f;
        for (int b = 0; b < B; ++b)
            for (int j = 0; j < 4; ++j) ss = fmaf(s_out[b * 7 + j], s_out[b * 7 + j], ss);
        s_norm = sqrtf(ss);
    }
    __syncthreads();
    const float nrm = s_norm;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float* q = s_out + b * 7;
        float* t = T + (size_t)b * 16;
        quat_to_T_row(q[0] / nrm, q[1] / nrm, q[2] / nrm, q[3] / nrm, q[4], q[5], q[6], t);
        if (kRescale) {
            const float f = factor[b];
            t[3] = __fmul_rn(t[3], f); t[7] = __fmul_rn(t[7], f); t[11] = __fmul_rn(t[11], f);
        }
    }
}

__device__ __forceinline__ bool stream_active(const int32_t* __restrict__ active, int s) {
    return active == nullptr || active[s] != 0;
}

// counts[i] = active ? clamp(n_points[i], 0, n_stride) : 0 (active NULL: every scan is): the projection never reads
// past a scan's stride, and an inactive stream's scatter does no work
__global__ void odometry_counts_kernel(const int32_t* __restrict__ n_in, const int32_t* __restrict__ active, int n,
                                       int n_stride, int32_t* __restrict__ n_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) n_out[i] = stream_active(active, i) ? min(max(n_in[i], 0), n_stride) : 0;
}

// ---------------------------------------------------------------- the model: layer sequence + weight-blob offsets
struct Linear {
    int K, N;
    int64_t blob_w, blob_b;
};
struct Model {
    TrunkPlan t;                       // the trunk's filters open the blob
    int n_lin;
    Linear lin[kMaxLinear];            // two heads: rot1, rot2, trans1, trans2; single MLP: 5 layers
    Linear fc;
    int64_t blob_floats;
};

static int check_desc(const delora_odometry_desc* d, const char* who) {
    DELORA_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
    DELORA_CHECK_ARG((long long)d->H * d->W < (1ll << 27), "%s: bad image size H=%d W=%d", who, d->H, d->W);
    if (check_trunk(d->layers, d->H, d->W, who)) return 1;
    DELORA_CHECK_ARG(d->n_stride >= 1, "%s: n_stride=%d must be >= 1", who, d->n_stride);
    DELORA_CHECK_ARG(d->max_batch >= 1 && d->max_batch <= kMaxBatch, "%s: max_batch=%d must be in [1, %d]", who,
                     d->max_batch, kMaxBatch);
    DELORA_CHECK_ARG(d->act == 1 || d->act == 2, "%s: act=%d must be 1 (relu) or 2 (tanh)", who, d->act);
    DELORA_CHECK_ARG(d->resnet_outputs >= 1 && d->resnet_outputs <= 65536, "%s: resnet_outputs=%d must be in [1, 65536]",
                     who, d->resnet_outputs);
    DELORA_CHECK_ARG(d->single_mlp == 0 || d->single_mlp == 1, "%s: single_mlp=%d must be 0 or 1", who, d->single_mlp);
    DELORA_CHECK_ARG(isfinite(d->hfov0) && isfinite(d->hfov1) && isfinite(d->vfov0) && isfinite(d->vfov1) &&
                     d->hfov1 > d->hfov0 && d->vfov1 > d->vfov0, "%s: bad field of view", who);
    return 0;
}

// Walks the model in state_dict order (src/models/resnet_modified.py:49-66 + model.py:58-84).  A pure function of the
// descriptor.
static void plan_model(const delora_odometry_desc* d, Model* m) {
    memset(m, 0, sizeof(Model));
    plan_trunk(d->layers, d->H, d->W, &m->t);
    int64_t blob = m->t.conv_floats;
    auto add_lin = [&](Linear& l, int K, int N) {
        l.K = K; l.N = N; l.blob_w = blob; blob += (int64_t)K * N; l.blob_b = blob; blob += N;
    };
    const int nout = d->resnet_outputs;
    add_lin(m->fc, 512, nout);
    if (d->single_mlp) {
        static const int dims[6] = {0, 512, 512, 256, 64, 7};
        int k = nout;
        for (int i = 1; i < 6; ++i) { add_lin(m->lin[m->n_lin++], k, dims[i]); k = dims[i]; }
    } else {
        add_lin(m->lin[0], nout, kHeadHidden); add_lin(m->lin[1], kHeadHidden, 4);     // fully_connected_rotation
        add_lin(m->lin[2], nout, kHeadHidden); add_lin(m->lin[3], kHeadHidden, 3);     // fully_connected_translation
        m->n_lin = 4;
    }
    m->blob_floats = blob;
}

// ---------------------------------------------------------------- workspace sections
// Each workspace kind (pairs / push, streams, training) has a plan: the Model plus the byte offsets of its own
// layout, built from the sections below.  Every buffer starts on a 256-byte boundary.

// The frame section: n_scans projected scans (depth keys, index map, clamped counts, fp32 images), n_cached cached
// previous images and, with has_prev, one "has a previous frame" flag per cached image.  The depth keys are sized for
// images key_w wide (>= W): the training step projects at the preprocessing width in them as well.
struct Frames {
    size_t keys, keys_bytes, index_map, counts, images;
    size_t prev_image;                 // n_cached > 0 only
    size_t has_prev;                   // with has_prev only
};

static Frames plan_frames(const delora_odometry_desc* d, int n_scans, int n_cached, bool has_prev, int key_w,
                          size_t& off) {
    const size_t HW = (size_t)d->H * d->W;
    Frames f;
    memset(&f, 0, sizeof(f));
    f.keys_bytes = (size_t)n_scans * d->H * key_w * 8;
    f.keys = take(off, f.keys_bytes);
    f.index_map = take(off, (size_t)n_scans * HW * 4);
    f.counts = take(off, (size_t)n_scans * 4);
    f.images = take(off, (size_t)n_scans * 4 * HW * 4);
    if (n_cached > 0) f.prev_image = take(off, (size_t)n_cached * 4 * HW * 4);
    if (has_prev) f.has_prev = take(off, (size_t)n_cached * 4);
    return f;
}

// The pairs / push and the streams workspaces: the trunk's inference buffers and its weight section without the
// flipped filters.  The tail reads fp32 copies of its weights (256-byte aligned).
struct InferPlan {
    Model m;
    Frames f;
    TrunkActs t;
    size_t pooled, fc_out, hid[2];
    TrunkWeights w;
    size_t fc_w, fc_b, lin_w[kMaxLinear], lin_b[kMaxLinear];
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
    size_t total;
};

// The frame section (see plan_frames), then the trunk and tail sections that run at up to B = max_batch
static void plan_inference(const delora_odometry_desc* d, int n_scans, int n_cached, bool has_prev, InferPlan* p) {
    memset(p, 0, sizeof(InferPlan));
    plan_model(d, &p->m);
    const Model& m = p->m;
    const int MB = d->max_batch, nout = d->resnet_outputs;
    size_t off = 0;
    p->f = plan_frames(d, n_scans, n_cached, has_prev, d->W, off);
    p->t = plan_trunk_acts(m.t, MB, false, off);
    p->pooled = take(off, (size_t)MB * 512 * 4);
    p->fc_out = take(off, (size_t)MB * nout * 4);
    p->hid[0] = take(off, (size_t)MB * 512 * 4);
    p->hid[1] = take(off, (size_t)MB * 512 * 4);
    p->w = plan_trunk_weights(m.t, false, off);
    p->fc_w = take(off, (size_t)m.fc.K * m.fc.N * 4);
    p->fc_b = take(off, (size_t)m.fc.N * 4);
    for (int i = 0; i < m.n_lin; ++i) {
        p->lin_w[i] = take(off, (size_t)m.lin[i].K * m.lin[i].N * 4);
        p->lin_b[i] = take(off, (size_t)m.lin[i].N * 4);
    }
    p->total = off;
}

// pairs / push: 2 * max_batch scans and the one cached image of _push
static void make_infer_plan(const delora_odometry_desc* d, InferPlan* p) {
    plan_inference(d, 2 * d->max_batch, 1, false, p);
}

// The streams workspace kinds.  Each one is the layout of the kind it extends with its own sections appended, so no
// offset of that layout moves and _streams_load_weights and _streams_reset work on every kind.
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
enum class Streams { plain, residual, normalized, pre, info, pre_info };

static void make_streams_plan(const delora_odometry_desc* d, Streams kind, InferPlan* p) {
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

// Where the tail reads its weights and writes its activations.  Inference: the workspace copies of the weights and two
// hidden buffers the layers alternate between; training: the fp32 master blob and one buffer per layer (the backward
// reads every activation).
struct TailIO {
    const float* fc_w;
    const float* fc_b;
    const float* w[kMaxLinear];
    const float* b[kMaxLinear];
    float* fc_out;                     // [B, nout]: act(resnet.fc(pooled))
    float* hid[kMaxLinear];            // output of lin[i], i < n_lin - 1; two heads: hid[0] = [rot1 | trans1], ld 200
    float* raw;                        // [B, 7] head outputs before the normalisation, or NULL
};

static TailLinear tail_args(const Linear& l, const float* w, const float* bias, const float* x, int ldx, float* y, int ldy) {
    TailLinear t;
    t.w = w;
    t.bias = bias;
    t.x = x; t.y = y; t.K = l.K; t.N = l.N; t.ldx = ldx; t.ldy = ldy;
    return t;
}

static TailIO inference_tail_io(const InferPlan& p, char* ws) {
    TailIO io;
    memset(&io, 0, sizeof(io));
    auto f = [&](size_t off) { return reinterpret_cast<float*>(ws + off); };
    io.fc_w = f(p.fc_w); io.fc_b = f(p.fc_b);
    for (int i = 0; i < p.m.n_lin; ++i) { io.w[i] = f(p.lin_w[i]); io.b[i] = f(p.lin_b[i]); }
    io.fc_out = f(p.fc_out);
    for (int i = 0; i < kMaxLinear; ++i) io.hid[i] = f(p.hid[i & 1]);
    return io;
}

// Whether row_dot4 may read t with float4 loads: K and ldx multiples of 4, w and x 16-byte aligned.  The workspace
// copies of inference are; the master blob of training puts a layer's weights at a float offset that is a multiple of
// 4 only when resnet_outputs is.
static int tail_vec(const TailLinear& t) {
    return t.K % 4 == 0 && t.ldx % 4 == 0 && (uintptr_t)t.w % 16 == 0 && (uintptr_t)t.x % 16 == 0;
}

// resnet.fc and the heads' hidden layers for B rows; rot / trans: the heads' last layers, for the output kernel
// drop.ctr non-NULL: resnet.fc's output goes through the fc dropout before the activation
static int run_tail_hidden(const Model& m, const TailIO& io, int act, const float* pooled, int B, TailLinear* rot_out,
                           TailLinear* trans_out, cudaStream_t st, DropoutCtr drop = DropoutCtr{nullptr, 0}) {
    float* fc_out = io.fc_out;
    TailLinear none;
    memset(&none, 0, sizeof(none));
    auto linear = [&](const TailLinear& a, const TailLinear& b) {
        const int vec = tail_vec(a) && (b.N == 0 || tail_vec(b));
        const int warps = a.N + b.N;
        odometry_linear_kernel<<<(warps + kTailWarps - 1) / kTailWarps, kTailWarps * 32, 0, st>>>(a, b, B, act, vec);
        DELORA_CHECK_LAUNCH("odometry_linear_kernel");
        return 0;
    };
    int rc;
    const int nout = m.fc.N;
    if (drop.ctr) {                                         // act(dropout(resnet.fc(x)))
        const TailLinear fc = tail_args(m.fc, io.fc_w, io.fc_b, pooled, 512, fc_out, nout);
        odometry_linear_dropout_kernel<<<(fc.N + kTailWarps - 1) / kTailWarps, kTailWarps * 32, 0, st>>>(
            fc, none, B, act, tail_vec(fc), drop);
        DELORA_CHECK_LAUNCH("odometry_linear_dropout_kernel");
    } else if ((rc = linear(tail_args(m.fc, io.fc_w, io.fc_b, pooled, 512, fc_out, nout), none))) {   // act(resnet.fc(x))
        return rc;
    }
    TailLinear rot, trans;
    if (m.n_lin == 4) {
        // hidden layers of both heads in one launch: hid[0] = [act(rot1 h) | act(trans1 h)], row stride 200
        const int ld = 2 * kHeadHidden;
        float* hid = io.hid[0];
        if ((rc = linear(tail_args(m.lin[0], io.w[0], io.b[0], fc_out, nout, hid, ld),
                         tail_args(m.lin[2], io.w[2], io.b[2], fc_out, nout, hid + kHeadHidden, ld)))) return rc;
        rot = tail_args(m.lin[1], io.w[1], io.b[1], hid, ld, nullptr, 0);
        trans = tail_args(m.lin[3], io.w[3], io.b[3], hid + kHeadHidden, ld, nullptr, 0);
    } else {
        const float* x = fc_out;
        int ldx = nout;
        for (int i = 0; i < m.n_lin - 1; ++i) {
            float* y = io.hid[i];
            if ((rc = linear(tail_args(m.lin[i], io.w[i], io.b[i], x, ldx, y, m.lin[i].N), none))) return rc;
            x = y; ldx = m.lin[i].N;
        }
        // fully_connected_rot_trans's last layer: rows 0..3 -> rotation, rows 4..6 -> translation
        const int last = m.n_lin - 1;
        const Linear& l = m.lin[last];
        rot = tail_args(l, io.w[last], io.b[last], x, ldx, nullptr, 0);
        rot.N = 4;
        trans = rot;
        trans.w = rot.w + 4 * (size_t)l.K;
        trans.bias = rot.bias + 4;
        trans.N = 3;
    }
    *rot_out = rot;
    *trans_out = trans;
    return 0;
}

// factor [B] or NULL: multiply each row's translation by its pair's normalisation factor
static int run_tail(const Model& m, const TailIO& io, int act, const float* pooled, int B, float* T, cudaStream_t st,
                    const float* factor = nullptr, DropoutCtr drop = DropoutCtr{nullptr, 0}) {
    TailLinear rot, trans;
    const int rc = run_tail_hidden(m, io, act, pooled, B, &rot, &trans, st, drop);
    if (rc) return rc;
    const int vec = tail_vec(rot) && tail_vec(trans);
    const size_t smem = (size_t)B * 7 * sizeof(float);
    if (factor)
        odometry_out_kernel<true><<<1, kTailWarps * 32, smem, st>>>(rot, trans, B, vec, T, io.raw, factor);
    else
        odometry_out_kernel<false><<<1, kTailWarps * 32, smem, st>>>(rot, trans, B, vec, T, io.raw, nullptr);
    DELORA_CHECK_LAUNCH("odometry_out_kernel");
    return 0;
}

// counts = the clamped n_points of n scans (active: see odometry_counts_kernel)
static int clamp_counts(const Frames& f, char* ws, const int32_t* n_points, const int32_t* active, int n, int n_stride,
                        cudaStream_t st) {
    odometry_counts_kernel<<<(n + 255) / 256, 256, 0, st>>>(n_points, active, n, n_stride,
                                                            reinterpret_cast<int32_t*>(ws + f.counts));
    DELORA_CHECK_LAUNCH("odometry_counts_kernel");
    return 0;
}

static int project(const Frames& f, const delora_odometry_desc* d, char* ws, const float* points, const int32_t* n_points,
                   const int32_t* active, int n_scans, cudaStream_t st) {
    const int rc = clamp_counts(f, ws, n_points, active, n_scans, d->n_stride, st);
    if (rc) return rc;
    return delora_project_fwd(points, reinterpret_cast<int32_t*>(ws + f.counts), n_scans, 3, d->n_stride, d->H, d->W,
                              d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0, reinterpret_cast<uint64_t*>(ws + f.keys),
                              reinterpret_cast<float*>(ws + f.images), reinterpret_cast<int32_t*>(ws + f.index_map), st);
}

// The 2B scans of B pairs divided by their pair's normalisation factor, then projected: the clamped counts, the factor
// of every pair into factor [B], and the scaled instantiations of the projection's two passes.
static int project_normalized(const Frames& f, const delora_odometry_desc* d, char* ws, const float* points,
                              const int32_t* n_points, int B, float* factor, cudaStream_t st) {
    int rc = clamp_counts(f, ws, n_points, nullptr, 2 * B, d->n_stride, st);
    if (rc) return rc;
    const int32_t* counts = reinterpret_cast<const int32_t*>(ws + f.counts);
    if ((rc = launch_normalization_factors(points, counts, B, d->n_stride, factor, st))) return rc;
    const GridParams g = make_grid(d->H, d->W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0);
    return project_fwd(points, counts, 2 * B, 3, d->n_stride, g, reinterpret_cast<uint64_t*>(ws + f.keys),
                       reinterpret_cast<float*>(ws + f.images), reinterpret_cast<int32_t*>(ws + f.index_map), factor, B,
                       st);
}

// The loss and normals' settings of delora_odometry_train_params and delora_odometry_residual_params
static int check_icp_params(float lambda_po2pl, uint32_t loss_flags, int nb_h, int nb_w, float epsilon_range,
                            int min_neighbors, const char* who) {
    DELORA_CHECK_ARG(isfinite(lambda_po2pl), "%s: lambda_po2pl=%g must be finite", who, (double)lambda_po2pl);
    DELORA_CHECK_ARG((loss_flags & (DELORA_LOSS_PO2PO | DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL)) != 0,
                     "%s: loss_flags=0x%x sets no loss bit", who, loss_flags);
    DELORA_CHECK_ARG(nb_h >= 1 && nb_h % 2 == 1, "%s: nb_h=%d must be odd and positive", who, nb_h);
    DELORA_CHECK_ARG(nb_w >= 1 && nb_w % 2 == 1, "%s: nb_w=%d must be odd and positive", who, nb_w);
    DELORA_CHECK_ARG(isfinite(epsilon_range) && epsilon_range >= 0.0f, "%s: epsilon_range=%g must be >= 0", who,
                     (double)epsilon_range);
    DELORA_CHECK_ARG(min_neighbors >= 0, "%s: min_neighbors=%d must be >= 0", who, min_neighbors);
    return 0;
}

// Every workspace starts zeroed, with its depth keys at all ones (the projection's empty key).  from > 0: only bytes
// [from, total) are zeroed (a training workspace's geometry section, delora_odometry_train_use_geometry).
static int init_workspace(const Frames& f, size_t total, void* workspace, cudaStream_t st, const char* who,
                          size_t from = 0) {
    char* ws = (char*)workspace;
    cudaError_t e = cudaMemsetAsync(ws + from, 0, total - from, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(ws + f.keys, 0xFF, f.keys_bytes, st);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

// The bf16 filters of the weight section w from the fp32 weight blob
static int prep_blob_weights(const Model& m, const TrunkWeights& w, char* ws, const float* blob, cudaStream_t st,
                             const char* who) {
    const float* src[kMaxConv];
    for (int i = 0; i < m.t.n_conv; ++i) src[i] = blob + m.t.conv[i].blob;
    return prep_trunk_weights(m.t, w, ws, src, st, who);
}

static int load_weights(const InferPlan& p, const float* weights, void* workspace, cudaStream_t st, const char* who) {
    char* ws = (char*)workspace;
    const Model& m = p.m;
    int rc = prep_blob_weights(m, p.w, ws, weights, st, who);
    if (rc) return rc;
    auto copy = [&](size_t dst, int64_t src, int64_t n) {
        return cudaMemcpyAsync(ws + dst, weights + src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, st);
    };
    cudaError_t e = copy(p.fc_w, m.fc.blob_w, (int64_t)m.fc.K * m.fc.N);
    if (e == cudaSuccess) e = copy(p.fc_b, m.fc.blob_b, m.fc.N);
    for (int i = 0; i < m.n_lin && e == cudaSuccess; ++i) {
        e = copy(p.lin_w[i], m.lin[i].blob_w, (int64_t)m.lin[i].K * m.lin[i].N);
        if (e == cudaSuccess) e = copy(p.lin_b[i], m.lin[i].blob_b, m.lin[i].N);
    }
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

}  // namespace delora

using namespace delora;

extern "C" int64_t delora_odometry_weight_floats(const delora_odometry_desc* d) {
    if (check_desc(d, "delora_odometry_weight_floats")) return -1;
    Model m;
    plan_model(d, &m);
    return m.blob_floats;
}

extern "C" int64_t delora_odometry_workspace_bytes(const delora_odometry_desc* d) {
    if (check_desc(d, "delora_odometry_workspace_bytes")) return -1;
    InferPlan p;
    make_infer_plan(d, &p);
    return (int64_t)p.total;
}

extern "C" int delora_odometry_init(const delora_odometry_desc* d, void* workspace, void* stream) {
    if (check_desc(d, "delora_odometry_init")) return 1;
    DELORA_CHECK_ARG(workspace, "delora_odometry_init: null workspace");
    InferPlan p;
    make_infer_plan(d, &p);
    return init_workspace(p.f, p.total, workspace, (cudaStream_t)stream, "delora_odometry_init");
}

extern "C" int delora_odometry_load_weights(const delora_odometry_desc* d, const float* weights, void* workspace,
                                            void* stream) {
    if (check_desc(d, "delora_odometry_load_weights")) return 1;
    DELORA_CHECK_ARG(weights && workspace, "delora_odometry_load_weights: null pointer");
    InferPlan p;
    make_infer_plan(d, &p);
    return load_weights(p, weights, workspace, (cudaStream_t)stream, "delora_odometry_load_weights");
}

// delora_odometry_pairs and, with factor non-NULL, delora_odometry_pairs_normalized (arguments checked by the caller)
static int run_pairs(const delora_odometry_desc* d, const float* points, const int32_t* n_points, int B, void* workspace,
                     float* T, float* pooled, float* factor, cudaStream_t st, const char* who) {
    InferPlan p;
    make_infer_plan(d, &p);
    char* ws = (char*)workspace;
    float* images = reinterpret_cast<float*>(ws + p.f.images);
    const size_t img = (size_t)4 * d->H * d->W;
    float* pooled_ws = reinterpret_cast<float*>(ws + p.pooled);
    int rc;
    if (factor) rc = project_normalized(p.f, d, ws, points, n_points, B, factor, st);
    else rc = project(p.f, d, ws, points, n_points, nullptr, 2 * B, st);
    if (rc) return rc;
    if ((rc = trunk_input(p.m.t, p.t, ws, images, images + (size_t)B * img, B, st))) return rc;
    if ((rc = trunk_forward(p.m.t, p.t, ws, p.w, ws, d->act, B, pooled_ws, nullptr, st))) return rc;
    if ((rc = run_tail(p.m, inference_tail_io(p, ws), d->act, pooled_ws, B, T, st, factor))) return rc;
    if (pooled) {
        const cudaError_t e = cudaMemcpyAsync(pooled, pooled_ws, (size_t)B * 512 * sizeof(float), cudaMemcpyDeviceToDevice, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    }
    return 0;
}

extern "C" int delora_odometry_pairs(const delora_odometry_desc* d, const float* points, const int32_t* n_points, int B,
                                     void* workspace, float* T, float* pooled, void* stream) {
    if (check_desc(d, "delora_odometry_pairs")) return 1;
    DELORA_CHECK_ARG(points && n_points && workspace && T, "delora_odometry_pairs: null pointer");
    DELORA_CHECK_ARG(B >= 1 && B <= d->max_batch, "delora_odometry_pairs: B=%d outside [1, max_batch=%d]", B,
                     d->max_batch);
    return run_pairs(d, points, n_points, B, workspace, T, pooled, nullptr, (cudaStream_t)stream, "delora_odometry_pairs");
}

extern "C" int delora_odometry_pairs_normalized(const delora_odometry_desc* d, const float* points,
                                                const int32_t* n_points, int B, void* workspace, float* T,
                                                float* pooled, float* factor, void* stream) {
    const char* who = "delora_odometry_pairs_normalized";
    if (check_desc(d, who)) return 1;
    DELORA_CHECK_ARG(points, "%s: null points", who);
    DELORA_CHECK_ARG(n_points, "%s: null n_points", who);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    DELORA_CHECK_ARG(T, "%s: null T", who);
    DELORA_CHECK_ARG(factor, "%s: null factor", who);
    DELORA_CHECK_ARG(B >= 1 && B <= d->max_batch, "%s: B=%d outside [1, max_batch=%d]", who, B, d->max_batch);
    return run_pairs(d, points, n_points, B, workspace, T, pooled, factor, (cudaStream_t)stream, who);
}

extern "C" int delora_odometry_push(const delora_odometry_desc* d, const float* points, const int32_t* n_points,
                                    void* workspace, float* T, void* stream) {
    if (check_desc(d, "delora_odometry_push")) return 1;
    DELORA_CHECK_ARG(points && n_points && workspace, "delora_odometry_push: null pointer");
    InferPlan p;
    make_infer_plan(d, &p);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    float* image = reinterpret_cast<float*>(ws + p.f.images);
    float* prev = reinterpret_cast<float*>(ws + p.f.prev_image);
    int rc;
    if ((rc = project(p.f, d, ws, points, n_points, nullptr, 1, st))) return rc;
    if (T) {
        float* pooled_ws = reinterpret_cast<float*>(ws + p.pooled);
        if ((rc = trunk_input(p.m.t, p.t, ws, prev, image, 1, st))) return rc;
        if ((rc = trunk_forward(p.m.t, p.t, ws, p.w, ws, d->act, 1, pooled_ws, nullptr, st))) return rc;
        if ((rc = run_tail(p.m, inference_tail_io(p, ws), d->act, pooled_ws, 1, T, st))) return rc;
    }
    const cudaError_t e = cudaMemcpyAsync(prev, image, (size_t)4 * d->H * d->W * sizeof(float), cudaMemcpyDeviceToDevice, st);
    DELORA_CHECK_ARG(e == cudaSuccess, "delora_odometry_push: %s", cudaGetErrorString(e));
    return 0;
}

// ================================================================================================ streams
// delora_odometry_streams_push: S = max_batch independent streams in one workspace.  Per tick: the masked count clamp,
// the projection of the S new frames (inactive streams project 0 points), the fused input conversion + cache update,
// the trunk and the fc / hidden layers at B = S (the launches of _pairs), and the per-row output kernel.  A stream's row
// goes through the same instructions as _push's batch-1 call: the trunk's kernels and the tail's row_dot4 sum a row
// in an order that does not depend on B, and the output kernel divides each quaternion by its own norm, which at B = 1
// is the block norm of odometry_out_kernel.  Every launch is unconditional; activity and per-stream state are read on
// the device only.
namespace delora {

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

// The last layer of the heads and quaternion -> T for every stream with an active frame and a previous one; each
// quaternion is divided by the norm of its own row, with the instructions odometry_out_kernel runs at B = 1 (row_dot4
// with nb = 1, fmaf over the 4 components in order, sqrtf, the four divisions, quat_to_T_row).  valid[s] = 1 for those
// streams, 0 for the others (whose T row is not written); then every active stream has a previous frame.
// kRescale (delora_odometry_streams_push_normalized): T[:3, 3] of a valid row is then multiplied by factor[s] with the
// instructions of odometry_out_kernel<true>; factor_out[s] = factor[s] where valid, 0 elsewhere; and the count of this
// tick's frame, counts[S + s], becomes the count of each active stream's last frame, counts[2S + s].
// raw [S, 7] or NULL (delora_odometry_streams_push_adapt): the head outputs of the valid rows, which the backward reads;
// n_valid or NULL: the number of valid streams.
template <bool kRescale>
__global__ void __launch_bounds__(kTailWarps * 32)
odometry_streams_out_kernel(TailLinear rot, TailLinear trans, int S, int vec, const int32_t* __restrict__ active,
                            int32_t* __restrict__ has_prev, float* __restrict__ T, int32_t* __restrict__ valid,
                            const float* __restrict__ factor, float* __restrict__ factor_out,
                            int32_t* __restrict__ counts, float* __restrict__ raw = nullptr,
                            int32_t* __restrict__ n_valid = nullptr) {
    extern __shared__ float s_out[];                        // [S, 7]: quaternion (x, y, z, w), translation
    head_outputs(rot, trans, S, vec, [&](int b) { return stream_active(active, b) && has_prev[b] != 0; }, s_out);
    __syncthreads();
    for (int b = threadIdx.x; b < S; b += blockDim.x) {
        const bool act = stream_active(active, b);
        const bool ok = act && has_prev[b] != 0;
        if (ok) {
            const float* q = s_out + b * 7;
            float ss = 0.0f;
            for (int j = 0; j < 4; ++j) ss = fmaf(q[j], q[j], ss);
            const float nrm = sqrtf(ss);
            float* t = T + (size_t)b * 16;
            quat_to_T_row(q[0] / nrm, q[1] / nrm, q[2] / nrm, q[3] / nrm, q[4], q[5], q[6], t);
            if (kRescale) {
                const float f = factor[b];
                t[3] = __fmul_rn(t[3], f); t[7] = __fmul_rn(t[7], f); t[11] = __fmul_rn(t[11], f);
            }
            if (raw)
                for (int j = 0; j < 7; ++j) raw[b * 7 + j] = q[j];
        }
        valid[b] = ok ? 1 : 0;
        if (kRescale) {
            factor_out[b] = ok ? factor[b] : 0.0f;
            if (act) counts[2 * S + b] = counts[S + b];
        }
        if (act) has_prev[b] = 1;
    }
    if (n_valid) {
        __syncthreads();
        if (threadIdx.x == 0) {
            int n = 0;
            for (int b = 0; b < S; ++b) n += valid[b];
            *n_valid = n;
        }
    }
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
    InferPlan p;
    make_streams_plan(d, kind, &p);
    return (int64_t)p.total;
}

// The n cells of the cached grids at offsets pts / nrm start empty: the target of a stream that has not had a frame yet
static int clear_grids(char* ws, size_t pts, size_t nrm, size_t n, cudaStream_t st) {
    odometry_streams_grid_clear_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        reinterpret_cast<float4*>(ws + pts), reinterpret_cast<float4*>(ws + nrm), n);
    DELORA_CHECK_LAUNCH("odometry_streams_grid_clear_kernel");
    return 0;
}

// The residual, information and recipe kinds' ICP scratch is zeroed here, once, and their cached grids start empty
static int streams_init(const delora_odometry_desc* d, Streams kind, void* workspace, cudaStream_t st, const char* who) {
    if (check_streams_desc(d, kind, who)) return 1;
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    InferPlan p;
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
static int check_tick(const float* points, const int32_t* n_points, const void* workspace, const float* T,
                      const int32_t* valid, const float* extra, const char* extra_name, const char* who) {
    DELORA_CHECK_ARG(points, "%s: null points", who);
    DELORA_CHECK_ARG(n_points, "%s: null n_points", who);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    DELORA_CHECK_ARG(T, "%s: null T", who);
    DELORA_CHECK_ARG(valid, "%s: null valid", who);
    DELORA_CHECK_ARG(!extra_name || extra, "%s: null %s", who, extra_name);
    return 0;
}

// The residual's settings: loss_flags may have the ICP losses and DELORA_NORMAL_LINEAR and, with scaling (the recipe
// streams), DELORA_TRAIN_NORMALIZATION_SCALING
static int check_residual_params(const delora_odometry_residual_params* rp, bool scaling, const char* who) {
    DELORA_CHECK_ARG(rp, "%s: null residual_params", who);
    if (check_icp_params(rp->lambda_po2pl, rp->loss_flags, rp->nb_h, rp->nb_w, rp->epsilon_range, rp->min_neighbors, who))
        return 1;
    const uint32_t bits = DELORA_LOSS_PO2PO | DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL | DELORA_NORMAL_LINEAR |
                          (scaling ? DELORA_TRAIN_NORMALIZATION_SCALING : 0u);
    DELORA_CHECK_ARG((rp->loss_flags & ~bits) == 0u, "%s: loss_flags=0x%x has a bit other than %s", who, rp->loss_flags,
                     scaling ? "the ICP losses, DELORA_NORMAL_LINEAR and DELORA_TRAIN_NORMALIZATION_SCALING"
                             : "the ICP losses and DELORA_NORMAL_LINEAR");
    return 0;
}

// The model at B = S on the trunk input of t: the trunk into pooled, the tail's hidden layers and
// odometry_streams_out_kernel<kRescale>, which reads io.raw (see the kernel for its other arguments)
template <bool kRescale>
static int streams_forward(const Model& m, const TailIO& io, const TrunkActs& t, const TrunkWeights& w, char* ws,
                           int act, float* pooled, int S, const int32_t* active, int32_t* has_prev, float* T,
                           int32_t* valid, const float* factor, float* factor_out, int32_t* counts, int32_t* n_valid,
                           cudaStream_t st) {
    int rc;
    if ((rc = trunk_forward(m.t, t, ws, w, ws, act, S, pooled, nullptr, st))) return rc;
    TailLinear rot, trans;
    if ((rc = run_tail_hidden(m, io, act, pooled, S, &rot, &trans, st))) return rc;
    odometry_streams_out_kernel<kRescale><<<1, kTailWarps * 32, (size_t)S * 7 * sizeof(float), st>>>(
        rot, trans, S, tail_vec(rot) && tail_vec(trans), active, has_prev, T, valid, factor, factor_out, counts, io.raw,
        n_valid);
    DELORA_CHECK_LAUNCH(kRescale ? "odometry_streams_out_kernel<true>" : "odometry_streams_out_kernel");
    return 0;
}

// The ICP entry point whose work icp_dense_launch does with these info and factor pointers: the name its refusals give
static const char* icp_entry(const float* info, const float* factor) {
    return !info ? "delora_icp_dense_fwd_bwd" : factor ? "delora_icp_dense_information_scaled"
                                                       : "delora_icp_dense_information";
}

// The ICP at B = S on a residual or recipe plan's H x W grids: source pts_grid moved by T12, target prev_pts_grid,
// into its losses and grad_T; on an information plan (p.info set) also into its information rows, in metres with the
// pair factors of a normalised recipe (factor non-NULL).  The recipe's DELORA_TRAIN_NORMALIZATION_SCALING is not an
// ICP bit.
static int streams_icp(const delora_odometry_desc* d, const delora_odometry_residual_params* rp, const InferPlan& p,
                       char* ws, const float* factor, cudaStream_t st) {
    auto f = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
    auto f4 = [&](size_t o) { return reinterpret_cast<delora_f4*>(ws + o); };
    const uint32_t flags = rp->loss_flags & ~DELORA_TRAIN_NORMALIZATION_SCALING;
    float* info = p.info ? f(p.info) : nullptr;
    if (!info) factor = nullptr;
    return icp_dense_launch(f4(p.pts_grid), f4(p.nrm_grid), f(p.T12), f4(p.prev_pts_grid), f4(p.prev_nrm_grid),
                            d->max_batch, d->H, d->W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, rp->lambda_po2pl, flags,
                            f(p.losses), f(p.grad_T), f(p.icp), info, info ? f(p.info_scratch) : nullptr, factor, st,
                            icp_entry(info, factor));
}

// out [S, kRow] = the rows [S, kRow] at `rows` of the valid streams, zeros for the others
template <int kRow>
static int streams_rows_out(const int32_t* valid, int S, const float* rows, float* out, cudaStream_t st) {
    odometry_streams_rows_kernel<kRow><<<(S * kRow + 255) / 256, 256, 0, st>>>(valid, S, rows, out);
    DELORA_CHECK_LAUNCH(kRow == DELORA_INFO_ROW ? "odometry_streams_rows_kernel<DELORA_INFO_ROW>"
                                                : "odometry_streams_rows_kernel<DELORA_LOSS_ROW>");
    return 0;
}

// delora_odometry_streams_reset and _streams_adapt_reset, on the has_prev flags at that offset
static int reset_streams(const delora_odometry_desc* d, const int32_t* mask, void* workspace, size_t has_prev,
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
    InferPlan p;
    make_streams_plan(d, Streams::plain, &p);
    return load_weights(p, weights, workspace, (cudaStream_t)stream, who);
}

// delora_odometry_streams_push (rp NULL), delora_odometry_streams_push_residual and, with info, _streams_push_info
// (arguments checked by the callers)
static int run_streams_push(const delora_odometry_desc* d, const delora_odometry_residual_params* rp, const float* points,
                            const int32_t* n_points, const int32_t* active, void* workspace, float* T, int32_t* valid,
                            float* losses, float* info, cudaStream_t st) {
    InferPlan p;
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
        if ((rc = delora_project_normals_fwd(points, reinterpret_cast<int32_t*>(ws + p.f.counts), S, 3, d->n_stride, H, W,
                                             d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0,
                                             reinterpret_cast<uint64_t*>(ws + p.f.keys), cur,
                                             reinterpret_cast<int32_t*>(ws + p.f.index_map), rp->nb_h, rp->nb_w,
                                             rp->epsilon_range, rp->min_neighbors,
                                             reinterpret_cast<delora_f4*>(pts_grid), reinterpret_cast<delora_f4*>(nrm_grid),
                                             nullptr, st))) return rc;
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
    if ((rc = streams_forward<false>(p.m, inference_tail_io(p, ws), p.t, p.w, ws, d->act,
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
    return info ? streams_rows_out<DELORA_INFO_ROW>(valid, S, reinterpret_cast<float*>(ws + p.info), info, st) : 0;
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
    InferPlan p;
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
    return streams_forward<true>(p.m, inference_tail_io(p, ws), p.t, p.w, ws, d->act,
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
    InferPlan p;
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
    if ((rc = delora_project_normals_fwd(points, reinterpret_cast<int32_t*>(ws + p.f.counts), S, 3, d->n_stride, H, Wp,
                                         d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0,
                                         reinterpret_cast<uint64_t*>(ws + p.pre_keys), f(p.pre_image),
                                         reinterpret_cast<int32_t*>(ws + p.pre_index_map), rp->nb_h, rp->nb_w,
                                         rp->epsilon_range, rp->min_neighbors, pre_cur_pts, pre_cur_nrm, nullptr, st)))
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
    if ((rc = streams_forward<false>(p.m, inference_tail_io(p, ws), p.t, p.w, ws, d->act, f(p.pooled), S, active,
                                     has_prev, f(p.T16), valid, nullptr, nullptr, nullptr, nullptr, st))) return rc;
    int per_stream = HWp > HW ? HWp : HW;
    if (per_stream < 16) per_stream = 16;
    const size_t cells = (size_t)S * per_stream;
    odometry_streams_pre_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, st>>>(
        f(p.T16), factor, active, valid, S, HW, HWp, T, f(p.T12), factor_out, reinterpret_cast<float4*>(ws + p.pts_grid),
        reinterpret_cast<float4*>(ws + p.nrm_grid), reinterpret_cast<const float4*>(pre_cur_pts),
        reinterpret_cast<const float4*>(pre_cur_nrm), reinterpret_cast<float4*>(pre_prev_pts),
        reinterpret_cast<float4*>(pre_prev_nrm));
    DELORA_CHECK_LAUNCH("odometry_streams_pre_kernel");
    if ((rc = streams_icp(d, rp, p, ws, factor, st))) return rc;
    if ((rc = streams_rows_out<DELORA_LOSS_ROW>(valid, S, f(p.losses), losses, st))) return rc;
    return info ? streams_rows_out<DELORA_INFO_ROW>(valid, S, f(p.info), info, st) : 0;
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
    InferPlan p;
    make_streams_plan(d, Streams::plain, &p);
    return reset_streams(d, mask, workspace, p.f.has_prev, stream, who);
}

// ================================================================================================ training
// delora_odometry_train_step: projection + normals of the 2B scans (with w_pre > 0: at H x w_pre, then re-projected at
// H x W by delora_project_grids_fwd), the trunk forward keeping its activations (trunk.cuh), the tail forward keeping
// its activations, the dense ICP losses with dL/dT, the tail backward (below), the trunk backward, one Adam update of
// the fp32 master blob and one re-prep of the bf16 filters from it.  Weight gradients land in a gradient blob with
// the layout of the weight blob: the wgrad kernels write each filter at its blob offset ([Cout, Cin, k, k] is both
// the state_dict layout and theirs), the tail kernels each fc / head tensor at its own.
//
// New kernels (fp32, fixed summation order, no atomics: bit-identical from run to run):
//   odometry_out_bwd_kernel (one CTA): grad_T / B -> quaternion -> T backward (quat_to_T_bwd_row, shared with
//     quat_to_T_bwd_kernel) -> backward of the division by the norm of the whole [B, 4] block (all rows coupled) ->
//     d(head outputs) [B, 7]; the last Linear of each head (dW, db) and d(hidden) * act'.  With
//     DELORA_LOSS_IDENTITY_FIT its dL/dT is the identity fit's, 2 (T - I) / (16 B) on the last row, taken from the
//     forward's T, and thread 0 writes that objective (an ordered sum over the 16 entries) to losses[B-1][5].
//   odometry_linear_bwd_kernel: y = act(W x + b) backward for up to two layers that read the same x (the heads'
//     hidden layers: their contributions to dx are summed in a fixed order), dW / db and dx * act'(x) in one launch.
//   odometry_adam_kernel: torch's Adam (fused formula, no weight decay) over the whole blob, float4 per thread; the
//     step count is read from the workspace, so the bias corrections need no host value.
//   odometry_train_normalized_out_kernel (DELORA_TRAIN_NORMALIZATION_SCALING): T with its translation rescaled to the
//     caller's output, the factor to losses[b][6].
//   odometry_icp_rearm_kernel: zeroes the ICP scratch when B differs from the batch size of the previous step (the
//     scratch layout depends on B); otherwise every CTA exits at once.
//   DELORA_TRAIN_DROPOUT (masks from dropout.cuh, regenerated in the backward): the dropout variants of the trunk-input
//     conversion, of odometry_linear_kernel (the fc launch) and of odometry_linear_bwd_kernel (into dz_fc), and
//     odometry_channel_dropout_kernel (x3d in the forward, the data gradient of x3 in the backward).
namespace delora {

constexpr int kBwdThreads = 256;
constexpr int kDgradCols = 32;         // dx tile: 32 columns (one per lane) x 4 batch rows; the 8 warps split the outputs
constexpr int kDgradRows = 4;

// torch's activation backward from the stored output y: tanh' = 1 - y^2, relu' = [y > 0] (threshold_backward)
__device__ __forceinline__ float tail_act_bwd(float g, float y, int act) {
    if (act == 2) return g * (1.0f - y * y);
    if (act == 1) return y <= 0.0f ? 0.0f : g;
    return g;
}

struct TailGrad {
    const float* w;        // [N, K] row-major
    const float* x;        // [B, ldx]: the layer's input
    const float* dz;       // [B, ldz]: gradient w.r.t. the layer's output before its activation
    float* gw;             // [N, K]
    float* gb;             // [N]
    int K, N, ldx, ldz;
};

// blocks [0, p0.N + p1.N): one weight row n each, dW[n, k] = sum_b dz[b, n] x[b, k] and db[n] = sum_b dz[b, n], b in
// order.  The other blocks: dx tiles, dx[b, k] = sum over the concatenated outputs of p0 then p1 of W[n, k] dz[b, n]
// (warp w adds the w-th chunk of n in order, the chunks are added in warp order), times act_in'(x[b, k]) (0: none).
// kDrop (dx = dz_fc in a dropout training step): then times keep * 1.25f, element b * K + k of the fc mask.
template <bool kDrop>
__device__ __forceinline__ void linear_bwd_body(const TailGrad& p0, const TailGrad& p1, int B, int act_in,
                                                float* __restrict__ dx, int lddx, const DropoutCtr& drop) {
    const int nrows = p0.N + p1.N;
    if ((int)blockIdx.x < nrows) {
        int n = blockIdx.x;
        const bool second = n >= p0.N;
        const TailGrad p = second ? p1 : p0;
        if (second) n -= p0.N;
        for (int k = threadIdx.x; k < p.K; k += blockDim.x) {
            float acc = 0.0f;
            for (int b = 0; b < B; ++b) acc = fmaf(__ldg(p.dz + (size_t)b * p.ldz + n), __ldg(p.x + (size_t)b * p.ldx + k), acc);
            p.gw[(size_t)n * p.K + k] = acc;
        }
        if (threadIdx.x == 0) {
            float s = 0.0f;
            for (int b = 0; b < B; ++b) s += __ldg(p.dz + (size_t)b * p.ldz + n);
            p.gb[n] = s;
        }
        return;
    }
    __shared__ float s_part[kTailWarps][kDgradRows][kDgradCols];
    const int tile = blockIdx.x - nrows;
    const int tiles_k = (p0.K + kDgradCols - 1) / kDgradCols;
    const int k0 = (tile % tiles_k) * kDgradCols, b0 = (tile / tiles_k) * kDgradRows;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int k = k0 + lane;
    const int chunk = (nrows + kTailWarps - 1) / kTailWarps;
    const int n_lo = warp * chunk, n_hi = min(nrows, n_lo + chunk);
    float acc[kDgradRows] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (k < p0.K) {
        for (int n = n_lo; n < n_hi; ++n) {
            const bool second = n >= p0.N;
            const int nn = second ? n - p0.N : n;
            const float* __restrict__ w = second ? p1.w : p0.w;
            const float* __restrict__ dz = second ? p1.dz : p0.dz;
            const int ldz = second ? p1.ldz : p0.ldz;
            const float wv = __ldg(w + (size_t)nn * p0.K + k);
#pragma unroll
            for (int j = 0; j < kDgradRows; ++j)
                if (b0 + j < B) acc[j] = fmaf(__ldg(dz + (size_t)(b0 + j) * ldz + nn), wv, acc[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < kDgradRows; ++j) s_part[warp][j][lane] = acc[j];
    __syncthreads();
    if (threadIdx.x < kDgradRows * kDgradCols) {
        const int j = threadIdx.x / kDgradCols, c = threadIdx.x % kDgradCols;
        const int b = b0 + j, kk = k0 + c;
        if (b < B && kk < p0.K) {
            float s = 0.0f;
#pragma unroll
            for (int w = 0; w < kTailWarps; ++w) s += s_part[w][j][c];
            float g = tail_act_bwd(s, act_in ? p0.x[(size_t)b * p0.ldx + kk] : 0.0f, act_in);
            if (kDrop) {
                uint64_t seed, step;
                dropout_seed_step(drop, seed, step);
                g = dropout_keep(seed, step, kDropFc, (uint64_t)b * p0.K + kk) ? g * kDropScale : 0.0f;
            }
            dx[(size_t)b * lddx + kk] = g;
        }
    }
}

__global__ void __launch_bounds__(kBwdThreads)
odometry_linear_bwd_kernel(TailGrad p0, TailGrad p1, int B, int act_in, float* __restrict__ dx, int lddx) {
    linear_bwd_body<false>(p0, p1, B, act_in, dx, lddx, DropoutCtr{nullptr, 0});
}

__global__ void __launch_bounds__(kBwdThreads)
odometry_linear_bwd_dropout_kernel(TailGrad p0, TailGrad p1, int B, int act_in, float* __restrict__ dx, int lddx,
                                   DropoutCtr drop) {
    linear_bwd_body<true>(p0, p1, B, act_in, dx, lddx, drop);
}

struct OutBwd {
    const float* raw;                  // [B, 7] head outputs (odometry_out_kernel's raw)
    const float* grad_T;               // [B, 12] the ICP kernel's dL/dT of each pair
    const float* w_rot;                // [4, K] last layer of the rotation head (single MLP: rows 0..3)
    const float* w_trans;              // [3, K]
    const float* x_rot;                // [B, ldx] the hidden input of w_rot
    const float* x_trans;              // [B, ldx]
    float *gw_rot, *gb_rot, *gw_trans, *gb_trans;
    float* dz;                         // [B, ldz] out: gradient w.r.t. the hidden layer's pre-activation
    long long* ctr;                    // [0] Adam's step count, [1] the batch size of the ICP scratch
    const float* T16;                  // [B, 16] the forward's T (read in the identity fit only)
    float* losses;                     // [B, DELORA_LOSS_ROW]: the identity fit writes its objective to [B-1][5]
    int K, ldx, ldz, single;
    int identity;                      // DELORA_LOSS_IDENTITY_FIT: objective MSELoss(T_{B-1}, I) / B, not the ICP mean
    // delora_odometry_streams_push_adapt (NULL otherwise): the objective is the mean over the rows with valid[b] != 0,
    // *n_valid of them; each row's quaternion was divided by its own norm; the other rows get dL/dT = 0 and d = 0;
    // with *n_valid = 0 the step count does not advance
    const int32_t* valid;
    const int32_t* n_valid;
};

__global__ void __launch_bounds__(kBwdThreads)
odometry_out_bwd_kernel(OutBwd a, int B, float inv_B, int act) {
    extern __shared__ float s_d[];                          // [B, 7]: d(quaternion), d(translation); then [B] norms
    __shared__ float s_red[2];                              // and [B] d(norm) of the per-row form
    float* s_nrm = s_d + (size_t)B * 7;
    float* s_gn = s_nrm + B;
    const float* __restrict__ raw = a.raw;
    const bool rows = a.valid != nullptr;
    auto row_ok = [&](int b) { return !rows || a.valid[b] != 0; };
    if (rows) {                                             // each valid row's norm, the forward's ordered sum
        for (int b = threadIdx.x; b < B; b += blockDim.x) {
            if (!row_ok(b)) continue;
            float ss = 0.0f;
            for (int j = 0; j < 4; ++j) ss = fmaf(raw[b * 7 + j], raw[b * 7 + j], ss);
            s_nrm[b] = sqrtf(ss);
        }
    } else if (threadIdx.x == 0) {                          // the forward's ordered sum
        float ss = 0.0f;
        for (int b = 0; b < B; ++b)
            for (int j = 0; j < 4; ++j) ss = fmaf(raw[b * 7 + j], raw[b * 7 + j], ss);
        s_red[0] = sqrtf(ss);
        if (a.identity) {                                   // mean over the 16 entries of the last pair's T - I
            const float* t = a.T16 + (size_t)(B - 1) * 16;
            float se = 0.0f;
            for (int i = 0; i < 16; ++i) {
                const float e = t[i] - (i % 5 == 0 ? 1.0f : 0.0f);
                se = fmaf(e, e, se);
            }
            a.losses[(size_t)(B - 1) * DELORA_LOSS_ROW + 5] = se * (1.0f / 16.0f) * inv_B;
        }
    }
    __syncthreads();
    // d(mean over pairs): 1 / B, or 1 / n_valid over the valid rows (read only when a row is valid, so n_valid > 0)
    const float scale = rows ? 1.0f / (float)*a.n_valid : inv_B;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        if (!row_ok(b)) {
            for (int o = 0; o < 7; ++o) s_d[b * 7 + o] = 0.0f;
            continue;
        }
        const float nrm = rows ? s_nrm[b] : s_red[0];
        const float* q = raw + b * 7;
        float g[12];
        if (a.identity) {
            // d(MSELoss(T_{B-1}, I) / B) = 2 (T - I) / 16 / B on the 3x4 part of the last row (the reference overwrites
            // its loss inside the pair loop, so only the last pair counts), zero elsewhere
#pragma unroll
            for (int i = 0; i < 12; ++i)
                g[i] = b == B - 1 ? 0.125f * (a.T16[(size_t)b * 16 + i] - (i % 5 == 0 ? 1.0f : 0.0f)) * inv_B : 0.0f;
        } else {
#pragma unroll
            for (int i = 0; i < 12; ++i) g[i] = a.grad_T[(size_t)b * 12 + i] * scale;
        }
        quat_to_T_bwd_row(q[0] / nrm, q[1] / nrm, q[2] / nrm, q[3] / nrm, g, s_d + b * 7, s_d + b * 7 + 4);
    }
    __syncthreads();
    if (rows) {                                             // q / n of each row: d n = -sum(g * q) / n^2 over the row
        for (int b = threadIdx.x; b < B; b += blockDim.x) {
            if (!row_ok(b)) continue;
            float s = 0.0f;
            for (int j = 0; j < 4; ++j) s = fmaf(s_d[b * 7 + j], raw[b * 7 + j], s);
            s_gn[b] = -s / (s_nrm[b] * s_nrm[b]);
        }
    }
    if (threadIdx.x == 0) {                                 // q / n: d n = -sum(g * q) / n^2 over the whole block
        if (!rows) {
            float s = 0.0f;
            for (int b = 0; b < B; ++b)
                for (int j = 0; j < 4; ++j) s = fmaf(s_d[b * 7 + j], raw[b * 7 + j], s);
            s_red[1] = -s / (s_red[0] * s_red[0]);
        }
        if (!rows || *a.n_valid > 0) a.ctr[0] += 1;
        a.ctr[1] = B;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < B * 4; i += blockDim.x) {  // div backward + norm backward (q * dn / n)
        const int b = i >> 2, j = i & 3;
        if (!row_ok(b)) continue;
        const float nrm = rows ? s_nrm[b] : s_red[0], gn = rows ? s_gn[b] : s_red[1];
        s_d[b * 7 + j] = s_d[b * 7 + j] / nrm + raw[b * 7 + j] * (gn / nrm);
    }
    __syncthreads();
    const int K = a.K;
    for (int i = threadIdx.x; i < 7 * (K + 1); i += blockDim.x) {
        const int o = i / (K + 1), k = i - o * (K + 1);
        const float* __restrict__ x = o < 4 ? a.x_rot : a.x_trans;
        float acc = 0.0f;
        if (k < K) {
            for (int b = 0; b < B; ++b) acc = fmaf(s_d[b * 7 + o], x[(size_t)b * a.ldx + k], acc);
            (o < 4 ? a.gw_rot + (size_t)o * K : a.gw_trans + (size_t)(o - 4) * K)[k] = acc;
        } else {
            for (int b = 0; b < B; ++b) acc += s_d[b * 7 + o];
            (o < 4 ? a.gb_rot + o : a.gb_trans + (o - 4))[0] = acc;
        }
    }
    // hidden gradient: single MLP -> all 7 outputs read the same K inputs; two heads -> [rot hidden | trans hidden]
    const int ncol = a.single ? K : 2 * K;
    for (int i = threadIdx.x; i < B * ncol; i += blockDim.x) {
        const int b = i / ncol, c = i - b * ncol;
        const float* d = s_d + b * 7;
        float s = 0.0f, y;
        if (a.single) {
            for (int o = 0; o < 4; ++o) s = fmaf(a.w_rot[(size_t)o * K + c], d[o], s);
            for (int o = 0; o < 3; ++o) s = fmaf(a.w_trans[(size_t)o * K + c], d[4 + o], s);
            y = a.x_rot[(size_t)b * a.ldx + c];
        } else if (c < K) {
            for (int o = 0; o < 4; ++o) s = fmaf(a.w_rot[(size_t)o * K + c], d[o], s);
            y = a.x_rot[(size_t)b * a.ldx + c];
        } else {
            const int cc = c - K;
            for (int o = 0; o < 3; ++o) s = fmaf(a.w_trans[(size_t)o * K + cc], d[4 + o], s);
            y = a.x_trans[(size_t)b * a.ldx + cc];
        }
        a.dz[(size_t)b * a.ldz + c] = tail_act_bwd(s, y, act);
    }
}

// The gradient slices of geometries 1 .. n of delora_odometry_streams_push_adapt_geometries (blob layout each)
constexpr int kMaxGeometries = 16;
struct GradSlices {
    const float* g[kMaxGeometries - 1];
    int n;
};

// The gradient Adam reads at float4 i (or float i): g's, or with kSum g + more.g[0] + ... + more.g[n-1] in that order,
// which is written back to g
template <bool kSum>
__device__ __forceinline__ float4 adam_grad4(float* __restrict__ g, const GradSlices& more, long long i) {
    if (!kSum) return __ldg(reinterpret_cast<const float4*>(g) + i);
    float4 a = reinterpret_cast<const float4*>(g)[i];
    for (int k = 0; k < more.n; ++k) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(more.g[k]) + i);
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    reinterpret_cast<float4*>(g)[i] = a;
    return a;
}

template <bool kSum>
__device__ __forceinline__ float adam_grad1(float* __restrict__ g, const GradSlices& more, long long i) {
    if (!kSum) return g[i];
    float a = g[i];
    for (int k = 0; k < more.n; ++k) a += more.g[k][i];
    g[i] = a;
    return a;
}

// torch.optim.Adam (the fused implementation's formula; no weight decay, no amsgrad) on n floats.  run (device, or
// NULL for always): the update runs only where *run != 0 (the adapting streams' count of valid pairs).
// kSum (delora_odometry_streams_push_adapt_geometries): the gradient is g plus the slices of `more`, summed per float
// in geometry order and written back to g before the update.
template <bool kSum>
__global__ void __launch_bounds__(256)
odometry_adam_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                     long long n, const long long* __restrict__ ctr, float lr, float beta1, float beta2, float eps,
                     const int32_t* __restrict__ run, const __grid_constant__ GradSlices more) {
    if (run && *run == 0) return;                           // run non-NULL: update only when *run != 0
    const float t = (float)ctr[0];
    const float bc1 = 1.0f - powf(beta1, t);
    const float step_size = lr / bc1;
    const float bc2_sqrt = sqrtf(1.0f - powf(beta2, t));
    auto upd = [&](float& pp, float gg, float& mm, float& vv) {
        mm = beta1 * mm + (1.0f - beta1) * gg;
        vv = beta2 * vv + (1.0f - beta2) * gg * gg;
        const float denom = sqrtf(vv) / bc2_sqrt + eps;
        pp -= step_size * mm / denom;
    };
    const long long n4 = n >> 2;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 pp = reinterpret_cast<float4*>(p)[i];
        const float4 gg = adam_grad4<kSum>(g, more, i);
        float4 mm = reinterpret_cast<float4*>(m)[i];
        float4 vv = reinterpret_cast<float4*>(v)[i];
        upd(pp.x, gg.x, mm.x, vv.x); upd(pp.y, gg.y, mm.y, vv.y);
        upd(pp.z, gg.z, mm.z, vv.z); upd(pp.w, gg.w, mm.w, vv.w);
        reinterpret_cast<float4*>(p)[i] = pp;
        reinterpret_cast<float4*>(m)[i] = mm;
        reinterpret_cast<float4*>(v)[i] = vv;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const long long i = n4 * 4 + threadIdx.x;
        upd(p[i], adam_grad1<kSum>(g, more, i), m[i], v[i]);
    }
}

// The training step of a normalised model (DELORA_TRAIN_NORMALIZATION_SCALING), after the ICP finalize: T_out [B, 16] =
// the forward's T with T[:3, 3] multiplied by the pair's factor (or no copy when T_out is NULL), losses[b][6] = factor[b].
__global__ void odometry_train_normalized_out_kernel(const float* __restrict__ T16, const float* __restrict__ factor,
                                                     int B, float* __restrict__ T_out, float* __restrict__ losses) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 16) return;
    const int b = i >> 4, e = i & 15;
    const float f = factor[b];
    if (T_out) T_out[i] = (e == 3 || e == 7 || e == 11) ? __fmul_rn(T16[i], f) : T16[i];
    if (e == 0) losses[(size_t)b * DELORA_LOSS_ROW + 6] = f;
}

__global__ void odometry_icp_rearm_kernel(float4* __restrict__ s, long long n4, int B, const long long* __restrict__ ctr) {
    if (ctr[1] == B) return;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += stride)
        s[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

// ---------------------------------------------------------------- training plan: workspace layout
struct TrainPlan {
    Model m;
    size_t master, grad, adam_m, adam_v, ctr;
    TrunkWeights w;
    Frames f;                          // 2 * max_batch scans, no cached image
    size_t pts_grid, nrm_grid, icp, losses, grad_T, T16, T12;
    TrunkActs t;                       // the trunk's saving buffers
    // w_pre > 0 only: the preprocessing projection of the 2 * max_batch scans at H x w_pre (image, index map and the
    // dense grids with their normals), placed after every other buffer
    size_t pre_image, pre_index_map, pre_pts_grid, pre_nrm_grid;
    // tail activations and gradients
    size_t pooled, fc_out, hid[kMaxLinear], raw, dz_hid[kMaxLinear], dz_fc, g_pooled;
    size_t total;
};

// Two sections.  The model section (master weights, gradient, Adam's m and v, the counters, the bf16 filters) comes
// first and depends only on act, layers, resnet_outputs, single_mlp and the parity of W (the stem's filter layout).
// The geometry section (frames, grids, ICP scratch, activations, tail buffers, the w_pre buffers) starts at f.keys.
// delora_odometry_train_geometries_* rely on this split: one model section serves several geometry sections.
// geometry_at > 0: the geometry section starts at that byte offset instead (delora_odometry_streams_*_geometries: one
// model section and one geometry section per descriptor, each further one after the previous geometry's sections).
static void make_train_plan(const delora_odometry_desc* d, TrainPlan* tp, size_t geometry_at = 0) {
    memset(tp, 0, sizeof(TrainPlan));
    plan_model(d, &tp->m);
    const Model& m = tp->m;
    const int MB = d->max_batch, H = d->H, W = d->W, HW = H * W, nout = d->resnet_outputs;
    size_t off = 0;
    const size_t blob = (size_t)m.blob_floats * 4;
    tp->master = take(off, blob); tp->grad = take(off, blob); tp->adam_m = take(off, blob); tp->adam_v = take(off, blob);
    // [0] Adam's step count, [1] the ICP scratch's batch size, [2] the dropout seed (the slot has 256 bytes)
    tp->ctr = take(off, 3 * sizeof(long long));
    tp->w = plan_trunk_weights(m.t, true, off);
    if (geometry_at) off = geometry_at;
    // one key buffer serves both projections of a step, one after the other
    tp->f = plan_frames(d, 2 * MB, 0, false, d->w_pre > W ? d->w_pre : W, off);
    tp->pts_grid = take(off, (size_t)2 * MB * HW * 16);
    tp->nrm_grid = take(off, (size_t)2 * MB * HW * 16);
    tp->icp = take(off, (size_t)delora_icp_scratch_floats(MB, HW) * 4);
    tp->losses = take(off, (size_t)MB * DELORA_LOSS_ROW * 4);
    tp->grad_T = take(off, (size_t)MB * 12 * 4);
    tp->T16 = take(off, (size_t)MB * 16 * 4);
    tp->T12 = take(off, (size_t)MB * 12 * 4);
    tp->t = plan_trunk_acts(m.t, MB, true, off);
    tp->pooled = take(off, (size_t)MB * 512 * 4);
    tp->g_pooled = take(off, (size_t)MB * 512 * 4);
    tp->fc_out = take(off, (size_t)MB * nout * 4);
    tp->dz_fc = take(off, (size_t)MB * nout * 4);
    tp->raw = take(off, (size_t)MB * 7 * 4);
    if (m.n_lin == 4) {
        tp->hid[0] = take(off, (size_t)MB * 2 * kHeadHidden * 4);
        tp->dz_hid[0] = take(off, (size_t)MB * 2 * kHeadHidden * 4);
    } else {
        for (int i = 0; i < m.n_lin - 1; ++i) {
            tp->hid[i] = take(off, (size_t)MB * m.lin[i].N * 4);
            tp->dz_hid[i] = take(off, (size_t)MB * m.lin[i].N * 4);
        }
    }
    if (d->w_pre > 0) {
        const size_t HWp = (size_t)H * d->w_pre;
        tp->pre_image = take(off, (size_t)2 * MB * 4 * HWp * 4);
        tp->pre_index_map = take(off, (size_t)2 * MB * HWp * 4);
        tp->pre_pts_grid = take(off, (size_t)2 * MB * HWp * 16);
        tp->pre_nrm_grid = take(off, (size_t)2 * MB * HWp * 16);
    }
    tp->total = off;
}

// check_desc plus the field only training reads
static int check_train_desc(const delora_odometry_desc* d, const char* who) {
    if (check_desc(d, who)) return 1;
    DELORA_CHECK_ARG(d->w_pre == 0 || (d->w_pre >= 2 && (long long)d->H * d->w_pre < (1ll << 27)),
                     "%s: w_pre=%d must be 0 or >= 2 with H * w_pre < 2^27 (H=%d)", who, d->w_pre, d->H);
    return 0;
}

static int check_train_params(const delora_odometry_train_params* hp, const char* who) {
    DELORA_CHECK_ARG(hp != nullptr, "%s: null hyperparameters", who);
    DELORA_CHECK_ARG(isfinite(hp->lr) && hp->lr >= 0.0f, "%s: lr=%g must be finite and >= 0", who, (double)hp->lr);
    DELORA_CHECK_ARG(hp->beta1 >= 0.0f && hp->beta1 < 1.0f, "%s: beta1=%g must be in [0, 1)", who, (double)hp->beta1);
    DELORA_CHECK_ARG(hp->beta2 >= 0.0f && hp->beta2 < 1.0f, "%s: beta2=%g must be in [0, 1)", who, (double)hp->beta2);
    DELORA_CHECK_ARG(isfinite(hp->eps) && hp->eps > 0.0f, "%s: eps=%g must be > 0", who, (double)hp->eps);
    return check_icp_params(hp->lambda_po2pl, hp->loss_flags, hp->nb_h, hp->nb_w, hp->epsilon_range, hp->min_neighbors,
                            who);
}

static TailIO train_tail_io(const TrainPlan& tp, char* ws) {
    const Model& m = tp.m;
    TailIO io;
    memset(&io, 0, sizeof(io));
    const float* master = reinterpret_cast<const float*>(ws + tp.master);
    io.fc_w = master + m.fc.blob_w; io.fc_b = master + m.fc.blob_b;
    for (int i = 0; i < m.n_lin; ++i) { io.w[i] = master + m.lin[i].blob_w; io.b[i] = master + m.lin[i].blob_b; }
    io.fc_out = reinterpret_cast<float*>(ws + tp.fc_out);
    for (int i = 0; i < m.n_lin - 1; ++i) io.hid[i] = reinterpret_cast<float*>(ws + tp.hid[m.n_lin == 4 ? 0 : i]);
    io.raw = reinterpret_cast<float*>(ws + tp.raw);
    return io;
}

// drop.ctr non-NULL: dx is the gradient of resnet.fc's output, multiplied by the fc mask
static int linear_bwd(const TailGrad& p0, const TailGrad& p1, int B, int act_in, float* dx, int lddx, cudaStream_t st,
                      DropoutCtr drop = DropoutCtr{nullptr, 0}) {
    const int tiles = ((p0.K + kDgradCols - 1) / kDgradCols) * ((B + kDgradRows - 1) / kDgradRows);
    if (drop.ctr) {
        odometry_linear_bwd_dropout_kernel<<<p0.N + p1.N + tiles, kBwdThreads, 0, st>>>(p0, p1, B, act_in, dx, lddx, drop);
        DELORA_CHECK_LAUNCH("odometry_linear_bwd_dropout_kernel");
        return 0;
    }
    odometry_linear_bwd_kernel<<<p0.N + p1.N + tiles, kBwdThreads, 0, st>>>(p0, p1, B, act_in, dx, lddx);
    DELORA_CHECK_LAUNCH("odometry_linear_bwd_kernel");
    return 0;
}

// drop.ctr non-NULL: the gradient of resnet.fc's output (dz_fc) is multiplied by keep * 1.25 after act'
// valid / n_valid (delora_odometry_streams_push_adapt): see OutBwd
static int train_tail_backward(const TrainPlan& tp, char* ws, int act, int B, bool identity, cudaStream_t st,
                               DropoutCtr drop = DropoutCtr{nullptr, 0}, const int32_t* valid = nullptr,
                               const int32_t* n_valid = nullptr) {
    const Model& m = tp.m;
    auto f = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
    const float* master = f(tp.master);
    float* grad = f(tp.grad);
    const int nout = m.fc.N;
    OutBwd a;
    memset(&a, 0, sizeof(a));
    a.raw = f(tp.raw); a.grad_T = f(tp.grad_T); a.ctr = reinterpret_cast<long long*>(ws + tp.ctr);
    a.T16 = f(tp.T16); a.losses = f(tp.losses); a.identity = identity ? 1 : 0;
    a.valid = valid; a.n_valid = n_valid;
    if (m.n_lin == 4) {
        a.K = kHeadHidden; a.ldx = a.ldz = 2 * kHeadHidden; a.single = 0;
        a.w_rot = master + m.lin[1].blob_w; a.w_trans = master + m.lin[3].blob_w;
        a.x_rot = f(tp.hid[0]); a.x_trans = f(tp.hid[0]) + kHeadHidden;
        a.gw_rot = grad + m.lin[1].blob_w; a.gb_rot = grad + m.lin[1].blob_b;
        a.gw_trans = grad + m.lin[3].blob_w; a.gb_trans = grad + m.lin[3].blob_b;
        a.dz = f(tp.dz_hid[0]);
    } else {
        const int last = m.n_lin - 1;
        const Linear& l = m.lin[last];
        a.K = l.K; a.ldx = a.ldz = l.K; a.single = 1;
        a.w_rot = master + l.blob_w; a.w_trans = a.w_rot + 4 * (size_t)l.K;
        a.x_rot = a.x_trans = f(tp.hid[last - 1]);
        a.gw_rot = grad + l.blob_w; a.gw_trans = a.gw_rot + 4 * (size_t)l.K;
        a.gb_rot = grad + l.blob_b; a.gb_trans = a.gb_rot + 4;
        a.dz = f(tp.dz_hid[last - 1]);
    }
    odometry_out_bwd_kernel<<<1, kBwdThreads, (size_t)B * 9 * sizeof(float), st>>>(a, B, 1.0f / (float)B, act);
    DELORA_CHECK_LAUNCH("odometry_out_bwd_kernel");
    auto tg = [&](const Linear& l, const float* x, int ldx, const float* dz, int ldz) {
        TailGrad t;
        t.w = master + l.blob_w; t.x = x; t.dz = dz; t.gw = grad + l.blob_w; t.gb = grad + l.blob_b;
        t.K = l.K; t.N = l.N; t.ldx = ldx; t.ldz = ldz;
        return t;
    };
    TailGrad none;
    memset(&none, 0, sizeof(none));
    int rc;
    float* fc_out = f(tp.fc_out);
    float* dz_fc = f(tp.dz_fc);
    if (m.n_lin == 4) {
        // the heads' hidden layers read the same fc output: dx = rot1^T dz_rot + trans1^T dz_trans, then act'(fc_out)
        const int ld = 2 * kHeadHidden;
        if ((rc = linear_bwd(tg(m.lin[0], fc_out, nout, f(tp.dz_hid[0]), ld),
                             tg(m.lin[2], fc_out, nout, f(tp.dz_hid[0]) + kHeadHidden, ld), B, act, dz_fc, nout, st, drop)))
            return rc;
    } else {
        for (int i = m.n_lin - 2; i >= 0; --i) {
            const float* x = i == 0 ? fc_out : f(tp.hid[i - 1]);
            const int ldx = i == 0 ? nout : m.lin[i - 1].N;
            float* dx = i == 0 ? dz_fc : f(tp.dz_hid[i - 1]);
            if ((rc = linear_bwd(tg(m.lin[i], x, ldx, f(tp.dz_hid[i]), m.lin[i].N), none, B, act, dx, ldx, st,
                                 i == 0 ? drop : DropoutCtr{nullptr, 0}))) return rc;
        }
    }
    // resnet.fc: its input is the pooled trunk output; the last block's act' is applied by the average pool's backward
    return linear_bwd(tg(m.fc, f(tp.pooled), 512, dz_fc, nout), none, B, 0, f(tp.g_pooled), 512, st);
}

}  // namespace delora

extern "C" int64_t delora_odometry_train_workspace_bytes(const delora_odometry_desc* d) {
    if (check_train_desc(d, "delora_odometry_train_workspace_bytes")) return -1;
    TrainPlan tp;
    make_train_plan(d, &tp);
    return (int64_t)tp.total;
}

namespace delora {

// _train_init on a workspace of `total` bytes (>= d's size), armed for d
static int train_init(const delora_odometry_desc* d, size_t total, const float* weights, void* workspace,
                      cudaStream_t st, const char* who) {
    DELORA_CHECK_ARG(weights && workspace, "%s: null pointer", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    char* ws = (char*)workspace;
    int rc = init_workspace(tp.f, total, ws, st, who);
    if (rc) return rc;
    const cudaError_t e = cudaMemcpyAsync(ws + tp.master, weights, (size_t)tp.m.blob_floats * 4, cudaMemcpyDeviceToDevice,
                                          st);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return prep_blob_weights(tp.m, tp.w, ws, reinterpret_cast<const float*>(ws + tp.master), st, who);
}

// The descriptors of one shared training workspace: each valid for training, with d[0]'s model fields and W parity,
// so that all of them plan the same model section
static int check_geometries(const delora_odometry_desc* d, int n, const char* who) {
    DELORA_CHECK_ARG(d != nullptr, "%s: null descriptor array", who);
    DELORA_CHECK_ARG(n >= 1, "%s: n=%d must be >= 1", who, n);
    for (int g = 0; g < n; ++g) {
        char w[192];
        snprintf(w, sizeof w, "%s: d[%d]", who, g);
        if (check_train_desc(&d[g], w)) return 1;
        const delora_odometry_desc &a = d[0], &b = d[g];
        DELORA_CHECK_ARG(b.act == a.act, "%s: d[%d].act=%d differs from d[0].act=%d", who, g, b.act, a.act);
        for (int s = 0; s < 4; ++s)
            DELORA_CHECK_ARG(b.layers[s] == a.layers[s], "%s: d[%d].layers[%d]=%d differs from d[0].layers[%d]=%d", who,
                             g, s, b.layers[s], s, a.layers[s]);
        DELORA_CHECK_ARG(b.resnet_outputs == a.resnet_outputs, "%s: d[%d].resnet_outputs=%d differs from "
                         "d[0].resnet_outputs=%d", who, g, b.resnet_outputs, a.resnet_outputs);
        DELORA_CHECK_ARG(b.single_mlp == a.single_mlp, "%s: d[%d].single_mlp=%d differs from d[0].single_mlp=%d", who,
                         g, b.single_mlp, a.single_mlp);
        DELORA_CHECK_ARG(b.W % 2 == a.W % 2, "%s: d[%d].W=%d and d[0].W=%d differ in parity: the stem's filter layout, "
                         "and with it the model section, would differ", who, g, b.W, a.W);
    }
    return 0;
}

// The shared workspace: the model section and the largest geometry section, i.e. the largest single-geometry size
static size_t geometries_bytes(const delora_odometry_desc* d, int n) {
    size_t total = 0;
    for (int g = 0; g < n; ++g) {
        TrainPlan tp;
        make_train_plan(&d[g], &tp);
        total = tp.total > total ? tp.total : total;
    }
    return total;
}

}  // namespace delora

extern "C" int delora_odometry_train_init(const delora_odometry_desc* d, const float* weights, void* workspace,
                                          void* stream) {
    const char* who = "delora_odometry_train_init";
    if (check_train_desc(d, who)) return 1;
    TrainPlan tp;
    make_train_plan(d, &tp);
    return train_init(d, tp.total, weights, workspace, (cudaStream_t)stream, who);
}

extern "C" int64_t delora_odometry_train_geometries_workspace_bytes(const delora_odometry_desc* d, int n) {
    if (check_geometries(d, n, "delora_odometry_train_geometries_workspace_bytes")) return -1;
    return (int64_t)geometries_bytes(d, n);
}

extern "C" int delora_odometry_train_geometries_init(const delora_odometry_desc* d, int n, const float* weights,
                                                     void* workspace, void* stream) {
    const char* who = "delora_odometry_train_geometries_init";
    if (check_geometries(d, n, who)) return 1;
    return train_init(d, geometries_bytes(d, n), weights, workspace, (cudaStream_t)stream, who);
}

extern "C" int delora_odometry_train_use_geometry(const delora_odometry_desc* d, int n, int g, void* workspace,
                                                  void* stream) {
    const char* who = "delora_odometry_train_use_geometry";
    if (check_geometries(d, n, who)) return 1;
    DELORA_CHECK_ARG(g >= 0 && g < n, "%s: g=%d outside [0, n=%d)", who, g, n);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    TrainPlan tp;
    make_train_plan(&d[g], &tp);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    // the geometry section as _train_init leaves it, then the ICP scratch's batch marker ctr[1] as _train_init's zero
    int rc = init_workspace(tp.f, tp.total, ws, st, who, tp.f.keys);
    if (rc) return rc;
    const cudaError_t e = cudaMemsetAsync(ws + tp.ctr + sizeof(long long), 0, sizeof(long long), st);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

namespace delora {

__global__ void odometry_icp_batch_kernel(long long* __restrict__ ctr, int B) { ctr[1] = B; }

// One tick of delora_odometry_streams_push_adapt, as train_forward_losses sees it: the caller's arguments and the
// stream section of the workspace.
struct AdaptTick {
    const int32_t* active;             // [S] or NULL (every stream is)
    float* T;                          // [S, 16] the caller's T
    int32_t* valid;                    // [S] the caller's valid
    int32_t* has_prev;                 // [S]
    int32_t* n_valid;                  // [1] the number of valid streams this tick
    float* cache_image;                // [S, 4, H, W] w_pre = 0 only: each stream's previous image
    delora_f4* cache_pts;              // [S, H, W] (w_pre = 0) or [S, H, w_pre]: its previous stage-1 grids
    delora_f4* cache_nrm;
    float* info;                       // [S, DELORA_INFO_ROW] or NULL (_push_adapt_info): the information rows
    float* info_scratch;               // the information operator's info_scratch at B = S, with info
};

// Stages 1-3 of delora_odometry_train_step and all of delora_odometry_train_eval: the projection + normals of the 2B
// scans, the forward keeping its activations and the ICP losses with dL/dT, into the workspace (losses, grad_T, T16,
// pooled).  dropout: the forward draws this step's masks.  Normalised models: T_out [B, 16] or NULL gets T in metres.
// at (delora_odometry_streams_push_adapt, B = S): stage 1 projects only the B scans of this tick (scan_2 of each pair,
// inactive streams' counts masked to 0) and takes its first half, scan_1's, from the cache; the output kernel divides
// each quaternion by its own row's norm, writes raw for the valid rows only, valid, has_prev and n_valid; then the
// bookkeeping kernel writes at->T, T12, the masked cache write and empties the sources of the rows without a pair.
// With at->info the ICP is the information operator (losses and dL/dT are the same bits), in metres for normalised
// models: their grids were divided by the pair factors, kept in pre_image.
static int train_forward_losses(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const TrainPlan& tp,
                                char* ws, const float* points, const int32_t* n_points, int B, bool dropout, float* T_out,
                                cudaStream_t st, const char* who, const AdaptTick* at = nullptr) {
    const Model& m = tp.m;
    auto f = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
    const int H = d->H, W = d->W, HW = H * W;
    const bool normalized = (hp->loss_flags & DELORA_TRAIN_NORMALIZATION_SCALING) != 0u;
    long long* ctr = reinterpret_cast<long long*>(ws + tp.ctr);
    // the forward reads the step count before odometry_out_bwd_kernel advances it
    const DropoutCtr drop_fwd{dropout ? ctr : nullptr, 0};
    int rc;

    // 1. projection + normals of the 2B scans (scan_1 x B, then scan_2 x B).  w_pre > 0: the reference's two stages,
    // projection + normals at H x w_pre (its offline preprocessing), then those grids projected at H x W (Deployer.step)
    // at: only the B scan_2's are projected (from scan index `first` on), and scan_1's stage-1 output is the cache's
    const int n_proj = at ? B : 2 * B;
    const size_t first = at ? (size_t)B : 0;
    if ((rc = clamp_counts(tp.f, ws, n_points, at ? at->active : nullptr, n_proj, d->n_stride, st))) return rc;
    int32_t* counts = reinterpret_cast<int32_t*>(ws + tp.f.counts);
    delora_f4* pts_grid = reinterpret_cast<delora_f4*>(ws + tp.pts_grid);
    delora_f4* nrm_grid = reinterpret_cast<delora_f4*>(ws + tp.nrm_grid);
    float* images = f(tp.f.images);
    uint64_t* keys = reinterpret_cast<uint64_t*>(ws + tp.f.keys);
    const size_t HWc = (size_t)H * (d->w_pre > 0 ? d->w_pre : W);         // cells of a stage-1 grid
    auto from_cache = [&](void* dst, const void* src, size_t bytes) {
        const cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
        return 0;
    };
    if (d->w_pre > 0) {
        delora_f4* pre_pts = reinterpret_cast<delora_f4*>(ws + tp.pre_pts_grid);
        delora_f4* pre_nrm = reinterpret_cast<delora_f4*>(ws + tp.pre_nrm_grid);
        if ((rc = delora_project_normals_fwd(points, counts, n_proj, 3, d->n_stride, H, d->w_pre, d->hfov0, d->hfov1,
                                             d->vfov0, d->vfov1, 0, keys, f(tp.pre_image) + first * 4 * HWc,
                                             reinterpret_cast<int32_t*>(ws + tp.pre_index_map) + first * HWc, hp->nb_h,
                                             hp->nb_w, hp->epsilon_range, hp->min_neighbors, pre_pts + first * HWc,
                                             pre_nrm + first * HWc, nullptr, st)))
            return rc;
        if (at && ((rc = from_cache(pre_pts, at->cache_pts, (size_t)B * HWc * 16)) ||
                   (rc = from_cache(pre_nrm, at->cache_nrm, (size_t)B * HWc * 16)))) return rc;
        // normalised: the factor of each pair from its stored points (the valid H x w_pre cells), kept in the H x w_pre
        // image, which nothing reads after delora_project_normals_fwd; the stored points are divided by it before the
        // H x W projection, the normals are not
        float* factor = normalized ? f(tp.pre_image) : nullptr;
        if (normalized && (rc = launch_grid_normalization_factors(pre_pts, B, H * d->w_pre, factor, st))) return rc;
        const GridParams g = make_grid(H, W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0);
        if ((rc = project_grids_fwd(pre_pts, pre_nrm, 2 * B, d->w_pre, g, keys, images,
                                    reinterpret_cast<int32_t*>(ws + tp.f.index_map), pts_grid, nrm_grid, factor, B, st)))
            return rc;
    } else {
        if ((rc = delora_project_normals_fwd(points, counts, n_proj, 3, d->n_stride, H, W, d->hfov0, d->hfov1, d->vfov0,
                                             d->vfov1, 0, keys, images + first * 4 * HW,
                                             reinterpret_cast<int32_t*>(ws + tp.f.index_map) + first * HW, hp->nb_h,
                                             hp->nb_w, hp->epsilon_range, hp->min_neighbors, pts_grid + first * HW,
                                             nrm_grid + first * HW, nullptr, st)))
            return rc;
        if (at && ((rc = from_cache(images, at->cache_image, (size_t)B * 4 * HW * 4)) ||
                   (rc = from_cache(pts_grid, at->cache_pts, (size_t)B * HW * 16)) ||
                   (rc = from_cache(nrm_grid, at->cache_nrm, (size_t)B * HW * 16)))) return rc;
    }
    // 2. forward, keeping the activations
    if ((rc = trunk_input(m.t, tp.t, ws, images, images + (size_t)B * 4 * HW, B, st, drop_fwd))) return rc;
    if (at) {               // dropout is off: the served T is dropout-free
        if ((rc = streams_forward<false>(m, train_tail_io(tp, ws), tp.t, tp.w, ws, d->act, f(tp.pooled), B, at->active,
                                         at->has_prev, f(tp.T16), at->valid, nullptr, nullptr, nullptr, at->n_valid,
                                         st))) return rc;
        // T (normalised: the factor of the H x w_pre grids, kept in pre_image as below), T12, the cache, the sources
        size_t cells = HWc > (size_t)HW ? HWc : (size_t)HW;
        if (cells < 16) cells = 16;
        cells *= (size_t)B;
        float4* cur_pts = reinterpret_cast<float4*>(pts_grid + (size_t)B * HW);
        float4* cur_nrm = reinterpret_cast<float4*>(nrm_grid + (size_t)B * HW);
        const bool pre = d->w_pre > 0;
        odometry_streams_pre_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, st>>>(
            f(tp.T16), normalized ? f(tp.pre_image) : nullptr, at->active, at->valid, B, HW, (int)HWc, at->T, f(tp.T12),
            nullptr, cur_pts, cur_nrm,
            pre ? reinterpret_cast<const float4*>(ws + tp.pre_pts_grid) + (size_t)B * HWc : cur_pts,
            pre ? reinterpret_cast<const float4*>(ws + tp.pre_nrm_grid) + (size_t)B * HWc : cur_nrm,
            reinterpret_cast<float4*>(at->cache_pts), reinterpret_cast<float4*>(at->cache_nrm),
            pre ? nullptr : reinterpret_cast<const float4*>(images + (size_t)B * 4 * HW),
            reinterpret_cast<float4*>(at->cache_image));
        DELORA_CHECK_LAUNCH("odometry_streams_pre_kernel");
    } else {
        if ((rc = trunk_forward(m.t, tp.t, ws, tp.w, ws, d->act, B, f(tp.pooled), nullptr, st, drop_fwd))) return rc;
        if ((rc = run_tail(m, train_tail_io(tp, ws), d->act, f(tp.pooled), B, f(tp.T16), st, nullptr, drop_fwd)))
            return rc;
        const cudaError_t e = cudaMemcpy2DAsync(f(tp.T12), 12 * sizeof(float), f(tp.T16), 16 * sizeof(float),
                                                12 * sizeof(float), B, cudaMemcpyDeviceToDevice, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    }
    // 3. ICP losses and dL/dT: source = scan_2 moved by T, target = scan_1.  The identity fit still runs them: the
    // reference logs the ICP losses in that phase too
    const long long icp_n4 = (delora_icp_scratch_floats(B, HW) + 3) / 4;
    odometry_icp_rearm_kernel<<<2 * num_sms(), 256, 0, st>>>(reinterpret_cast<float4*>(ws + tp.icp), icp_n4, B, ctr);
    DELORA_CHECK_LAUNCH("odometry_icp_rearm_kernel");
    const uint32_t icp_flags =
        hp->loss_flags & ~(DELORA_LOSS_IDENTITY_FIT | DELORA_TRAIN_NORMALIZATION_SCALING | DELORA_TRAIN_DROPOUT);
    float* info = at ? at->info : nullptr;
    const float* factor = info && normalized ? f(tp.pre_image) : nullptr;
    if ((rc = icp_dense_launch(pts_grid + (size_t)B * HW, nrm_grid + (size_t)B * HW, f(tp.T12), pts_grid, nrm_grid, B,
                               H, W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, hp->lambda_po2pl, icp_flags,
                               f(tp.losses), f(tp.grad_T), f(tp.icp), info, at ? at->info_scratch : nullptr, factor,
                               st, icp_entry(info, factor)))) return rc;
    if (normalized) {               // T in metres for the caller, the factor in losses[b][6]
        odometry_train_normalized_out_kernel<<<(B * 16 + 255) / 256, 256, 0, st>>>(f(tp.T16), f(tp.pre_image), B, T_out,
                                                                                      f(tp.losses));
        DELORA_CHECK_LAUNCH("odometry_train_normalized_out_kernel");
    }
    return 0;
}

// losses, T (not for normalised models: train_forward_losses wrote it) and pooled of B pairs to the caller's buffers
static int train_outputs(const TrainPlan& tp, const char* ws, int B, bool normalized, float* losses, float* T,
                         float* pooled, cudaStream_t st, const char* who) {
    cudaError_t e = cudaSuccess;
    auto out = [&](float* dst, size_t src, size_t n) {
        if (dst && e == cudaSuccess) e = cudaMemcpyAsync(dst, ws + src, n * sizeof(float), cudaMemcpyDeviceToDevice, st);
    };
    out(losses, tp.losses, (size_t)B * DELORA_LOSS_ROW);
    if (!normalized) out(T, tp.T16, (size_t)B * 16);
    out(pooled, tp.pooled, (size_t)B * 512);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

// what _train_step and _train_eval refuse alike
static int check_train_call(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const float* points,
                            const int32_t* n_points, int B, const void* workspace, const char* who) {
    if (check_train_desc(d, who)) return 1;
    if (check_train_params(hp, who)) return 1;
    DELORA_CHECK_ARG(points && n_points && workspace, "%s: null pointer", who);
    DELORA_CHECK_ARG(B >= 1 && B <= d->max_batch, "%s: B=%d outside [1, max_batch=%d]", who, B, d->max_batch);
    DELORA_CHECK_ARG((hp->loss_flags & DELORA_TRAIN_NORMALIZATION_SCALING) == 0u || d->w_pre > 0,
                     "%s: DELORA_TRAIN_NORMALIZATION_SCALING needs w_pre > 0 (the reference's recipe: normals from the "
                     "unscaled points at H x w_pre), got w_pre=%d", who, d->w_pre);
    return 0;
}

}  // namespace delora

namespace delora {

// The group step's all-reduce schedule (delora_odometry_train_group_buckets): bucket k of kGroupBuckets in launch
// order, i.e. the backward's production order: heads + fc, layer4, layer3, layer2, stem + layer1.  Each boundary is a
// stage boundary rounded up to 4 floats, so a bucket may take up to 3 floats of the section after it in the blob (which
// the backward produced before it) and never one of the section before it (not produced yet).  The last bucket ends
// at most 3 floats past blob_floats, in the gradient section's 256-byte padding, which nothing reads.
constexpr int kGroupBuckets = DELORA_TRAIN_GROUP_BUCKETS;
static void plan_buckets(const Model& m, long long off[kGroupBuckets], long long cnt[kGroupBuckets]) {
    auto up4 = [](long long x) { return (x + 3) & ~3ll; };
    long long edge[kGroupBuckets + 1];            // stage starts in blob order: stem, layer2, layer3, layer4, fc, end
    edge[0] = 0;
    for (int s = 1; s < 4; ++s) {
        int i = 0;
        while (m.t.block[i].stage < s) ++i;
        edge[s] = up4(m.t.conv[m.t.block[i].c1].blob);
    }
    edge[4] = up4(m.fc.blob_w);
    edge[5] = up4(m.blob_floats);
    for (int k = 0; k < kGroupBuckets; ++k) {
        off[k] = edge[4 - k];
        cnt[k] = edge[5 - k] - edge[4 - k];
    }
}

static int check_group(const delora_odometry_train_group* g, const void* workspace, const char* who) {
    DELORA_CHECK_ARG(g != nullptr, "%s: null group", who);
    DELORA_CHECK_ARG(g->world >= 1 && g->world <= kArMaxWorld, "%s: world=%d must be in [1, %d]", who, g->world,
                     kArMaxWorld);
    DELORA_CHECK_ARG(g->rank >= 0 && g->rank < g->world, "%s: rank=%d outside [0, world=%d)", who, g->rank, g->world);
    for (int q = 0; q < g->world; ++q) {
        DELORA_CHECK_ARG(g->peer_ws[q] != 0 && (g->peer_ws[q] & 15) == 0, "%s: peer_ws[%d] is null or not 16-byte aligned",
                         who, q);
        DELORA_CHECK_ARG(g->peer_flags[q] != 0 && (g->peer_flags[q] & 3) == 0,
                         "%s: peer_flags[%d] is null or not 4-byte aligned", who, q);
    }
    DELORA_CHECK_ARG(g->peer_ws[g->rank] == (uint64_t)(uintptr_t)workspace, "%s: peer_ws[rank=%d] is not the workspace",
                     who, g->rank);
    DELORA_CHECK_ARG((g->multicast & 15) == 0, "%s: multicast is not 16-byte aligned", who);
    DELORA_CHECK_ARG(g->status != nullptr, "%s: null status", who);
    DELORA_CHECK_ARG(g->n_ctas >= 1 && g->n_ctas <= kArMaxCtas, "%s: n_ctas=%d outside [1, %d]", who, g->n_ctas,
                     kArMaxCtas);
    DELORA_CHECK_ARG(g->n_threads >= 32 && g->n_threads <= kArMaxThreads && g->n_threads % 32 == 0,
                     "%s: n_threads=%d must be 32, 64, 96 or 128", who, g->n_threads);
    if (g->world > 1) {
        for (int k = 0; k < kGroupBuckets; ++k)
            DELORA_CHECK_ARG(g->fork_events[k] != nullptr, "%s: null fork_events[%d]", who, k);
        DELORA_CHECK_ARG(g->join_event != nullptr, "%s: null join_event", who);
    }
    return 0;
}

// Stage 5 of the step: Adam on the master blob (only where *run != 0, run non-NULL), then the bf16 filters from the
// master weights.  more (n > 0): Adam reads tp.grad plus those gradient slices and leaves their sum in tp.grad.
static int adam_update(const TrainPlan& tp, char* ws, const delora_odometry_train_params* hp, const int32_t* run,
                       cudaStream_t st, const GradSlices* more = nullptr) {
    auto f = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
    const long long n = tp.m.blob_floats;
    const long long blocks = (n / 4 + 255) / 256;
    const int grid = (int)(blocks < 8ll * num_sms() ? (blocks > 0 ? blocks : 1) : 8ll * num_sms());
    const long long* ctr = reinterpret_cast<const long long*>(ws + tp.ctr);
    if (more && more->n > 0)
        odometry_adam_kernel<true><<<grid, 256, 0, st>>>(f(tp.master), f(tp.grad), f(tp.adam_m), f(tp.adam_v), n, ctr,
                                                         hp->lr, hp->beta1, hp->beta2, hp->eps, run, *more);
    else
        odometry_adam_kernel<false><<<grid, 256, 0, st>>>(f(tp.master), f(tp.grad), f(tp.adam_m), f(tp.adam_v), n, ctr,
                                                          hp->lr, hp->beta1, hp->beta2, hp->eps, run, GradSlices{});
    DELORA_CHECK_LAUNCH("odometry_adam_kernel");
    return delora_conv_weight_prep_multi(ws + tp.w.table, tp.m.t.n_conv, st);
}

// How the group form of a step all-reduces its gradient: bucket k times scale, seq = *seq_step * seq_stride +
// seq_first + k
struct GroupReduce {
    const delora_odometry_train_group* g;
    float scale;
    const long long* seq_step;
    unsigned seq_stride, seq_first;
};

// Stage 4 of the step at B pairs: the tail backward (see train_tail_backward for identity, drop, valid and n_valid),
// then the trunk backward of stage 3 down to 0.  With gr, bucket k of plan_buckets' schedule is all-reduced in place in
// every rank's gradient section as soon as the backward has produced it on `st` (bucket 0 after the tail, bucket 4 - s
// after stage s): g->side_stream waits for it through fork_events[k] and runs the all-reduce, and `st` then waits for
// every bucket through join_event.
static int step_backward(const TrainPlan& tp, char* ws, int act, int B, bool identity, DropoutCtr drop,
                         const int32_t* valid, const int32_t* n_valid, const GroupReduce* gr, cudaStream_t st,
                         const char* who) {
    const delora_odometry_train_group* g = gr ? gr->g : nullptr;
    cudaStream_t side = g ? (cudaStream_t)g->side_stream : nullptr;
    long long b_off[kGroupBuckets], b_cnt[kGroupBuckets];
    uint64_t peer_grad[kArMaxWorld];
    if (g) {
        plan_buckets(tp.m, b_off, b_cnt);
        for (int q = 0; q < g->world; ++q) peer_grad[q] = g->peer_ws[q] + tp.grad;
    }
    auto all_reduce = [&](int k) -> int {
        if (!g) return 0;
        cudaError_t e = cudaEventRecord((cudaEvent_t)g->fork_events[k], st);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(side, (cudaEvent_t)g->fork_events[k], 0);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: fork_events[%d]: %s", who, k, cudaGetErrorString(e));
        return grad_allreduce_launch(peer_grad, g->peer_flags, g->multicast ? g->multicast + tp.grad : 0ull, g->rank,
                                     g->world, b_off[k], b_cnt[k], gr->scale, gr->seq_first + (unsigned)k, gr->seq_step,
                                     gr->seq_stride, g->n_ctas, g->n_threads, g->status, side);
    };
    int rc;
    if ((rc = train_tail_backward(tp, ws, act, B, identity, st, drop, valid, n_valid))) return rc;
    if ((rc = all_reduce(0))) return rc;
    float* conv_dw[kMaxConv];
    for (int i = 0; i < tp.m.t.n_conv; ++i) conv_dw[i] = reinterpret_cast<float*>(ws + tp.grad) + tp.m.t.conv[i].blob;
    const float* g_pooled = reinterpret_cast<const float*>(ws + tp.g_pooled);
    for (int s = 3; s >= 0; --s) {
        if ((rc = trunk_backward(tp.m.t, tp.t, ws, tp.w, ws, act, B, g_pooled, conv_dw, s, st, drop))) return rc;
        if ((rc = all_reduce(4 - s))) return rc;
    }
    if (!g) return 0;
    cudaError_t e = cudaEventRecord((cudaEvent_t)g->join_event, side);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(st, (cudaEvent_t)g->join_event, 0);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: join_event: %s", who, cudaGetErrorString(e));
    return 0;
}

// delora_odometry_train_step, and with g (world > 1) its group form: bucket k is all-reduced on g->side_stream once
// the backward has produced it, and `stream` joins g->side_stream before the gradient is read.
static int train_step(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                      const delora_odometry_train_group* g, const float* points, const int32_t* n_points, int B,
                      void* workspace, float* losses, float* T, float* pooled, float* grads, void* stream,
                      const char* who) {
    const bool normalized = (hp->loss_flags & DELORA_TRAIN_NORMALIZATION_SCALING) != 0u;
    const bool dropout = (hp->loss_flags & DELORA_TRAIN_DROPOUT) != 0u;
    const bool identity = (hp->loss_flags & DELORA_LOSS_IDENTITY_FIT) != 0u;
    TrainPlan tp;
    make_train_plan(d, &tp);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    long long* ctr = reinterpret_cast<long long*>(ws + tp.ctr);
    // the masks of this step, regenerated after odometry_out_bwd_kernel has advanced the step count
    const DropoutCtr drop_bwd{dropout ? ctr : nullptr, 1};
    // the buckets are averaged; seq = the step count (advanced by odometry_out_bwd_kernel before bucket 0) *
    // kGroupBuckets + k
    const GroupReduce gr{g, g ? 1.0f / (float)g->world : 1.0f, ctr, (unsigned)kGroupBuckets, 0u};
    int rc;
    // 1-3. projection + normals, forward, ICP losses and dL/dT
    if ((rc = train_forward_losses(d, hp, tp, ws, points, n_points, B, dropout, T, st, who))) return rc;
    // 4. backward: tail (dL/dT of the ICP mean or of the identity fit), average pool, trunk
    if ((rc = step_backward(tp, ws, d->act, B, identity, drop_bwd, nullptr, nullptr, g ? &gr : nullptr, st, who)))
        return rc;
    // outputs (T: the weights before the update)
    if ((rc = train_outputs(tp, ws, B, normalized, losses, T, pooled, st, who))) return rc;
    if (grads) {
        const cudaError_t e = cudaMemcpyAsync(grads, ws + tp.grad, (size_t)tp.m.blob_floats * sizeof(float),
                                              cudaMemcpyDeviceToDevice, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    }
    // 5. Adam on the master blob, then the bf16 filters from the updated weights
    return adam_update(tp, ws, hp, nullptr, st);
}

}  // namespace delora

extern "C" int delora_odometry_train_step(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                          const float* points, const int32_t* n_points, int B, void* workspace,
                                          float* losses, float* T, float* pooled, float* grads, void* stream) {
    const char* who = "delora_odometry_train_step";
    if (check_train_call(d, hp, points, n_points, B, workspace, who)) return 1;
    return train_step(d, hp, nullptr, points, n_points, B, workspace, losses, T, pooled, grads, stream, who);
}

extern "C" int delora_odometry_train_step_group(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                                const delora_odometry_train_group* g, const float* points,
                                                const int32_t* n_points, int B, void* workspace, float* losses,
                                                float* T, float* pooled, float* grads, void* stream) {
    const char* who = "delora_odometry_train_step_group";
    if (check_train_call(d, hp, points, n_points, B, workspace, who)) return 1;
    if (check_group(g, workspace, who)) return 1;
    return train_step(d, hp, g->world > 1 ? g : nullptr, points, n_points, B, workspace, losses, T, pooled, grads,
                      stream, who);
}

extern "C" int64_t delora_odometry_train_grad_offset(const delora_odometry_desc* d) {
    if (check_train_desc(d, "delora_odometry_train_grad_offset")) return -1;
    TrainPlan tp;
    make_train_plan(d, &tp);
    return (int64_t)tp.grad;
}

extern "C" int delora_odometry_train_group_buckets(const delora_odometry_desc* d, int64_t* offsets, int64_t* counts) {
    const char* who = "delora_odometry_train_group_buckets";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(offsets && counts, "%s: null pointer", who);
    Model m;
    plan_model(d, &m);
    long long off[kGroupBuckets], cnt[kGroupBuckets];
    plan_buckets(m, off, cnt);
    for (int k = 0; k < kGroupBuckets; ++k) { offsets[k] = off[k]; counts[k] = cnt[k]; }
    return 0;
}

extern "C" int delora_odometry_train_eval(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                          const float* points, const int32_t* n_points, int B, void* workspace,
                                          float* losses, float* T, float* pooled, void* stream) {
    const char* who = "delora_odometry_train_eval";
    if (check_train_call(d, hp, points, n_points, B, workspace, who)) return 1;
    TrainPlan tp;
    make_train_plan(d, &tp);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    int rc;
    // dropout is the identity, as at inference; the identity fit's objective belongs to the step's backward
    if ((rc = train_forward_losses(d, hp, tp, ws, points, n_points, B, false, T, st, who))) return rc;
    // the ICP scratch now has the layout of B pairs: the next step or eval re-arms it if its batch size differs
    odometry_icp_batch_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long*>(ws + tp.ctr), B);
    DELORA_CHECK_LAUNCH("odometry_icp_batch_kernel");
    return train_outputs(tp, ws, B, (hp->loss_flags & DELORA_TRAIN_NORMALIZATION_SCALING) != 0u, losses, T, pooled, st,
                         who);
}

extern "C" int delora_odometry_train_weights(const delora_odometry_desc* d, const void* workspace, float* weights,
                                             void* stream) {
    const char* who = "delora_odometry_train_weights";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(workspace && weights, "%s: null pointer", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    const cudaError_t e = cudaMemcpyAsync(weights, (const char*)workspace + tp.master, (size_t)tp.m.blob_floats * 4,
                                          cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

extern "C" int delora_odometry_train_get_state(const delora_odometry_desc* d, const void* workspace, float* weights,
                                               float* exp_avg, float* exp_avg_sq, int64_t* step, void* stream) {
    const char* who = "delora_odometry_train_get_state";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    const char* ws = (const char*)workspace;
    const size_t blob = (size_t)tp.m.blob_floats * 4;
    cudaError_t e = cudaSuccess;
    auto out = [&](void* dst, size_t src, size_t bytes) {
        if (dst && e == cudaSuccess) e = cudaMemcpyAsync(dst, ws + src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
    };
    out(weights, tp.master, blob);
    out(exp_avg, tp.adam_m, blob);
    out(exp_avg_sq, tp.adam_v, blob);
    out(step, tp.ctr, sizeof(long long));
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

extern "C" int delora_odometry_train_set_state(const delora_odometry_desc* d, const float* weights, const float* exp_avg,
                                               const float* exp_avg_sq, const int64_t* step, void* workspace,
                                               void* stream) {
    const char* who = "delora_odometry_train_set_state";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(weights, "%s: null weights", who);
    DELORA_CHECK_ARG(exp_avg, "%s: null exp_avg", who);
    DELORA_CHECK_ARG(exp_avg_sq, "%s: null exp_avg_sq", who);
    DELORA_CHECK_ARG(step, "%s: null step", who);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    char* ws = (char*)workspace;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t blob = (size_t)tp.m.blob_floats * 4;
    cudaError_t e = cudaSuccess;
    auto in = [&](size_t dst, const void* src, size_t bytes) {
        if (e == cudaSuccess) e = cudaMemcpyAsync(ws + dst, src, bytes, cudaMemcpyDeviceToDevice, st);
    };
    in(tp.master, weights, blob);
    in(tp.adam_m, exp_avg, blob);
    in(tp.adam_v, exp_avg_sq, blob);
    in(tp.ctr, step, sizeof(long long));            // ctr[0] only: ctr[1], the ICP scratch's batch size, stays
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    // the bf16 filters from the new master weights, through the table _train_init wrote
    return delora_conv_weight_prep_multi(ws + tp.w.table, tp.m.t.n_conv, st);
}

// ================================================================================================ adapting streams
// delora_odometry_streams_push_adapt: S = max_batch streams served from a training workspace, which takes the training
// step on the pairs it has just served.  The workspace is the training layout of d (max_batch = S) followed by the
// stream section; no training offset moves, so every delora_odometry_train_* entry point works on it unchanged.
namespace delora {

struct AdaptPlan {
    size_t cache_image;                // w_pre = 0 only: [S, 4, H, W]
    size_t cache_pts, cache_nrm;       // [S, H, W] (w_pre = 0) or [S, H, w_pre]
    size_t has_prev, n_valid;          // [S], [1]
    size_t cache_cells;                // cells of one stream's cached grid
    size_t total;
    // The group section of delora_odometry_streams_push_adapt_group, one 256-byte block after the adapting-streams
    // layout: the tick counter (int64: group ticks with update = 1 so far), the fleet-wide count of valid pairs of the
    // last such tick (int32) and the count exchange's slots (int32 [2][kArMaxWorld], see count_allreduce_kernel).
    size_t tick, n_fleet, slots;
    size_t group_total;
    // The information section of delora_odometry_streams_push_adapt_info / _group_info, after the group section: the
    // information rows of the S pairs and the operator's info_scratch at B = S
    size_t info, info_scratch;
    size_t info_total;
};

// geometry_at: see make_train_plan; the stream section follows the geometry section wherever that starts
static void make_adapt_plan(const delora_odometry_desc* d, TrainPlan* tp, AdaptPlan* ap, size_t geometry_at = 0) {
    make_train_plan(d, tp, geometry_at);
    memset(ap, 0, sizeof(AdaptPlan));
    const size_t S = (size_t)d->max_batch, HW = (size_t)d->H * d->W;
    size_t off = tp->total;
    ap->cache_cells = d->w_pre > 0 ? (size_t)d->H * d->w_pre : HW;
    if (d->w_pre == 0) ap->cache_image = take(off, S * 4 * HW * 4);
    ap->cache_pts = take(off, S * ap->cache_cells * 16);
    ap->cache_nrm = take(off, S * ap->cache_cells * 16);
    ap->has_prev = take(off, S * 4);
    ap->n_valid = take(off, 4);
    ap->total = off;
    const size_t base = take(off, 8 + 8 + 2 * kArMaxWorld * 4);
    ap->tick = base;
    ap->n_fleet = base + 8;
    ap->slots = base + 16;
    ap->group_total = off;
    ap->info = take(off, S * DELORA_INFO_ROW * 4);
    ap->info_scratch = take(off, (size_t)delora_icp_information_scratch_floats(d->max_batch, d->H, d->W) * 4);
    ap->info_total = off;
}

// The adapting-streams workspace forms: _adapt (total), _adapt_group (group_total), _adapt_info (info_total)
enum class Adapt { plain, group, info };

static size_t adapt_bytes(const AdaptPlan& ap, Adapt form) {
    return form == Adapt::info ? ap.info_total : form == Adapt::group ? ap.group_total : ap.total;
}

// The adapting-streams workspace's size in one of its forms
static int64_t adapt_workspace_bytes(const delora_odometry_desc* d, Adapt form, const char* who) {
    if (check_train_desc(d, who)) return -1;
    TrainPlan tp;
    AdaptPlan ap;
    make_adapt_plan(d, &tp, &ap);
    return (int64_t)adapt_bytes(ap, form);
}

// _streams_adapt_init, _streams_adapt_group_init and _streams_adapt_info_init; the group and information sections are
// zeroed too, and the forms with a group section preload the collective kernels
static int adapt_init(const delora_odometry_desc* d, Adapt form, const float* weights, void* workspace, cudaStream_t st,
                      const char* who) {
    if (check_train_desc(d, who)) return 1;
    TrainPlan tp;
    AdaptPlan ap;
    make_adapt_plan(d, &tp, &ap);
    // _train_init over the whole workspace zeroes the stream section too; the cached grids then start empty
    int rc = train_init(d, adapt_bytes(ap, form), weights, workspace, st, who);
    if (rc) return rc;
    if ((rc = clear_grids((char*)workspace, ap.cache_pts, ap.cache_nrm, (size_t)d->max_batch * ap.cache_cells, st)))
        return rc;
    return form != Adapt::plain ? collective_kernels_preload(who) : 0;
}

// The hyperparameters and update value every adapting tick refuses alike
static int check_adapt_params(const delora_odometry_train_params* hp, int update, const char* who) {
    if (check_train_params(hp, who)) return 1;
    DELORA_CHECK_ARG(update == 0 || update == 1, "%s: update=%d must be 0 or 1", who, update);
    DELORA_CHECK_ARG((hp->loss_flags & DELORA_LOSS_IDENTITY_FIT) == 0u,
                     "%s: loss_flags=0x%x has DELORA_LOSS_IDENTITY_FIT, a pre-training phase, not adaptation", who,
                     hp->loss_flags);
    DELORA_CHECK_ARG((hp->loss_flags & DELORA_TRAIN_DROPOUT) == 0u,
                     "%s: loss_flags=0x%x has DELORA_TRAIN_DROPOUT: the served T is dropout-free, and one forward "
                     "cannot be both", who, hp->loss_flags);
    return 0;
}

// What _push_adapt and _push_adapt_group refuse alike
static int check_push_adapt(const delora_odometry_desc* d, const delora_odometry_train_params* hp, int update,
                            const float* points, const int32_t* n_points, void* workspace, float* T, int32_t* valid,
                            float* losses, const char* who) {
    if (check_train_desc(d, who)) return 1;
    if (check_adapt_params(hp, update, who)) return 1;
    if (check_tick(points, n_points, workspace, T, valid, losses, "losses", who)) return 1;
    return check_train_call(d, hp, points, n_points, d->max_batch, workspace, who);
}

// Stages 1-3 of one adapting tick of the S = d->max_batch streams of (tp, ap): T, valid, the loss rows and the cache
// write, with info (an information workspace) the information rows at the served T; update = 0 then records the ICP
// scratch's batch marker
static int serve_adapt(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const TrainPlan& tp,
                       const AdaptPlan& ap, int update, const float* points, const int32_t* n_points,
                       const int32_t* active, char* ws, float* T, int32_t* valid, float* losses, float* info,
                       cudaStream_t st, const char* who) {
    const int S = d->max_batch;
    auto f = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
    AdaptTick at;
    at.active = active;
    at.T = T;
    at.valid = valid;
    at.has_prev = reinterpret_cast<int32_t*>(ws + ap.has_prev);
    at.n_valid = reinterpret_cast<int32_t*>(ws + ap.n_valid);
    at.cache_image = d->w_pre == 0 ? f(ap.cache_image) : nullptr;
    at.cache_pts = reinterpret_cast<delora_f4*>(ws + ap.cache_pts);
    at.cache_nrm = reinterpret_cast<delora_f4*>(ws + ap.cache_nrm);
    at.info = info ? f(ap.info) : nullptr;
    at.info_scratch = info ? f(ap.info_scratch) : nullptr;
    int rc;
    // 1-3 at B = S, the first frame of every pair from the cache; T, valid, the cache and the emptied sources
    if ((rc = train_forward_losses(d, hp, tp, ws, points, n_points, S, false, nullptr, st, who, &at))) return rc;
    if ((rc = streams_rows_out<DELORA_LOSS_ROW>(valid, S, f(tp.losses), losses, st))) return rc;
    if (info && (rc = streams_rows_out<DELORA_INFO_ROW>(valid, S, f(ap.info), info, st))) return rc;
    if (!update) {          // the ICP scratch now has the layout of S pairs, as after _train_eval
        odometry_icp_batch_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long*>(ws + tp.ctr), S);
        DELORA_CHECK_LAUNCH("odometry_icp_batch_kernel");
    }
    return 0;
}

// One tick of _push_adapt, and with g (world > 1, update = 1) of its group form: the count of valid pairs is
// exchanged (collective k = 0) before the backward, which then divides by the fleet-wide count; the gradient buckets
// are summed over the ranks on g->side_stream (collectives k = 1 .. kGroupBuckets); Adam runs where that count is > 0.
// The group's sequence numbers come from its tick counter, seq = tick * (kGroupBuckets + 1) + k, which advances on
// every group tick with update = 1, so a tick without a valid pair still takes new numbers.
// info non-NULL: an information workspace (_push_adapt_info / _push_adapt_group_info).
static int push_adapt(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                      const delora_odometry_train_group* g, int update, const float* points, const int32_t* n_points,
                      const int32_t* active, void* workspace, float* T, int32_t* valid, float* losses, float* info,
                      void* stream, const char* who) {
    const int S = d->max_batch;
    TrainPlan tp;
    AdaptPlan ap;
    make_adapt_plan(d, &tp, &ap);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    int rc;
    if ((rc = serve_adapt(d, hp, tp, ap, update, points, n_points, active, ws, T, valid, losses, info, st, who)))
        return rc;
    if (!update) return 0;
    const int32_t* n_valid = reinterpret_cast<const int32_t*>(ws + ap.n_valid);
    long long* tick = reinterpret_cast<long long*>(ws + ap.tick);
    constexpr unsigned kSeqStride = kGroupBuckets + 1;
    if (g) {                // the fleet-wide count of valid pairs, on every rank before its backward
        uint64_t peer_slots[kArMaxWorld];
        for (int q = 0; q < g->world; ++q) peer_slots[q] = g->peer_ws[q] + ap.slots;
        int32_t* n_fleet = reinterpret_cast<int32_t*>(ws + ap.n_fleet);
        if ((rc = count_allreduce_launch(peer_slots, g->peer_flags, g->rank, g->world, kSeqStride, tick, n_valid,
                                         n_fleet, g->status, st))) return rc;
        n_valid = n_fleet;
    }
    // each rank divides by the fleet-wide count, so the buckets are summed (scale 1)
    const GroupReduce gr{g, 1.0f, tick, kSeqStride, 1u};
    // 4. the backward of the mean over the valid pairs (invalid rows: dL/dT = 0), then Adam where n_valid > 0
    if ((rc = step_backward(tp, ws, d->act, S, false, DropoutCtr{nullptr, 0}, valid, n_valid, g ? &gr : nullptr, st,
                            who))) return rc;
    return adam_update(tp, ws, hp, n_valid, st);
}

}  // namespace delora

extern "C" int64_t delora_odometry_streams_adapt_workspace_bytes(const delora_odometry_desc* d) {
    return adapt_workspace_bytes(d, Adapt::plain, "delora_odometry_streams_adapt_workspace_bytes");
}

extern "C" int delora_odometry_streams_adapt_init(const delora_odometry_desc* d, const float* weights, void* workspace,
                                                  void* stream) {
    return adapt_init(d, Adapt::plain, weights, workspace, (cudaStream_t)stream, "delora_odometry_streams_adapt_init");
}

extern "C" int delora_odometry_streams_push_adapt(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                                  int update, const float* points, const int32_t* n_points,
                                                  const int32_t* active, void* workspace, float* T, int32_t* valid,
                                                  float* losses, void* stream) {
    const char* who = "delora_odometry_streams_push_adapt";
    if (check_push_adapt(d, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    return push_adapt(d, hp, nullptr, update, points, n_points, active, workspace, T, valid, losses, nullptr, stream,
                      who);
}

extern "C" int64_t delora_odometry_streams_adapt_group_workspace_bytes(const delora_odometry_desc* d) {
    return adapt_workspace_bytes(d, Adapt::group, "delora_odometry_streams_adapt_group_workspace_bytes");
}

extern "C" int delora_odometry_streams_adapt_group_init(const delora_odometry_desc* d, const float* weights,
                                                        void* workspace, void* stream) {
    return adapt_init(d, Adapt::group, weights, workspace, (cudaStream_t)stream, "delora_odometry_streams_adapt_group_init");
}

extern "C" int delora_odometry_streams_push_adapt_group(const delora_odometry_desc* d,
                                                        const delora_odometry_train_params* hp,
                                                        const delora_odometry_train_group* g, int update,
                                                        const float* points, const int32_t* n_points,
                                                        const int32_t* active, void* workspace, float* T,
                                                        int32_t* valid, float* losses, void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_group";
    if (check_push_adapt(d, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    if (check_group(g, workspace, who)) return 1;
    return push_adapt(d, hp, g->world > 1 && update ? g : nullptr, update, points, n_points, active, workspace, T,
                      valid, losses, nullptr, stream, who);
}

extern "C" int64_t delora_odometry_streams_adapt_info_workspace_bytes(const delora_odometry_desc* d) {
    return adapt_workspace_bytes(d, Adapt::info, "delora_odometry_streams_adapt_info_workspace_bytes");
}

extern "C" int delora_odometry_streams_adapt_info_init(const delora_odometry_desc* d, const float* weights,
                                                       void* workspace, void* stream) {
    return adapt_init(d, Adapt::info, weights, workspace, (cudaStream_t)stream,
                      "delora_odometry_streams_adapt_info_init");
}

extern "C" int delora_odometry_streams_push_adapt_info(const delora_odometry_desc* d,
                                                       const delora_odometry_train_params* hp, int update,
                                                       const float* points, const int32_t* n_points,
                                                       const int32_t* active, void* workspace, float* T,
                                                       int32_t* valid, float* losses, float* info, void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_info";
    if (check_push_adapt(d, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    DELORA_CHECK_ARG(info, "%s: null info", who);
    return push_adapt(d, hp, nullptr, update, points, n_points, active, workspace, T, valid, losses, info, stream,
                      who);
}

extern "C" int delora_odometry_streams_push_adapt_group_info(const delora_odometry_desc* d,
                                                             const delora_odometry_train_params* hp,
                                                             const delora_odometry_train_group* g, int update,
                                                             const float* points, const int32_t* n_points,
                                                             const int32_t* active, void* workspace, float* T,
                                                             int32_t* valid, float* losses, float* info,
                                                             void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_group_info";
    if (check_push_adapt(d, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    DELORA_CHECK_ARG(info, "%s: null info", who);
    if (check_group(g, workspace, who)) return 1;
    return push_adapt(d, hp, g->world > 1 && update ? g : nullptr, update, points, n_points, active, workspace, T,
                      valid, losses, info, stream, who);
}

extern "C" int delora_odometry_streams_adapt_reset(const delora_odometry_desc* d, const int32_t* mask, void* workspace,
                                                   void* stream) {
    const char* who = "delora_odometry_streams_adapt_reset";
    if (check_train_desc(d, who)) return 1;
    TrainPlan tp;
    AdaptPlan ap;
    make_adapt_plan(d, &tp, &ap);
    return reset_streams(d, mask, workspace, ap.has_prev, stream, who);
}

// ================================================================================================ adapting streams of
// several sensor geometries
// delora_odometry_streams_push_adapt_geometries: one model adapted from the streams of n geometries in one workspace.
// Layout: the adapting-streams workspace of d[0], unchanged; then for g = 1 .. n-1 d[g]'s geometry section (its
// training plan with the geometry section at the running offset), its stream section and one gradient slice in blob
// layout; then, for n > 1, the fleet section: the count of valid pairs over every geometry (int32 at +0) and geometry
// g's counters at +8 + 24 (g - 1), in the layout of the model section's (int64 [3]: a backward count nothing reads,
// the batch marker of g's ICP scratch, unused).  Geometry g's plan keeps d[0]'s model-section offsets (check_geometries
// makes them equal) with grad and ctr moved to its slice and counters, so train_forward_losses and step_backward run
// on it unchanged, and geometry 0's plan is _push_adapt's.  The _adapt_geometries_info form appends the information
// section after all of that (see make_geometries_plan), so no other offset moves.
namespace delora {

struct GeometriesPlan {
    TrainPlan tp[kMaxGeometries];
    AdaptPlan ap[kMaxGeometries];
    int row[kMaxGeometries];           // the first stream of geometry g in the caller's arrays
    size_t fleet;                      // n > 1 only
    size_t total;
    size_t info_total;                 // with the information section of _push_adapt_geometries_info
};

// TrainPlan is large (the trunk plan's tables): the plans of up to kMaxGeometries geometries go on the heap
static std::unique_ptr<GeometriesPlan> make_geometries_plan(const delora_odometry_desc* d, int n) {
    std::unique_ptr<GeometriesPlan> p(new GeometriesPlan);
    make_adapt_plan(&d[0], &p->tp[0], &p->ap[0]);
    size_t off = p->ap[0].total;
    p->row[0] = 0;
    for (int g = 1; g < n; ++g) {
        make_adapt_plan(&d[g], &p->tp[g], &p->ap[g], off);
        off = p->ap[g].total;
        p->tp[g].grad = take(off, (size_t)p->tp[g].m.blob_floats * 4);
        p->row[g] = p->row[g - 1] + d[g - 1].max_batch;
    }
    p->fleet = 0;
    if (n > 1) {
        p->fleet = take(off, 8 + 24 * (size_t)(n - 1));
        for (int g = 1; g < n; ++g) p->tp[g].ctr = p->fleet + 8 + 24 * (size_t)(g - 1);
    }
    p->total = off;
    // the information section of _push_adapt_geometries_info: the rows of all S_total pairs, then one info_scratch
    // sized for the largest geometry (their ICPs run one after another on one stream, and the scratch needs no
    // initialisation).  make_adapt_plan put ap.info / ap.info_scratch after a single-geometry group section, which here
    // lies in the next geometry's sections: every geometry's, g = 0 included, are moved into this section
    const size_t rows = take(off, (size_t)(p->row[n - 1] + d[n - 1].max_batch) * DELORA_INFO_ROW * 4);
    int64_t scratch = 0;
    for (int g = 0; g < n; ++g) {
        const int64_t floats = delora_icp_information_scratch_floats(d[g].max_batch, d[g].H, d[g].W);
        if (floats > scratch) scratch = floats;
    }
    const size_t info_scratch = take(off, (size_t)scratch * 4);
    for (int g = 0; g < n; ++g) {
        p->ap[g].info = rows + (size_t)p->row[g] * DELORA_INFO_ROW * 4;
        p->ap[g].info_scratch = info_scratch;
    }
    p->info_total = off;
    return p;
}

static int check_adapt_geometries(const delora_odometry_desc* d, int n, const char* who) {
    DELORA_CHECK_ARG(n <= kMaxGeometries, "%s: n=%d must be <= %d", who, n, kMaxGeometries);
    return check_geometries(d, n, who);
}

struct FleetCounts {
    const int32_t* n_valid[kMaxGeometries];
    int n;
};

// *fleet = the sum of every geometry's count of valid pairs, in geometry order
__global__ void odometry_fleet_count_kernel(FleetCounts c, int32_t* __restrict__ fleet) {
    int s = 0;
    for (int g = 0; g < c.n; ++g) s += *c.n_valid[g];
    *fleet = s;
}

// One tick of _push_adapt_geometries; info non-NULL: of _push_adapt_geometries_info, each geometry's information rows
// into its rows of info
static int push_adapt_geometries(const delora_odometry_desc* d, int n, const delora_odometry_train_params* hp,
                                 int update, const float* const* points, const int32_t* const* n_points,
                                 const int32_t* active, void* workspace, float* T, int32_t* valid, float* losses,
                                 float* info, void* stream, const char* who) {
    const std::unique_ptr<GeometriesPlan> p = make_geometries_plan(d, n);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    int rc;
    // 1-3 per geometry at B = S_g into its rows of the caller's arrays
    for (int g = 0; g < n; ++g) {
        const int r = p->row[g];
        if ((rc = serve_adapt(&d[g], hp, p->tp[g], p->ap[g], update, points[g], n_points[g], active ? active + r : nullptr,
                              ws, T + (size_t)r * 16, valid + r, losses + (size_t)r * DELORA_LOSS_ROW,
                              info ? info + (size_t)r * DELORA_INFO_ROW : nullptr, st, who)))
            return rc;
    }
    if (!update) return 0;
    // 4. every geometry's backward divides by the fleet's count of valid pairs, geometry g >= 1 into its slice; Adam
    // sums the slices into the model's gradient section
    const int32_t* fleet = reinterpret_cast<const int32_t*>(ws + p->ap[0].n_valid);
    GradSlices more;
    memset(&more, 0, sizeof(more));
    if (n > 1) {
        FleetCounts c;
        memset(&c, 0, sizeof(c));
        c.n = n;
        for (int g = 0; g < n; ++g) c.n_valid[g] = reinterpret_cast<const int32_t*>(ws + p->ap[g].n_valid);
        odometry_fleet_count_kernel<<<1, 1, 0, st>>>(c, reinterpret_cast<int32_t*>(ws + p->fleet));
        DELORA_CHECK_LAUNCH("odometry_fleet_count_kernel");
        fleet = reinterpret_cast<const int32_t*>(ws + p->fleet);
        more.n = n - 1;
        for (int g = 1; g < n; ++g) more.g[g - 1] = reinterpret_cast<const float*>(ws + p->tp[g].grad);
    }
    for (int g = 0; g < n; ++g)
        if ((rc = step_backward(p->tp[g], ws, d[g].act, d[g].max_batch, false, DropoutCtr{nullptr, 0}, valid + p->row[g],
                                fleet, nullptr, st, who))) return rc;
    return adam_update(p->tp[0], ws, hp, fleet, st, &more);
}

}  // namespace delora

extern "C" int64_t delora_odometry_streams_adapt_geometries_workspace_bytes(const delora_odometry_desc* d, int n) {
    if (check_adapt_geometries(d, n, "delora_odometry_streams_adapt_geometries_workspace_bytes")) return -1;
    return (int64_t)make_geometries_plan(d, n)->total;
}

extern "C" int delora_odometry_streams_adapt_geometries_init(const delora_odometry_desc* d, int n, const float* weights,
                                                             void* workspace, void* stream) {
    const char* who = "delora_odometry_streams_adapt_geometries_init";
    if (check_adapt_geometries(d, n, who)) return 1;
    const std::unique_ptr<GeometriesPlan> p = make_geometries_plan(d, n);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    // _train_init over the whole workspace arms geometry 0 and zeroes every other section
    int rc = train_init(&d[0], p->total, weights, workspace, st, who);
    if (rc) return rc;
    for (int g = 0; g < n; ++g) {
        const AdaptPlan& ap = p->ap[g];
        if ((rc = clear_grids(ws, ap.cache_pts, ap.cache_nrm, (size_t)d[g].max_batch * ap.cache_cells, st))) return rc;
        if (g == 0) continue;
        const cudaError_t e = cudaMemsetAsync(ws + p->tp[g].f.keys, 0xFF, p->tp[g].f.keys_bytes, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    }
    return 0;
}

namespace delora {

// What _push_adapt_geometries and _push_adapt_geometries_info refuse alike
static int check_push_adapt_geometries(const delora_odometry_desc* d, int n, const delora_odometry_train_params* hp,
                                       int update, const float* const* points, const int32_t* const* n_points,
                                       void* workspace, float* T, int32_t* valid, float* losses, const char* who) {
    if (check_adapt_geometries(d, n, who)) return 1;
    if (check_adapt_params(hp, update, who)) return 1;
    DELORA_CHECK_ARG(points, "%s: null points", who);
    DELORA_CHECK_ARG(n_points, "%s: null n_points", who);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    DELORA_CHECK_ARG(T, "%s: null T", who);
    DELORA_CHECK_ARG(valid, "%s: null valid", who);
    DELORA_CHECK_ARG(losses, "%s: null losses", who);
    for (int g = 0; g < n; ++g) {
        DELORA_CHECK_ARG(points[g], "%s: points[%d] is null", who, g);
        DELORA_CHECK_ARG(n_points[g], "%s: n_points[%d] is null", who, g);
        char w[192];
        snprintf(w, sizeof w, "%s: d[%d]", who, g);
        if (check_train_call(&d[g], hp, points[g], n_points[g], d[g].max_batch, workspace, w)) return 1;
    }
    return 0;
}

}  // namespace delora

extern "C" int delora_odometry_streams_push_adapt_geometries(const delora_odometry_desc* d, int n,
                                                             const delora_odometry_train_params* hp, int update,
                                                             const float* const* points,
                                                             const int32_t* const* n_points, const int32_t* active,
                                                             void* workspace, float* T, int32_t* valid, float* losses,
                                                             void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_geometries";
    if (check_push_adapt_geometries(d, n, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    return push_adapt_geometries(d, n, hp, update, points, n_points, active, workspace, T, valid, losses, nullptr,
                                 stream, who);
}

extern "C" int64_t delora_odometry_streams_adapt_geometries_info_workspace_bytes(const delora_odometry_desc* d, int n) {
    if (check_adapt_geometries(d, n, "delora_odometry_streams_adapt_geometries_info_workspace_bytes")) return -1;
    return (int64_t)make_geometries_plan(d, n)->info_total;
}

extern "C" int delora_odometry_streams_push_adapt_geometries_info(const delora_odometry_desc* d, int n,
                                                                  const delora_odometry_train_params* hp, int update,
                                                                  const float* const* points,
                                                                  const int32_t* const* n_points,
                                                                  const int32_t* active, void* workspace, float* T,
                                                                  int32_t* valid, float* losses, float* info,
                                                                  void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_geometries_info";
    if (check_push_adapt_geometries(d, n, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    DELORA_CHECK_ARG(info, "%s: null info", who);
    return push_adapt_geometries(d, n, hp, update, points, n_points, active, workspace, T, valid, losses, info, stream,
                                 who);
}

extern "C" int delora_odometry_streams_adapt_geometries_reset(const delora_odometry_desc* d, int n, const int32_t* mask,
                                                              void* workspace, void* stream) {
    const char* who = "delora_odometry_streams_adapt_geometries_reset";
    if (check_adapt_geometries(d, n, who)) return 1;
    DELORA_CHECK_ARG(mask, "%s: null mask", who);
    const std::unique_ptr<GeometriesPlan> p = make_geometries_plan(d, n);
    for (int g = 0; g < n; ++g) {
        const int rc = reset_streams(&d[g], mask + p->row[g], workspace, p->ap[g].has_prev, stream, who);
        if (rc) return rc;
    }
    return 0;
}

// ================================================================================================ dropout
namespace delora {

__global__ void odometry_set_seed_kernel(long long* __restrict__ ctr, unsigned long long seed) {
    ctr[2] = (long long)seed;
}

// keep[i] = 1 if element i of tensor t is kept at (seed, step), else 0; one thread per 4 elements (one Philox block)
__global__ void __launch_bounds__(256)
dropout_keep_mask_kernel(unsigned long long seed, unsigned long long step, int t, long long n, uint8_t* __restrict__ keep) {
    const long long q = (long long)blockIdx.x * 256 + threadIdx.x;
    if (q * 4 >= n) return;
    const Philox4 r = dropout_words(seed, step, t, (uint64_t)q);
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (q * 4 + k < n) keep[q * 4 + k] = dropout_word_keeps(philox_word(r, k)) ? 1 : 0;
}

}  // namespace delora

extern "C" int delora_odometry_train_set_dropout_seed(const delora_odometry_desc* d, uint64_t seed, void* workspace,
                                                      void* stream) {
    const char* who = "delora_odometry_train_set_dropout_seed";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    odometry_set_seed_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<long long*>((char*)workspace + tp.ctr),
                                                                (unsigned long long)seed);
    DELORA_CHECK_LAUNCH("odometry_set_seed_kernel");
    return 0;
}

extern "C" int delora_dropout_keep_mask(uint64_t seed, int64_t step, int tensor, int64_t n, uint8_t* keep, void* stream) {
    const char* who = "delora_dropout_keep_mask";
    DELORA_CHECK_ARG(keep, "%s: null keep", who);
    DELORA_CHECK_ARG(n >= 0, "%s: n=%lld must be >= 0", who, (long long)n);
    DELORA_CHECK_ARG(tensor >= 0 && tensor <= 2, "%s: tensor=%d must be 0 (input), 1 (stage-3 channels) or 2 (fc output)",
                     who, tensor);
    if (n == 0) return 0;
    const long long blocks = ((n + 3) / 4 + 255) / 256;
    dropout_keep_mask_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(seed, (unsigned long long)step, tensor, n,
                                                                                keep);
    DELORA_CHECK_LAUNCH("dropout_keep_mask_kernel");
    return 0;
}
