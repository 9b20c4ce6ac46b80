// Odometry inference through the C ABI (sm_90a): raw scans -> relative transforms in one call.
//
// The trunk is the layer chain of the Python encoder (models/tc_encoder.py, TensorCoreEncoder.features + avgpool),
// written once here and run through the same entry points in the same order: projection, stem (16-channel layout
// when W is even, channel-padded conv2d_fprop otherwise), max-pool, the BasicBlocks with their 1x1 downsamples and
// fused residual + activation, average pool.  Inference keeps no activations, so each stage owns three buffers that
// its blocks rotate through.
//
// New here: the fully connected tail (reference: src/models/model.py:58-84, :103-116) in fp32.
//   odometry_linear_kernel: y = act(W x + b) for all B rows; one warp per output neuron, a float4 per lane per step.
//     The weight row is read from HBM once per call (batch rows after the first four hit L1), which is what bounds the
//     tail at small B: fc 512 x 1000 (2.05 MB) + heads (0.8 MB two heads / 1.7 MB single MLP).
//   odometry_out_kernel: the last Linear of each head (7 outputs per row), the division of the quaternion by the norm
//     of the WHOLE [B, 4] block (a quirk of the reference, :114) and quaternion -> T, in one CTA.
// Every sum has a fixed order (lane partials in k order, then an xor butterfly; the norm is one thread's loop), there
// are no atomics, so results are bit-identical from run to run and do not depend on B except through the norm.
#include <math.h>
#include <string.h>

#include "common.cuh"

namespace delora {

constexpr int kTailWarps = 8;
constexpr int kMaxBlocksPerStage = 16;
constexpr int kMaxConv = 1 + 4 * (2 * kMaxBlocksPerStage) + 3;
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
// warps [0, p0.N) compute p0's outputs, the next p1.N warps p1's.
__global__ void __launch_bounds__(kTailWarps * 32)
odometry_linear_kernel(TailLinear p0, TailLinear p1, int B, int act_out, int vec) {
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
        if (lane < nb) p.y[(size_t)(b0 + lane) * p.ldy + n] = tail_act(v + bn, act_out);
    }
}

// Last layer of the heads (rot: 4 outputs, trans: 3), quaternion / ||quaternion block||_F, quaternion -> T.
__global__ void __launch_bounds__(kTailWarps * 32)
odometry_out_kernel(TailLinear rot, TailLinear trans, int B, int vec, float* __restrict__ T) {
    extern __shared__ float s_out[];                        // [B, 7]: quaternion (x, y, z, w), translation
    __shared__ float s_norm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = warp; i < B * 7; i += kTailWarps) {
        const int b = i / 7, o = i - b * 7;
        const TailLinear p = o < 4 ? rot : trans;
        const int n = o < 4 ? o : o - 4;
        float acc[4];
        row_dot4(p.w + (size_t)n * p.K, p.x + (size_t)b * p.ldx, p.ldx, p.K, 1, lane, vec, acc);
        if (lane == 0) s_out[i] = acc[0] + __ldg(p.bias + n);
    }
    __syncthreads();
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
        quat_to_T_row(q[0] / nrm, q[1] / nrm, q[2] / nrm, q[3] / nrm, q[4], q[5], q[6], T + (size_t)b * 16);
    }
}

// counts[i] = clamp(n_points[i], 0, n_stride): the projection never reads past a scan's stride
__global__ void odometry_counts_kernel(const int32_t* __restrict__ n_in, int n, int n_stride, int32_t* __restrict__ n_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) n_out[i] = min(max(n_in[i], 0), n_stride);
}

// ---------------------------------------------------------------- the plan: layer sequence + workspace layout
struct ConvLayer {
    int cout, cin, k;
    int64_t blob;          // offset in floats of the fp32 filter in the weight blob
    size_t ws;             // byte offset of the bf16 w_fwd [cout, k*k, cin_pad] in the workspace
};
struct Block {
    int stage, sh, sw, c1, c2, ds;     // conv indices (ds = -1: identity shortcut)
    int hin, win, hout, wout, cin, cout;
};
struct Linear {
    int K, N;
    int64_t blob_w, blob_b;
    size_t ws_w, ws_b;
};
struct Plan {
    int H, W, w2, w4, stem_fast, MB;
    int n_conv, n_block, n_lin;
    ConvLayer conv[kMaxConv];
    Block block[4 * kMaxBlocksPerStage];
    Linear lin[kMaxLinear];            // two heads: rot1, rot2, trans1, trans2; single MLP: 5 layers
    Linear fc;
    int64_t blob_floats;
    int stage_h[4], stage_w[4], stage_c[4];
    // byte offsets
    size_t keys, index_map, counts, images, prev_image, x_in, stem, pool, act[4][3], table, pooled, fc_out, hid[2];
    size_t w_stem, total;
};

static size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }
static int out_size(int n, int s) { return (n - 1) / s + 1; }
static size_t nhwc_bytes(int b, int h, int w, int c) { return (size_t)b * (h + 2) * (w + 2) * c * 2; }

static int check_desc(const delora_odometry_desc* d, const char* who) {
    DELORA_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
    DELORA_CHECK_ARG(d->H >= 1 && d->W >= 2 && (long long)d->H * d->W < (1ll << 27),
                     "%s: bad image size H=%d W=%d", who, d->H, d->W);
    DELORA_CHECK_ARG(out_size(d->W, 2) % 2 == 0,
                     "%s: W=%d: the stem output width (W-1)/2+1 must be even for the max-pool", who, d->W);
    DELORA_CHECK_ARG(d->n_stride >= 1, "%s: n_stride=%d must be >= 1", who, d->n_stride);
    DELORA_CHECK_ARG(d->max_batch >= 1 && d->max_batch <= kMaxBatch, "%s: max_batch=%d must be in [1, %d]", who,
                     d->max_batch, kMaxBatch);
    DELORA_CHECK_ARG(d->act == 1 || d->act == 2, "%s: act=%d must be 1 (relu) or 2 (tanh)", who, d->act);
    for (int s = 0; s < 4; ++s)
        DELORA_CHECK_ARG(d->layers[s] >= 1 && d->layers[s] <= kMaxBlocksPerStage, "%s: layers[%d]=%d must be in [1, %d]",
                         who, s, d->layers[s], kMaxBlocksPerStage);
    DELORA_CHECK_ARG(d->resnet_outputs >= 1 && d->resnet_outputs <= 65536, "%s: resnet_outputs=%d must be in [1, 65536]",
                     who, d->resnet_outputs);
    DELORA_CHECK_ARG(d->single_mlp == 0 || d->single_mlp == 1, "%s: single_mlp=%d must be 0 or 1", who, d->single_mlp);
    DELORA_CHECK_ARG(isfinite(d->hfov0) && isfinite(d->hfov1) && isfinite(d->vfov0) && isfinite(d->vfov1) &&
                     d->hfov1 > d->hfov0 && d->vfov1 > d->vfov0, "%s: bad field of view", who);
    return 0;
}

// Walks the model in state_dict order (src/models/resnet_modified.py:49-66 + model.py:58-84) and lays out the
// workspace.  A pure function of the descriptor.
static void make_plan(const delora_odometry_desc* d, Plan* p) {
    memset(p, 0, sizeof(Plan));
    p->H = d->H; p->W = d->W; p->MB = d->max_batch;
    p->w2 = out_size(d->W, 2); p->w4 = p->w2 / 2;
    p->stem_fast = d->W % 2 == 0;
    int64_t blob = 0;
    auto add_conv = [&](int cout, int cin, int k) {
        ConvLayer& c = p->conv[p->n_conv];
        c.cout = cout; c.cin = cin; c.k = k; c.blob = blob;
        blob += (int64_t)cout * cin * k * k;
        return p->n_conv++;
    };
    add_conv(64, 8, 3);                                     // resnet.conv1
    static const int widths[4] = {64, 128, 256, 512};
    static const int strides_h[4] = {1, 1, 1, 2}, strides_w[4] = {1, 2, 2, 2};
    int inplanes = 64, h = d->H, w = p->w4;
    for (int s = 0; s < 4; ++s) {
        for (int bi = 0; bi < d->layers[s]; ++bi) {
            Block& b = p->block[p->n_block++];
            b.stage = s;
            b.sh = bi == 0 ? strides_h[s] : 1; b.sw = bi == 0 ? strides_w[s] : 1;
            b.hin = h; b.win = w; b.hout = out_size(h, b.sh); b.wout = out_size(w, b.sw);
            b.cin = inplanes; b.cout = widths[s];
            b.c1 = add_conv(b.cout, b.cin, 3);
            b.c2 = add_conv(b.cout, b.cout, 3);
            const bool strided = b.sh != 1 || b.sw != 1;
            b.ds = (bi == 0 && (strided || inplanes != widths[s])) ? add_conv(b.cout, b.cin, 1) : -1;
            inplanes = b.cout; h = b.hout; w = b.wout;
        }
        p->stage_h[s] = h; p->stage_w[s] = w; p->stage_c[s] = widths[s];
    }
    auto add_lin = [&](Linear& l, int K, int N) {
        l.K = K; l.N = N; l.blob_w = blob; blob += (int64_t)K * N; l.blob_b = blob; blob += N;
    };
    const int nout = d->resnet_outputs;
    add_lin(p->fc, 512, nout);
    if (d->single_mlp) {
        static const int dims[6] = {0, 512, 512, 256, 64, 7};
        int k = nout;
        for (int i = 1; i < 6; ++i) { add_lin(p->lin[p->n_lin++], k, dims[i]); k = dims[i]; }
    } else {
        add_lin(p->lin[0], nout, kHeadHidden); add_lin(p->lin[1], kHeadHidden, 4);     // fully_connected_rotation
        add_lin(p->lin[2], nout, kHeadHidden); add_lin(p->lin[3], kHeadHidden, 3);     // fully_connected_translation
        p->n_lin = 4;
    }
    p->blob_floats = blob;

    // workspace
    const int MB = d->max_batch, HW = d->H * d->W;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align256(bytes); return o; };
    p->keys = take((size_t)2 * MB * HW * 8);
    p->index_map = take((size_t)2 * MB * HW * 4);
    p->counts = take((size_t)2 * MB * 4);
    p->images = take((size_t)2 * MB * 4 * HW * 4);
    p->prev_image = take((size_t)4 * HW * 4);
    p->x_in = take(nhwc_bytes(MB, d->H, d->W, p->stem_fast ? 16 : 64));
    p->stem = take(nhwc_bytes(MB, d->H, p->w2, 64));
    // stage s buffers: [0] the pool output (stage 0) / the downsample output, [1] conv1 output, [2] block output;
    // later blocks of the stage alternate their output between [0] and [2]
    for (int s = 0; s < 4; ++s)
        for (int j = 0; j < 3; ++j) p->act[s][j] = take(nhwc_bytes(MB, p->stage_h[s], p->stage_w[s], p->stage_c[s]));
    p->pool = p->act[0][0];
    p->pooled = take((size_t)MB * 512 * 4);
    p->fc_out = take((size_t)MB * nout * 4);
    p->hid[0] = take((size_t)MB * 512 * 4);
    p->hid[1] = take((size_t)MB * 512 * 4);
    p->table = take((size_t)(kMaxConv + 1) * 8 * 8);
    p->w_stem = take(p->stem_fast ? (size_t)3 * 64 * 64 * 2 : (size_t)64 * 9 * 64 * 2);
    for (int i = 1; i < p->n_conv; ++i) {
        ConvLayer& c = p->conv[i];
        c.ws = take((size_t)c.cout * c.k * c.k * c.cin * 2);
    }
    p->conv[0].ws = p->w_stem;
    p->fc.ws_w = take((size_t)p->fc.K * p->fc.N * 4);
    p->fc.ws_b = take((size_t)p->fc.N * 4);
    for (int i = 0; i < p->n_lin; ++i) {
        p->lin[i].ws_w = take((size_t)p->lin[i].K * p->lin[i].N * 4);
        p->lin[i].ws_b = take((size_t)p->lin[i].N * 4);
    }
    p->total = off;
}

static int run_trunk(const Plan& p, char* ws, int act, const float* img1, const float* img2, int B, float* pooled,
                     cudaStream_t st) {
    int rc;
    const int H = p.H, W = p.W;
    void* x_in = ws + p.x_in;
    void* stem = ws + p.stem;
    if (p.stem_fast) {
        if ((rc = delora_images_to_nhwc16_bf16(img1, img2, B, H, W, x_in, st))) return rc;
        if ((rc = delora_stem_fprop_bf16(x_in, ws + p.w_stem, stem, B, H, W, act, 0, st))) return rc;
    } else {
        if ((rc = delora_images_to_nhwc_bf16(img1, img2, B, H, W, 64, x_in, st))) return rc;
        if ((rc = delora_conv2d_fprop_bf16(x_in, ws + p.w_stem, nullptr, nullptr, stem, B, H, W, 64, 64, 3, 1, 2, act, st)))
            return rc;
    }
    if ((rc = delora_maxpool_w_nhwc_bf16(stem, B, H, p.w2, 64, ws + p.pool, st))) return rc;
    char* cur = ws + p.pool;
    for (int i = 0; i < p.n_block; ++i) {
        const Block& b = p.block[i];
        char* r[3] = {ws + p.act[b.stage][0], ws + p.act[b.stage][1], ws + p.act[b.stage][2]};
        char* t1 = r[1];
        char* ident = cur;
        char* out = (cur == r[2]) ? r[0] : r[2];
        if ((rc = delora_conv2d_fprop_bf16(cur, ws + p.conv[b.c1].ws, nullptr, nullptr, t1, B, b.hin, b.win, b.cin, b.cout,
                                           3, b.sh, b.sw, act, st))) return rc;
        if (b.ds >= 0) {
            ident = r[0];
            out = r[2];
            if ((rc = delora_conv2d_fprop_bf16(cur, ws + p.conv[b.ds].ws, nullptr, nullptr, ident, B, b.hin, b.win, b.cin,
                                               b.cout, 1, b.sh, b.sw, 0, st))) return rc;
        }
        if ((rc = delora_conv2d_fprop_bf16(t1, ws + p.conv[b.c2].ws, ident, nullptr, out, B, b.hout, b.wout, b.cout, b.cout,
                                           3, 1, 1, act, st))) return rc;
        cur = out;
    }
    return delora_avgpool_nhwc_bf16(cur, B, p.stage_h[3], p.stage_w[3], 512, pooled, st);
}

static TailLinear tail_args(const Plan& p, char* ws, const Linear& l, const float* x, int ldx, float* y, int ldy) {
    TailLinear t;
    t.w = reinterpret_cast<const float*>(ws + l.ws_w);
    t.bias = reinterpret_cast<const float*>(ws + l.ws_b);
    t.x = x; t.y = y; t.K = l.K; t.N = l.N; t.ldx = ldx; t.ldy = ldy;
    return t;
}

static int run_tail(const Plan& p, char* ws, int act, const float* pooled, int B, float* T, cudaStream_t st) {
    float* fc_out = reinterpret_cast<float*>(ws + p.fc_out);
    float* hid[2] = {reinterpret_cast<float*>(ws + p.hid[0]), reinterpret_cast<float*>(ws + p.hid[1])};
    TailLinear none;
    memset(&none, 0, sizeof(none));
    auto linear = [&](const TailLinear& a, const TailLinear& b) {
        const int vec = (a.K % 4 == 0 && a.ldx % 4 == 0 && (b.N == 0 || (b.K % 4 == 0 && b.ldx % 4 == 0))) ? 1 : 0;
        const int warps = a.N + b.N;
        odometry_linear_kernel<<<(warps + kTailWarps - 1) / kTailWarps, kTailWarps * 32, 0, st>>>(a, b, B, act, vec);
        DELORA_CHECK_LAUNCH("odometry_linear_kernel");
        return 0;
    };
    int rc;
    const int nout = p.fc.N;
    if ((rc = linear(tail_args(p, ws, p.fc, pooled, 512, fc_out, nout), none))) return rc;     // act(resnet.fc(x))
    TailLinear rot, trans;
    if (p.n_lin == 4) {
        // hidden layers of both heads in one launch: hid[0] = [act(rot1 h) | act(trans1 h)], row stride 200
        const int ld = 2 * kHeadHidden;
        if ((rc = linear(tail_args(p, ws, p.lin[0], fc_out, nout, hid[0], ld),
                         tail_args(p, ws, p.lin[2], fc_out, nout, hid[0] + kHeadHidden, ld)))) return rc;
        rot = tail_args(p, ws, p.lin[1], hid[0], ld, nullptr, 0);
        trans = tail_args(p, ws, p.lin[3], hid[0] + kHeadHidden, ld, nullptr, 0);
    } else {
        const float* x = fc_out;
        int ldx = nout;
        for (int i = 0; i < p.n_lin - 1; ++i) {
            float* y = hid[i & 1];
            if ((rc = linear(tail_args(p, ws, p.lin[i], x, ldx, y, p.lin[i].N), none))) return rc;
            x = y; ldx = p.lin[i].N;
        }
        // fully_connected_rot_trans's last layer: rows 0..3 -> rotation, rows 4..6 -> translation
        const Linear& l = p.lin[p.n_lin - 1];
        rot = tail_args(p, ws, l, x, ldx, nullptr, 0);
        rot.N = 4;
        trans = rot;
        trans.w = rot.w + 4 * (size_t)l.K;
        trans.bias = rot.bias + 4;
        trans.N = 3;
    }
    const int vec = (rot.K % 4 == 0 && rot.ldx % 4 == 0) ? 1 : 0;
    odometry_out_kernel<<<1, kTailWarps * 32, (size_t)B * 7 * sizeof(float), st>>>(rot, trans, B, vec, T);
    DELORA_CHECK_LAUNCH("odometry_out_kernel");
    return 0;
}

static int project(const Plan& p, const delora_odometry_desc* d, char* ws, const float* points, const int32_t* n_points,
                   int n_scans, float* images, cudaStream_t st) {
    int32_t* counts = reinterpret_cast<int32_t*>(ws + p.counts);
    odometry_counts_kernel<<<(n_scans + 255) / 256, 256, 0, st>>>(n_points, n_scans, d->n_stride, counts);
    DELORA_CHECK_LAUNCH("odometry_counts_kernel");
    return delora_project_fwd(points, counts, n_scans, 3, d->n_stride, d->H, d->W, d->hfov0, d->hfov1, d->vfov0, d->vfov1,
                              0, reinterpret_cast<uint64_t*>(ws + p.keys), images,
                              reinterpret_cast<int32_t*>(ws + p.index_map), st);
}

}  // namespace delora

using namespace delora;

extern "C" int64_t delora_odometry_weight_floats(const delora_odometry_desc* d) {
    if (check_desc(d, "delora_odometry_weight_floats")) return -1;
    Plan p;
    make_plan(d, &p);
    return p.blob_floats;
}

extern "C" int64_t delora_odometry_workspace_bytes(const delora_odometry_desc* d) {
    if (check_desc(d, "delora_odometry_workspace_bytes")) return -1;
    Plan p;
    make_plan(d, &p);
    return (int64_t)p.total;
}

extern "C" int delora_odometry_init(const delora_odometry_desc* d, void* workspace, void* stream) {
    if (check_desc(d, "delora_odometry_init")) return 1;
    DELORA_CHECK_ARG(workspace, "delora_odometry_init: null workspace");
    Plan p;
    make_plan(d, &p);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    cudaError_t e = cudaMemsetAsync(ws, 0, p.total, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(ws + p.keys, 0xFF, (size_t)2 * p.MB * p.H * p.W * 8, st);
    DELORA_CHECK_ARG(e == cudaSuccess, "delora_odometry_init: %s", cudaGetErrorString(e));
    return 0;
}

extern "C" int delora_odometry_load_weights(const delora_odometry_desc* d, const float* weights, void* workspace,
                                            void* stream) {
    if (check_desc(d, "delora_odometry_load_weights")) return 1;
    DELORA_CHECK_ARG(weights && workspace, "delora_odometry_load_weights: null pointer");
    Plan p;
    make_plan(d, &p);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    // one delora_conv_weight_prep_multi row per filter: {fp32 src, w_fwd, w_flip, Cout, Cin, k, Cin_pad, kind};
    // the stem in the 16-channel layout (kind 1) when W is even, channel-padded to 64 otherwise
    long long table[kMaxConv * 8];
    for (int i = 0; i < p.n_conv; ++i) {
        const ConvLayer& c = p.conv[i];
        long long* r = table + (size_t)i * 8;
        r[0] = (long long)(uintptr_t)(weights + c.blob);
        r[1] = (long long)(uintptr_t)(ws + c.ws);
        r[2] = 0;
        r[3] = c.cout; r[4] = c.cin; r[5] = c.k;
        r[6] = (i == 0) ? (p.stem_fast ? 16 : 64) : c.cin;
        r[7] = (i == 0 && p.stem_fast) ? 1 : 0;
    }
    cudaError_t e = cudaMemcpyAsync(ws + p.table, table, (size_t)p.n_conv * 8 * sizeof(long long), cudaMemcpyHostToDevice, st);
    DELORA_CHECK_ARG(e == cudaSuccess, "delora_odometry_load_weights: %s", cudaGetErrorString(e));
    int rc = delora_conv_weight_prep_multi(ws + p.table, p.n_conv, st);
    if (rc) return rc;
    auto copy = [&](size_t dst, int64_t src, int64_t n) {
        return cudaMemcpyAsync(ws + dst, weights + src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, st);
    };
    e = copy(p.fc.ws_w, p.fc.blob_w, (int64_t)p.fc.K * p.fc.N);
    if (e == cudaSuccess) e = copy(p.fc.ws_b, p.fc.blob_b, p.fc.N);
    for (int i = 0; i < p.n_lin && e == cudaSuccess; ++i) {
        e = copy(p.lin[i].ws_w, p.lin[i].blob_w, (int64_t)p.lin[i].K * p.lin[i].N);
        if (e == cudaSuccess) e = copy(p.lin[i].ws_b, p.lin[i].blob_b, p.lin[i].N);
    }
    DELORA_CHECK_ARG(e == cudaSuccess, "delora_odometry_load_weights: %s", cudaGetErrorString(e));
    return 0;
}

extern "C" int delora_odometry_pairs(const delora_odometry_desc* d, const float* points, const int32_t* n_points, int B,
                                     void* workspace, float* T, float* pooled, void* stream) {
    if (check_desc(d, "delora_odometry_pairs")) return 1;
    DELORA_CHECK_ARG(points && n_points && workspace && T, "delora_odometry_pairs: null pointer");
    DELORA_CHECK_ARG(B >= 1 && B <= d->max_batch, "delora_odometry_pairs: B=%d outside [1, max_batch=%d]", B,
                     d->max_batch);
    Plan p;
    make_plan(d, &p);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    float* images = reinterpret_cast<float*>(ws + p.images);
    const size_t img = (size_t)4 * d->H * d->W;
    float* pooled_ws = reinterpret_cast<float*>(ws + p.pooled);
    int rc;
    if ((rc = project(p, d, ws, points, n_points, 2 * B, images, st))) return rc;
    if ((rc = run_trunk(p, ws, d->act, images, images + (size_t)B * img, B, pooled_ws, st))) return rc;
    if ((rc = run_tail(p, ws, d->act, pooled_ws, B, T, st))) return rc;
    if (pooled) {
        const cudaError_t e = cudaMemcpyAsync(pooled, pooled_ws, (size_t)B * 512 * sizeof(float), cudaMemcpyDeviceToDevice, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "delora_odometry_pairs: %s", cudaGetErrorString(e));
    }
    return 0;
}

extern "C" int delora_odometry_push(const delora_odometry_desc* d, const float* points, const int32_t* n_points,
                                    void* workspace, float* T, void* stream) {
    if (check_desc(d, "delora_odometry_push")) return 1;
    DELORA_CHECK_ARG(points && n_points && workspace, "delora_odometry_push: null pointer");
    Plan p;
    make_plan(d, &p);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    float* image = reinterpret_cast<float*>(ws + p.images);
    float* prev = reinterpret_cast<float*>(ws + p.prev_image);
    int rc;
    if ((rc = project(p, d, ws, points, n_points, 1, image, st))) return rc;
    if (T) {
        float* pooled_ws = reinterpret_cast<float*>(ws + p.pooled);
        if ((rc = run_trunk(p, ws, d->act, prev, image, 1, pooled_ws, st))) return rc;
        if ((rc = run_tail(p, ws, d->act, pooled_ws, 1, T, st))) return rc;
    }
    const cudaError_t e = cudaMemcpyAsync(prev, image, (size_t)4 * d->H * d->W * sizeof(float), cudaMemcpyDeviceToDevice, st);
    DELORA_CHECK_ARG(e == cudaSuccess, "delora_odometry_push: %s", cudaGetErrorString(e));
    return 0;
}
