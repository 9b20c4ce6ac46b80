// The encoder trunk (trunk.cuh): plan, weight section, activation buffers, forward and backward launch sequences, and
// the delora_trunk_* entry points.  No kernel of its own but the stage-3 channel dropout of a dropout training step.
#include <cuda_bf16.h>
#include <string.h>

#include "trunk.cuh"

namespace delora {

thread_local TakeLog* take_log = nullptr;

int check_trunk(const int* layers, int H, int W, const char* who) {
    DELORA_CHECK_ARG(layers != nullptr, "%s: null layers", who);
    DELORA_CHECK_ARG(H >= 1 && W >= 2, "%s: bad image size H=%d W=%d", who, H, W);
    DELORA_CHECK_ARG(out_size(W, 2) % 2 == 0,
                     "%s: W=%d: the stem output width (W-1)/2+1 must be even for the max-pool", who, W);
    for (int s = 0; s < 4; ++s)
        DELORA_CHECK_ARG(layers[s] >= 1 && layers[s] <= kMaxBlocksPerStage, "%s: layers[%d]=%d must be in [1, %d]",
                         who, s, layers[s], kMaxBlocksPerStage);
    return 0;
}

void plan_trunk(const int* layers, int H, int W, TrunkPlan* m) {
    memset(m, 0, sizeof(TrunkPlan));
    m->H = H; m->W = W;
    m->w2 = out_size(W, 2); m->w4 = m->w2 / 2;
    m->stem_fast = W % 2 == 0;
    int64_t blob = 0;
    auto add_conv = [&](int cout, int cin, int k) {
        ConvLayer& c = m->conv[m->n_conv];
        c.cout = cout; c.cin = cin; c.k = k; c.blob = blob;
        blob += (int64_t)cout * cin * k * k;
        return m->n_conv++;
    };
    add_conv(64, 8, 3);                                     // resnet.conv1
    static const int widths[4] = {64, 128, 256, 512};
    static const int strides_h[4] = {1, 1, 1, 2}, strides_w[4] = {1, 2, 2, 2};
    int inplanes = 64, h = H, w = m->w4;
    for (int s = 0; s < 4; ++s) {
        for (int bi = 0; bi < layers[s]; ++bi) {
            Block& b = m->block[m->n_block++];
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
        m->stage_h[s] = h; m->stage_w[s] = w; m->stage_c[s] = widths[s];
    }
    m->conv_floats = blob;
}

TrunkWeights plan_trunk_weights(const TrunkPlan& m, bool flip, size_t& off) {
    TrunkWeights w;
    memset(&w, 0, sizeof(w));
    w.flip = flip;
    w.table = take(off, (size_t)m.n_conv * 8 * 8);
    for (int i = 0; i < m.n_conv; ++i) {
        const ConvLayer& c = m.conv[i];
        if (i == 0) {
            w.w_fwd[0] = take(off, m.stem_fast ? (size_t)3 * 64 * 64 * 2 : (size_t)64 * 9 * 64 * 2);
        } else {
            w.w_fwd[i] = take(off, (size_t)c.cout * c.k * c.k * c.cin * 2);
            if (flip) w.w_flip[i] = take(off, (size_t)c.cin * c.k * c.k * c.cout * 2);
        }
    }
    return w;
}

TrunkActs plan_trunk_acts(const TrunkPlan& m, int B, bool saving, size_t& off) {
    TrunkActs a;
    memset(&a, 0, sizeof(a));
    a.saving = saving;
    a.x_in = take(off, nhwc_bytes(B, m.H, m.W, m.stem_fast ? 16 : 64));
    a.stem = take(off, nhwc_bytes(B, m.H, m.w2, 64));
    if (!saving) {
        size_t act[4][3];
        for (int s = 0; s < 4; ++s)
            for (int j = 0; j < 3; ++j) act[s][j] = take(off, nhwc_bytes(B, m.stage_h[s], m.stage_w[s], m.stage_c[s]));
        a.pool = act[0][0];
        size_t cur = a.pool;
        for (int i = 0; i < m.n_block; ++i) {
            const Block& b = m.block[i];
            const size_t* r = act[b.stage];
            a.t1[i] = r[1];
            if (b.ds >= 0) {
                a.ds[i] = r[0];
                a.out[i] = r[2];
            } else {
                a.out[i] = cur == r[2] ? r[0] : r[2];
            }
            cur = a.out[i];
        }
        return a;
    }
    a.pool = take(off, nhwc_bytes(B, m.H, m.w4, 64));
    a.idx = take(off, (size_t)B * m.H * m.w4 * 64);
    for (int i = 0; i < m.n_block; ++i) {
        const Block& b = m.block[i];
        a.t1[i] = take(off, nhwc_bytes(B, b.hout, b.wout, b.cout));
        a.out[i] = take(off, nhwc_bytes(B, b.hout, b.wout, b.cout));
        if (b.ds >= 0) a.ds[i] = take(off, nhwc_bytes(B, b.hout, b.wout, b.cout));
    }
    for (int s = 0; s < 4; ++s)
        for (int j = 0; j < 3; ++j) a.g[s][j] = take(off, nhwc_bytes(B, m.stage_h[s], m.stage_w[s], m.stage_c[s]));
    for (int i = 0; i < m.n_block; ++i) {
        const Block& b = m.block[i];
        a.phase_dgrad[i] = b.ds >= 0 && i > 0 && delora_conv2d_dgrad_eligible(b.cin, b.cout, b.win, b.sh, b.sw);
        if (b.ds < 0) continue;
        a.gds[b.stage] = take(off, nhwc_bytes(B, b.hout, b.wout, b.cin));
        if (!a.phase_dgrad[i]) a.gu1[b.stage] = take(off, nhwc_bytes(B, b.hin, b.win, b.cout));
    }
    a.g_stem = take(off, nhwc_bytes(B, m.H, m.w2, 64));
    // the largest split-K need of any wgrad launch at B (the need grows with the batch)
    int64_t wg = m.stem_fast ? delora_stem_wgrad_scratch_floats(B, m.H, m.W)
                             : delora_conv2d_wgrad_scratch_floats(B, m.H, m.w2, 64, 64, 3);
    for (int i = 0; i < m.n_block; ++i) {
        const Block& b = m.block[i];
        int64_t n = delora_conv2d_wgrad_scratch_floats(B, b.hout, b.wout, b.cin, b.cout, 3);
        wg = n > wg ? n : wg;
        n = delora_conv2d_wgrad_scratch_floats(B, b.hout, b.wout, b.cout, b.cout, 3);
        wg = n > wg ? n : wg;
        if (b.ds >= 0) {
            n = delora_conv2d_wgrad_scratch_floats(B, b.hout, b.wout, b.cin, b.cout, 1);
            wg = n > wg ? n : wg;
        }
    }
    a.wg_scratch = take(off, (size_t)wg * 4);
    return a;
}

// The table rows {fp32 src, w_fwd, w_flip or 0, Cout, Cin, k, Cin_pad, kind}: the stem in the 16-channel layout
// (kind 1) when W is even, channel-padded to 64 otherwise.
int prep_trunk_weights(const TrunkPlan& m, const TrunkWeights& w, char* wbase, const float* const* src, cudaStream_t st,
                       const char* who) {
    long long table[kMaxConv * 8];
    for (int i = 0; i < m.n_conv; ++i) {
        const ConvLayer& c = m.conv[i];
        long long* r = table + (size_t)i * 8;
        r[0] = (long long)(uintptr_t)src[i];
        r[1] = (long long)(uintptr_t)(wbase + w.w_fwd[i]);
        r[2] = (w.flip && i > 0) ? (long long)(uintptr_t)(wbase + w.w_flip[i]) : 0;
        r[3] = c.cout; r[4] = c.cin; r[5] = c.k;
        r[6] = (i == 0) ? (m.stem_fast ? 16 : 64) : c.cin;
        r[7] = (i == 0 && m.stem_fast) ? 1 : 0;
    }
    const cudaError_t e = cudaMemcpyAsync(wbase + w.table, table, (size_t)m.n_conv * 8 * sizeof(long long),
                                          cudaMemcpyHostToDevice, st);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return delora_conv_weight_prep_multi(wbase + w.table, m.n_conv, st);
}

int trunk_input(const TrunkPlan& m, const TrunkActs& a, char* abase, const float* img1, const float* img2, int B,
                cudaStream_t st, DropoutCtr drop) {
    if (drop.ctr)
        return m.stem_fast ? launch_images_to_nhwc16_dropout(img1, img2, B, m.H, m.W, abase + a.x_in, drop, st)
                           : launch_images_to_nhwc_dropout(img1, img2, B, m.H, m.W, 64, abase + a.x_in, drop, st);
    return m.stem_fast ? delora_images_to_nhwc16_bf16(img1, img2, B, m.H, m.W, abase + a.x_in, st)
                       : delora_images_to_nhwc_bf16(img1, img2, B, m.H, m.W, 64, abase + a.x_in, st);
}

// The stage-3 channel dropout, Dropout2d on layer3's output: x, y [B, Hp, Wp, C] bf16, the padded NHWC layout with its
// halos (pix = Hp * Wp per pair).  y = bf16_rn(float(x) * 1.25f) where (pair b, channel c) is kept (element b * C + c
// of the stage-3 mask), 0 where it is dropped.  One thread per 8 channels (two Philox words); y may be x.  The forward
// writes x3d from layer3's output with it; the backward multiplies the data gradient of layer3's output in place.
__global__ void __launch_bounds__(256)
odometry_channel_dropout_kernel(const __nv_bfloat16* x, __nv_bfloat16* y, int B, int pix, int C, DropoutCtr drop) {
    const int groups = C / 8;
    const size_t total = (size_t)B * pix * groups;
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const int c0 = (int)(i % groups) * 8;
    const int b = (int)(i / ((size_t)groups * pix));
    uint64_t seed, step;
    dropout_seed_step(drop, seed, step);
    const uint64_t e0 = (uint64_t)b * C + c0;              // a multiple of 8: two whole Philox blocks
    const Philox4 r0 = dropout_words(seed, step, kDropStage3, e0 >> 2);
    const Philox4 r1 = dropout_words(seed, step, kDropStage3, (e0 >> 2) + 1);
    const uint32_t words[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
    uint4 v = reinterpret_cast<const uint4*>(x)[i];
    __nv_bfloat16* h = reinterpret_cast<__nv_bfloat16*>(&v);
#pragma unroll
    for (int k = 0; k < 8; ++k)
        h[k] = dropout_word_keeps(words[k]) ? __float2bfloat16_rn(__bfloat162float(h[k]) * kDropScale)
                                            : __float2bfloat16_rn(0.0f);
    reinterpret_cast<uint4*>(y)[i] = v;
}

static int channel_dropout(const TrunkPlan& m, const char* x, char* y, int B, DropoutCtr drop, cudaStream_t st) {
    const int C = m.stage_c[2], pix = (m.stage_h[2] + 2) * (m.stage_w[2] + 2);
    const size_t total = (size_t)B * pix * (C / 8);
    odometry_channel_dropout_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(y), B, pix, C, drop);
    DELORA_CHECK_LAUNCH("odometry_channel_dropout_kernel");
    return 0;
}

// The block whose output is layer3's (x3): the last block of stage 2
static int last_stage3_block(const TrunkPlan& m) {
    int i = 0;
    while (i + 1 < m.n_block && m.block[i + 1].stage <= 2) ++i;
    return i;
}

int trunk_forward(const TrunkPlan& m, const TrunkActs& a, char* abase, const TrunkWeights& w, const char* wbase, int act,
                  int B, float* pooled, void** stage_out, cudaStream_t st, DropoutCtr drop) {
    int rc;
    const bool saving = a.saving;
    const int H = m.H, W = m.W, stem_act = saving ? 0 : act;
    char* stem = abase + a.stem;
    if (m.stem_fast)
        rc = delora_stem_fprop_bf16(abase + a.x_in, wbase + w.w_fwd[0], stem, B, H, W, stem_act, saving ? 1 : 0, st);
    else
        rc = delora_conv2d_fprop_bf16(abase + a.x_in, wbase + w.w_fwd[0], nullptr, nullptr, stem, B, H, W, 64, 64, 3, 1,
                                      2, stem_act, st);
    if (rc) return rc;
    if (saving) rc = delora_maxpool_w_idx_nhwc_bf16(stem, B, H, m.w2, 64, abase + a.pool, abase + a.idx, act,
                                                    m.stem_fast, st);
    else rc = delora_maxpool_w_nhwc_bf16(stem, B, H, m.w2, 64, abase + a.pool, st);
    if (rc) return rc;
    const char* cur = abase + a.pool;
    for (int i = 0; i < m.n_block; ++i) {
        const Block& b = m.block[i];
        char* t1 = abase + a.t1[i];
        const char* ident = cur;
        if ((rc = delora_conv2d_fprop_bf16(cur, wbase + w.w_fwd[b.c1], nullptr, nullptr, t1, B, b.hin, b.win, b.cin,
                                           b.cout, 3, b.sh, b.sw, act, st))) return rc;
        if (b.ds >= 0) {
            ident = abase + a.ds[i];
            if ((rc = delora_conv2d_fprop_bf16(cur, wbase + w.w_fwd[b.ds], nullptr, nullptr, abase + a.ds[i], B, b.hin,
                                               b.win, b.cin, b.cout, 1, b.sh, b.sw, 0, st))) return rc;
        }
        if ((rc = delora_conv2d_fprop_bf16(t1, wbase + w.w_fwd[b.c2], ident, nullptr, abase + a.out[i], B, b.hout,
                                           b.wout, b.cout, b.cout, 3, 1, 1, act, st))) return rc;
        cur = abase + a.out[i];
        if (stage_out && (i + 1 == m.n_block || m.block[i + 1].stage != b.stage)) stage_out[b.stage] = (void*)cur;
        if (drop.ctr && i == last_stage3_block(m)) {
            if ((rc = channel_dropout(m, cur, abase + a.g[2][2], B, drop, st))) return rc;
            cur = abase + a.g[2][2];
        }
    }
    return delora_avgpool_nhwc_bf16(cur, B, m.stage_h[3], m.stage_w[3], 512, pooled, st);
}

// drop.ctr non-NULL (a dropout training step): layer4's first block read x3d (in g[2][2], see trunk_forward), so its
// two weight gradients read it too, while its act' epilogue reads x3; the data gradient of x3 is then multiplied by
// keep * 1.25 in place (one more bf16 rounding).  g[2][2] is first written by layer3's own backward, after that.
int trunk_backward(const TrunkPlan& m, const TrunkActs& a, char* abase, const TrunkWeights& w, const char* wbase, int act,
                   int B, const float* g_pooled, float* const* conv_dw, int stage, cudaStream_t st, DropoutCtr drop) {
    const int x3_block = last_stage3_block(m);
    int rc;
    const int act_bwd = act == 1 ? 4 : 3;                 // ACT_RELU_BWD / ACT_TANH_BWD: multiply by act'(saved)
    float* scratch = reinterpret_cast<float*>(abase + a.wg_scratch);
    // every stage's backward starts from the data gradient of its output in g[stage][0]
    char* dz2 = abase + a.g[stage][0];
    int first = 0;
    while (m.block[first].stage < stage) ++first;
    int last = first;
    while (last + 1 < m.n_block && m.block[last + 1].stage == stage) ++last;
    if (stage == 3 && (rc = delora_avgpool_bwd_nhwc_bf16(g_pooled, abase + a.out[last], B, m.stage_h[3], m.stage_w[3],
                                                         512, act, dz2, st))) return rc;
    for (int i = last; i >= first; --i) {
        const Block& b = m.block[i];
        const int s = b.stage;
        const char* x = i == 0 ? abase + a.pool : abase + a.out[i - 1];
        // the input the forward's convolutions read: x3d for layer4's first block in a dropout step
        const bool reads_x3d = drop.ctr && i == x3_block + 1;
        const char* xin = reads_x3d ? abase + a.g[2][2] : x;
        char* dz1 = abase + a.g[s][2];
        // the data gradient of the block input: the other buffer of this stage, or a buffer of the previous stage
        char* next;
        if (i > 0 && m.block[i - 1].stage != s) next = abase + a.g[m.block[i - 1].stage][0];
        else next = (dz2 == abase + a.g[s][0]) ? abase + a.g[s][1] : abase + a.g[s][0];
        if ((rc = delora_conv2d_wgrad_bf16(abase + a.t1[i], dz2, conv_dw[b.c2], scratch, B, b.hout, b.wout, b.cout,
                                           b.cout, b.cout, 3, 1, 1, st))) return rc;
        if ((rc = delora_conv2d_fprop_bf16(dz2, wbase + w.w_flip[b.c2], nullptr, abase + a.t1[i], dz1, B, b.hout, b.wout,
                                           b.cout, b.cout, 3, 1, 1, act_bwd, st))) return rc;
        if ((rc = delora_conv2d_wgrad_bf16(xin, dz1, conv_dw[b.c1], scratch, B, b.hin, b.win, b.cin, b.cin, b.cout, 3,
                                           b.sh, b.sw, st))) return rc;
        const char* resid = dz2;
        const char* src = dz1;
        if (b.ds >= 0) {
            if ((rc = delora_conv2d_wgrad_bf16(xin, dz2, conv_dw[b.ds], scratch, B, b.hin, b.win, b.cin, b.cin, b.cout, 1,
                                               b.sh, b.sw, st))) return rc;
            // the 1x1 strided downsample's data gradient: 1x1 convolution of the small dz, scattered afterwards
            char* small = abase + a.gds[s];
            if ((rc = delora_conv2d_fprop_bf16(dz2, wbase + w.w_flip[b.ds], nullptr, nullptr, small, B, b.hout, b.wout,
                                               b.cout, b.cin, 1, 1, 1, 0, st))) return rc;
            if (a.phase_dgrad[i]) {
                if ((rc = delora_conv2d_dgrad_bf16(dz1, wbase + w.w_flip[b.c1], small, x, next, B, b.hin, b.win, b.cin,
                                                   b.cout, b.sh, b.sw, act_bwd, 1, st))) return rc;
                if (reads_x3d && (rc = channel_dropout(m, next, next, B, drop, st))) return rc;
                dz2 = next;
                continue;
            }
            char* up_resid = abase + a.g[m.block[i - 1].stage][1];
            char* up_src = abase + a.gu1[s];
            if ((rc = delora_zero_upsample_nhwc_bf16(small, B, b.hout, b.wout, b.cin, b.sh, b.sw, b.hin, b.win, up_resid,
                                                     st))) return rc;
            if ((rc = delora_zero_upsample_nhwc_bf16(dz1, B, b.hout, b.wout, b.cout, b.sh, b.sw, b.hin, b.win, up_src,
                                                     st))) return rc;
            resid = up_resid;
            src = up_src;
        }
        // i > 0: the block input is the previous block's activation output, act' folds into the epilogue; the first
        // block reads the max-pool output (ACT_NONE: the pool's backward applies the stem's act')
        if ((rc = delora_conv2d_fprop_bf16(src, wbase + w.w_flip[b.c1], resid, i > 0 ? x : nullptr, next, B, b.hin,
                                           b.win, b.cout, b.cin, 3, 1, 1, i > 0 ? act_bwd : 0, st))) return rc;
        if (reads_x3d && (rc = channel_dropout(m, next, next, B, drop, st))) return rc;
        dz2 = next;
    }
    if (stage > 0) return 0;
    if ((rc = delora_maxpool_w_bwd_nhwc_bf16(dz2, abase + a.idx, abase + a.stem, B, m.H, m.w2, 64, 4 + act,
                                             abase + a.g_stem, m.stem_fast, st))) return rc;
    if (m.stem_fast)
        return delora_stem_wgrad_bf16(abase + a.x_in, abase + a.g_stem, conv_dw[0], scratch, B, m.H, m.W, 8, st);
    return delora_conv2d_wgrad_bf16(abase + a.x_in, abase + a.g_stem, conv_dw[0], scratch, B, m.H, m.W, 64, 8, 64, 3, 1,
                                    2, st);
}

}  // namespace delora

using namespace delora;

// The entry points' weight section always carries the flipped filters: the encoder that calls them trains.
extern "C" int64_t delora_trunk_weight_bytes(const int* layers, int W) {
    if (check_trunk(layers, 1, W, "delora_trunk_weight_bytes")) return -1;
    TrunkPlan m;
    plan_trunk(layers, 1, W, &m);
    size_t off = 0;
    plan_trunk_weights(m, true, off);
    return (int64_t)off;
}

extern "C" int delora_trunk_prep_weights(const int* layers, int W, const float* const* filters, void* weights,
                                         void* stream) {
    const char* who = "delora_trunk_prep_weights";
    if (check_trunk(layers, 1, W, who)) return 1;
    DELORA_CHECK_ARG(filters, "%s: null filters", who);
    DELORA_CHECK_ARG(weights, "%s: null weights", who);
    TrunkPlan m;
    plan_trunk(layers, 1, W, &m);
    for (int i = 0; i < m.n_conv; ++i) DELORA_CHECK_ARG(filters[i], "%s: null filters[%d]", who, i);
    size_t off = 0;
    const TrunkWeights w = plan_trunk_weights(m, true, off);
    return prep_trunk_weights(m, w, (char*)weights, filters, (cudaStream_t)stream, who);
}

static int check_batch(int B, int saving, const char* who) {
    DELORA_CHECK_ARG(B >= 1, "%s: B=%d must be >= 1", who, B);
    DELORA_CHECK_ARG(saving == 0 || saving == 1, "%s: saving=%d must be 0 or 1", who, saving);
    return 0;
}

extern "C" int64_t delora_trunk_activation_bytes(const int* layers, int B, int H, int W, int saving) {
    const char* who = "delora_trunk_activation_bytes";
    if (check_trunk(layers, H, W, who) || check_batch(B, saving, who)) return -1;
    TrunkPlan m;
    plan_trunk(layers, H, W, &m);
    size_t off = 0;
    plan_trunk_acts(m, B, saving != 0, off);
    return (int64_t)off;
}

// dropout_ctr (device int64[3], the training workspace's counter-slot layout: [0] the step, [2] the seed) non-NULL: the
// input and stage-3 dropouts of a training step at that step, read as DropoutCtr{ctr, 0} by the forward and by every
// backward call; NULL: no dropout.
static DropoutCtr trunk_dropout(const int64_t* dropout_ctr) {
    return DropoutCtr{reinterpret_cast<const long long*>(dropout_ctr), 0};
}

extern "C" int delora_trunk_forward_dropout(const int* layers, int B, int H, int W, int act, int saving,
                                            const float* img1, const float* img2, const void* weights, void* acts,
                                            float* pooled, void** stage_out, const int64_t* dropout_ctr,
                                            void* stream) {
    const char* who = dropout_ctr ? "delora_trunk_forward_dropout" : "delora_trunk_forward";
    if (check_trunk(layers, H, W, who) || check_batch(B, saving, who)) return 1;
    DELORA_CHECK_ARG(act == 1 || act == 2, "%s: act=%d must be 1 (relu) or 2 (tanh)", who, act);
    DELORA_CHECK_ARG(img1, "%s: null img1", who);
    DELORA_CHECK_ARG(img2, "%s: null img2", who);
    DELORA_CHECK_ARG(weights, "%s: null weights", who);
    DELORA_CHECK_ARG(acts, "%s: null acts", who);
    DELORA_CHECK_ARG(pooled, "%s: null pooled", who);
    // x3d lives in a backward buffer of the saving layout
    DELORA_CHECK_ARG(!dropout_ctr || saving == 1, "%s: dropout_ctr needs saving=1 (saving=%d)", who, saving);
    TrunkPlan m;
    plan_trunk(layers, H, W, &m);
    size_t woff = 0, aoff = 0;
    const TrunkWeights w = plan_trunk_weights(m, true, woff);
    const TrunkActs a = plan_trunk_acts(m, B, saving != 0, aoff);
    cudaStream_t st = (cudaStream_t)stream;
    const DropoutCtr drop = trunk_dropout(dropout_ctr);
    const int rc = trunk_input(m, a, (char*)acts, img1, img2, B, st, drop);
    if (rc) return rc;
    return trunk_forward(m, a, (char*)acts, w, (const char*)weights, act, B, pooled, stage_out, st, drop);
}

extern "C" int delora_trunk_forward(const int* layers, int B, int H, int W, int act, int saving, const float* img1,
                                    const float* img2, const void* weights, void* acts, float* pooled, void** stage_out,
                                    void* stream) {
    return delora_trunk_forward_dropout(layers, B, H, W, act, saving, img1, img2, weights, acts, pooled, stage_out,
                                        nullptr, stream);
}

extern "C" int delora_trunk_backward_dropout(const int* layers, int B, int H, int W, int act, const void* weights,
                                             void* acts, const float* g_pooled, float* const* conv_dw, int stage,
                                             const int64_t* dropout_ctr, void* stream) {
    const char* who = dropout_ctr ? "delora_trunk_backward_dropout" : "delora_trunk_backward";
    if (check_trunk(layers, H, W, who) || check_batch(B, 1, who)) return 1;
    DELORA_CHECK_ARG(act == 1 || act == 2, "%s: act=%d must be 1 (relu) or 2 (tanh)", who, act);
    DELORA_CHECK_ARG(stage >= 0 && stage <= 3, "%s: stage=%d must be in [0, 3]", who, stage);
    DELORA_CHECK_ARG(weights, "%s: null weights", who);
    DELORA_CHECK_ARG(acts, "%s: null acts", who);
    DELORA_CHECK_ARG(stage != 3 || g_pooled, "%s: null g_pooled", who);
    DELORA_CHECK_ARG(conv_dw, "%s: null conv_dw", who);
    TrunkPlan m;
    plan_trunk(layers, H, W, &m);
    for (int i = 0; i < m.n_block; ++i) {
        const Block& b = m.block[i];
        if (b.stage != stage) continue;
        DELORA_CHECK_ARG(conv_dw[b.c1] && conv_dw[b.c2] && (b.ds < 0 || conv_dw[b.ds]),
                         "%s: null conv_dw entry for block %d", who, i);
    }
    DELORA_CHECK_ARG(stage != 0 || conv_dw[0], "%s: null conv_dw[0] (the stem)", who);
    size_t woff = 0, aoff = 0;
    const TrunkWeights w = plan_trunk_weights(m, true, woff);
    const TrunkActs a = plan_trunk_acts(m, B, true, aoff);
    return trunk_backward(m, a, (char*)acts, w, (const char*)weights, act, B, g_pooled, conv_dw, stage,
                          (cudaStream_t)stream, trunk_dropout(dropout_ctr));
}

extern "C" int delora_trunk_backward(const int* layers, int B, int H, int W, int act, const void* weights, void* acts,
                                     const float* g_pooled, float* const* conv_dw, int stage, void* stream) {
    return delora_trunk_backward_dropout(layers, B, H, W, act, weights, acts, g_pooled, conv_dw, stage, nullptr,
                                         stream);
}
