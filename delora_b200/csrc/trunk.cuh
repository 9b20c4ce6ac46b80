// The encoder trunk (ResNetModified up to its average pool), decided once: the conv/block plan, the bf16 weight section,
// the activation buffers and the launch sequences of its forward and backward.  The odometry entry points
// (odometry*.cu) and the delora_trunk_* entry points that models/tc_encoder.py calls both run it.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "common.cuh"
#include "dropout.cuh"

namespace delora {

constexpr int kMaxBlocksPerStage = 64;
constexpr int kMaxBlocks = 4 * kMaxBlocksPerStage;
constexpr int kMaxConv = 1 + 2 * kMaxBlocks + 3;   // stem, two 3x3 per block, the 1x1 downsamples of stages 1..3

inline size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

// Every take() of a plan build while take_log is armed (delora_odometry_workspace_sections): its offset and the bytes
// asked for, in call order.  Unarmed (nullptr, every other caller) take() records nothing.
struct TakeLog {
    std::vector<size_t> off, bytes;
};
extern thread_local TakeLog* take_log;

inline size_t take(size_t& off, size_t bytes) {
    const size_t o = off;
    off += align256(bytes);
    if (take_log) { take_log->off.push_back(o); take_log->bytes.push_back(bytes); }
    return o;
}
inline int out_size(int n, int s) { return (n - 1) / s + 1; }
inline size_t nhwc_bytes(int b, int h, int w, int c) { return (size_t)b * (h + 2) * (w + 2) * c * 2; }

struct ConvLayer {
    int cout, cin, k;
    int64_t blob;          // offset in floats of the fp32 filter among the trunk's filters, in state_dict order
};
struct Block {
    int stage, sh, sw, c1, c2, ds;     // conv indices (ds = -1: identity shortcut)
    int hin, win, hout, wout, cin, cout;
};

// The layer sequence at one image size (src/models/resnet_modified.py:49-66): the stem (16-channel layout when W is
// even, channel-padded to 64 otherwise), the 3x3/(1,2) max-pool, the BasicBlocks of the four stages.
struct TrunkPlan {
    int H, W, w2, w4, stem_fast;
    int n_conv, n_block;
    ConvLayer conv[kMaxConv];
    Block block[kMaxBlocks];
    int64_t conv_floats;               // all filters
    int stage_h[4], stage_w[4], stage_c[4];
};

// The weight section: the delora_conv_weight_prep_multi table (one row per filter), each filter's bf16 forward copy
// w_fwd [cout, k*k, cin_pad] and, with flip (training), its flipped copy w_flip for the data gradient (every filter but
// the stem's).
struct TrunkWeights {
    bool flip;
    size_t table, w_fwd[kMaxConv], w_flip[kMaxConv];
};

// The activation buffers.  The input (16 channels when W is even, 64 otherwise), the stem output and the max-pool
// output, then for every block i its conv1 output t1[i], its downsample output ds[i] and its output out[i].
// Inference keeps no activations: each stage owns three buffers, [0] the pool output (stage 0) / the downsample output,
// [1] conv1 output, [2] block output; later blocks of the stage alternate their output between [0] and [2].
// saving (training) keeps every activation, the pool's argmax and the stem's pre-activation, plus the backward's:
// per stage two alternating data-gradient buffers and the conv1 gradient g[s][0..2]; per downsampling block the
// downsample's gradient at the output size and (zero-upsample path) the upsampled conv1 gradient; the stem's gradient;
// one split-K scratch for every wgrad launch.
struct TrunkActs {
    bool saving;
    size_t x_in, stem, pool, idx, t1[kMaxBlocks], ds[kMaxBlocks], out[kMaxBlocks];
    size_t g[4][3], gds[4], gu1[4], g_stem, wg_scratch;
    int phase_dgrad[kMaxBlocks];       // the block's strided conv1 takes the phase-decomposed data gradient
};

// layers[4] in [1, kMaxBlocksPerStage], H >= 1, W >= 2 with out_size(W, 2) even (the max-pool halves it)
int check_trunk(const int* layers, int H, int W, const char* who);
// a pure function of its arguments (checked by check_trunk)
void plan_trunk(const int* layers, int H, int W, TrunkPlan* m);
TrunkWeights plan_trunk_weights(const TrunkPlan& m, bool flip, size_t& off);
// buffers for up to B pairs
TrunkActs plan_trunk_acts(const TrunkPlan& m, int B, bool saving, size_t& off);

// The bf16 filters of the section at wbase from the fp32 filters src[i] (conv order): the table rows, then one
// delora_conv_weight_prep_multi launch.  The table is copied from host memory.
int prep_trunk_weights(const TrunkPlan& m, const TrunkWeights& w, char* wbase, const float* const* src, cudaStream_t st,
                       const char* who);

// (img1, img2) fp32 [B, 4, H, W] each -> the trunk input; drop.ctr non-NULL: with the input dropout applied
int trunk_input(const TrunkPlan& m, const TrunkActs& a, char* abase, const float* img1, const float* img2, int B,
                cudaStream_t st, DropoutCtr drop = DropoutCtr{nullptr, 0});

// The trunk from its input to the pooled features [B, 512] fp32.  a.saving: the stem keeps its PRE-activation (fp16 on
// the 16-channel path) and the max-pool applies the activation and records its argmax; otherwise the stem applies it.
// stage_out non-NULL: the addresses of x1..x4 (each stage's output).  drop.ctr non-NULL (a dropout training step,
// saving): layer3's output x3 stays as it is (the backward's act' reads it), the channel-dropped x3d is written to
// g[2][2] (which nothing writes before layer3's own backward) and layer4's first block reads it.
int trunk_forward(const TrunkPlan& m, const TrunkActs& a, char* abase, const TrunkWeights& w, const char* wbase, int act,
                  int B, float* pooled, void** stage_out, cudaStream_t st, DropoutCtr drop = DropoutCtr{nullptr, 0});

// The backward of one stage, run for stage 3, 2, 1, 0 in turn after a saving trunk_forward: stage 3 starts with the
// average pool's backward from g_pooled [B, 512] fp32, stage 0 ends with the max-pool's backward and the stem's wgrad.
// The weight gradient of conv c goes to conv_dw[c] ([cout, cin, k, k] fp32).
int trunk_backward(const TrunkPlan& m, const TrunkActs& a, char* abase, const TrunkWeights& w, const char* wbase, int act,
                   int B, const float* g_pooled, float* const* conv_dw, int stage, cudaStream_t st,
                   DropoutCtr drop = DropoutCtr{nullptr, 0});

}  // namespace delora
