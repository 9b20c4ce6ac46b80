// Encoder stem on the Hopper tensor cores (wgmma): conv3x3, stride (1,2), 8 -> 64 channels, circular W / zero H padding, + activation
// (reference: src/models/resnet_modified.py:40 `self.conv1`, used at :97-99; the 8 input channels are
// cat(image_1, image_2), src/models/model.py:98).
//
// Input precision: the range images hold metres (up to ~100): a single bf16 would quantise them to 0.25-0.5 m steps.  The
// 8 spare channels carry the rounding residual: channel c = bf16(x), channel c + 8 = bf16(x - bf16(x)), both multiplied
// by the same filter weight, so the stem sees the input with ~16 mantissa bits at no extra tensor-core work.
//
// Round 1 ran this layer through the generic kernel with the 8 channels padded to 64: K = 9 taps x 64 = 576 for 72
// real products per output (8x wasted MMAs, 277 MB input tensor).  Here the input is stored with 16 channels
// [B, H+2, W+2, 16] bf16 (8 real + 8 zero, 32 B per pixel) and ONE tensor-map row gives, for output pixel wo and filter
// row r, the 4 consecutive input pixels 2 wo .. 2 wo + 3 of padded row h + r = 64 contiguous elements (128 B): the
// tensor map's pixel dimension advances by 2 pixels (64 B) while a row is 4 pixels long -- overlapping strides in the
// tensor map.  The three filter columns are the first three pixels of that window (the fourth
// has zero weights), so the convolution is a GEMM with K = 3 rows x 64 and no im2col buffer.
//   fprop:  M = 128 output pixels of one row (two consumer warpgroups of 64), N = 64 output channels, 12 wgmma per
//           tile, filters resident in smem, persistent CTAs.
//   wgrad:  the plan-driven kernel of conv_wgrad.cu (mode 2) on the same tensor map.
#include <string.h>
#include <cuda_fp16.h>
#include "conv_internal.cuh"
#include "dropout.cuh"

namespace delora {

constexpr int kStemThreads = 288;               // two consumer warpgroups + one producer warp (warp 8)
constexpr int kStemStages = 3;
constexpr int kStemTile = 128 * 128;            // one filter row of a tile: 128 pixels x 128 B

struct StemParams {
    int B, H, Wout, segs, n_jobs, act;
    int out_f16;        // 1: store fp16 instead of bf16 (training: the pre-activation feeds only the two pool kernels,
                        //    3 more mantissa bits keep the pool's argmax on the fp32 winner in near-ties)
};

__global__ void __launch_bounds__(kStemThreads, 1)
stem_fprop_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                     __nv_bfloat16* __restrict__ y, const __grid_constant__ StemParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = DELORA_ALIGNED_SMEM(smem_raw);
    uint8_t* smem_w = smem;                                         // 3 x [64 co][64 k] K-major = 24 KB
    uint8_t* smem_a = smem + 3 * 8192;                              // ring of 3 stages x 3 filter rows x 16 KB
    float* acc_tiles = reinterpret_cast<float*>(smem_a + kStemStages * 3 * kStemTile);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(acc_tiles) + 2 * kAccTileBytes);
    uint64_t* empty_bar = full_bar + kStemStages;
    uint64_t* w_bar = empty_bar + kStemStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStemStages; ++s) { mbar_init(full_bar + s, 1); mbar_init(empty_bar + s, 8); }
        mbar_init(w_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            tma_prefetch_desc(&map_x);
            mbar_expect_tx(w_bar, 3 * 8192);
            for (int r = 0; r < 3; ++r) tma_load_2d(smem_w + r * 8192, &map_w, w_bar, 0, r * 64);
            uint32_t s = 0, ph = 0;
            for (int job = blockIdx.x; job < p.n_jobs; job += gridDim.x) {
                int t = job;
                const int seg = t % p.segs; t /= p.segs;
                const int h = t % p.H;
                const int b = t / p.H;
                mbar_wait(empty_bar + s, ph ^ 1);
                mbar_expect_tx(full_bar + s, 3 * kStemTile);
                for (int r = 0; r < 3; ++r)
                    tma_load_4d(smem_a + (s * 3 + r) * kStemTile, &map_x, full_bar + s, 0, seg * 128, h + r, b);
                if (++s == kStemStages) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    // warpgroup wg: output pixels 64 wg .. 64 wg + 63 of the 128-pixel row segment
    const int wg = warp >> 2;
    const int row = threadIdx.x & 63, half = (threadIdx.x >> 6) & 1;
    float* tile = acc_tiles + wg * (kAccTileBytes / 4);
    const int Wp = p.Wout + 2, Hp = p.H + 2;
    mbar_wait(w_bar, 0);
    uint32_t s = 0, ph = 0;
    for (int job = blockIdx.x; job < p.n_jobs; job += gridDim.x) {
        int t = job;
        const int seg = t % p.segs; t /= p.segs;
        const int h = t % p.H;
        const int b = t / p.H;
        float acc[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] = 0.0f;
        mbar_wait(full_bar + s, ph);
        wgmma_fence();
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int k = 0; k < 4; ++k)
                wgmma_64x64x16<0, 0>(acc, make_smem_desc(smem_u32(smem_a + (s * 3 + r) * kStemTile + wg * 8192)) + (uint64_t)(k * 2),
                                     make_smem_desc(smem_u32(smem_w + r * 8192)) + (uint64_t)(k * 2));
        wgmma_commit();
        wgmma_wait_all();
        if (lane == 0) mbar_arrive(empty_bar + s);
        if (++s == kStemStages) { s = 0; ph ^= 1; }
        wg_sync(wg);
        acc_stage(acc, tile);
        wg_sync(wg);
        const int wo = seg * 128 + wg * 64 + row, c0 = half * 32;
        const size_t pix = ((size_t)b * Hp + (h + 1)) * Wp + (wo + 1);
        if (wo < p.Wout) {
            float v[32];
            acc_row32(tile, row, c0, v);
            if (p.out_f16) {
                uint4 out[4];
#pragma unroll
                for (int j4 = 0; j4 < 4; ++j4) {
                    __half2 hh[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        hh[e] = __floats2half2_rn(apply_act(v[j4 * 8 + e * 2], p.act), apply_act(v[j4 * 8 + e * 2 + 1], p.act));
                    out[j4] = *reinterpret_cast<uint4*>(hh);
                }
                uint4* yp = reinterpret_cast<uint4*>(y + pix * 64 + c0);
#pragma unroll
                for (int j4 = 0; j4 < 4; ++j4) yp[j4] = out[j4];
                if (wo == 0) {
                    uint4* hp = reinterpret_cast<uint4*>(y + (pix + p.Wout) * 64 + c0);
#pragma unroll
                    for (int j4 = 0; j4 < 4; ++j4) hp[j4] = out[j4];
                }
                if (wo == p.Wout - 1) {
                    uint4* hp = reinterpret_cast<uint4*>(y + (pix - p.Wout) * 64 + c0);
#pragma unroll
                    for (int j4 = 0; j4 < 4; ++j4) hp[j4] = out[j4];
                }
            } else {
                epilogue_store32(v, nullptr, nullptr, y, pix * 64 + c0, p.act, wo == 0, wo == p.Wout - 1, (size_t)p.Wout * 64);
            }
        }
    }
}

// two [B,4,H,W] fp32 range images -> [B, H+2, W+2, 16] bf16: channels 0..7 = bf16(cat(image_1, image_2))
// (src/models/model.py:98), 8..15 = bf16 of the rounding residual; circular halo columns, zero halo rows.
// kDrop (the training step's input dropout): element (b, c, h, w) is first multiplied by keep * 1.25f in fp32, so the
// split sees the bits of images that were multiplied beforehand.
template <bool kDrop>
__device__ __forceinline__ void images_to_nhwc16_body(const float* __restrict__ img1, const float* __restrict__ img2,
                                                      int B, int H, int W, __nv_bfloat16* __restrict__ x,
                                                      const DropoutCtr& drop) {
    const int Wp = W + 2, Hp = H + 2;
    const size_t total = (size_t)B * Hp * Wp;
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const int wp = (int)(i % Wp), hp = (int)((i / Wp) % Hp), b = (int)(i / ((size_t)Wp * Hp));
    uint4 lo = make_uint4(0u, 0u, 0u, 0u), hi_part = make_uint4(0u, 0u, 0u, 0u);
    if (hp != 0 && hp != Hp - 1) {
        int w = wp - 1;
        if (w < 0) w = W - 1;
        if (w >= W) w = 0;
        const int h = hp - 1;
        const size_t base = ((size_t)b * 4 * H + h) * W + w, plane = (size_t)H * W;
        float f[8];
#pragma unroll
        for (int c = 0; c < 4; ++c) { f[c] = __ldg(img1 + base + c * plane); f[4 + c] = __ldg(img2 + base + c * plane); }
        if (kDrop) {
            uint64_t seed, step;
            dropout_seed_step(drop, seed, step);
            const size_t e0 = ((size_t)b * 8 * H + h) * W + w;         // element (b, 0, h, w); channel c adds c * plane
#pragma unroll
            for (int c = 0; c < 8; ++c)
                f[c] = dropout_keep(seed, step, kDropInput, e0 + c * plane) ? f[c] * kDropScale : 0.0f;
        }
        __nv_bfloat16 hv[8], lv[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            hv[c] = __float2bfloat16_rn(f[c]);
            lv[c] = __float2bfloat16_rn(f[c] - __bfloat162float(hv[c]));     // rounding residual (exact difference)
        }
        lo = *reinterpret_cast<uint4*>(hv);
        hi_part = *reinterpret_cast<uint4*>(lv);
    }
    uint4* dst = reinterpret_cast<uint4*>(x + i * 16);
    dst[0] = lo;
    dst[1] = hi_part;
}

__global__ void __launch_bounds__(256)
images_to_nhwc16_kernel(const float* __restrict__ img1, const float* __restrict__ img2, int B, int H, int W,
                        __nv_bfloat16* __restrict__ x) {
    images_to_nhwc16_body<false>(img1, img2, B, H, W, x, DropoutCtr{nullptr, 0});
}

__global__ void __launch_bounds__(256)
images_to_nhwc16_dropout_kernel(const float* __restrict__ img1, const float* __restrict__ img2, int B, int H, int W,
                                __nv_bfloat16* __restrict__ x, DropoutCtr drop) {
    images_to_nhwc16_body<true>(img1, img2, B, H, W, x, drop);
}

// fp32 stem filter [64, 8, 3, 3] -> bf16 [3 rows][64 co][64 k], k = q * 16 + c (q < 3, c < 8), zero elsewhere
__global__ void __launch_bounds__(256)
stem_weight_prep_kernel(const float* __restrict__ w, int Cin, __nv_bfloat16* __restrict__ w_stem) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= 3 * 64 * 64) return;
    const int k = i & 63, co = (i >> 6) & 63, r = i >> 12;
    const int q = k >> 4, c = k & 15;
    const int cr = c & 7;                                 // channels 8..15 (input residuals) reuse the weights of 0..7
    const float v = (q < 3 && cr < Cin) ? __ldg(w + ((size_t)co * Cin + cr) * 9 + r * 3 + q) : 0.0f;
    w_stem[i] = __float2bfloat16_rn(v);
}

// All filters of the encoder in ONE launch: table[l] = {fp32 weight ptr, fwd ptr, flip ptr, Cout, Cin, k, Cin_pad, kind}
// (int64 each; kind 0 = the two layouts of weight_prep_kernel (conv_tc.cu), kind 1 = the stem layout above).
// blockIdx.y = layer, blockIdx.x strides over the layer's elements.
constexpr int kPrepTile = 32;
__global__ void __launch_bounds__(256)
weight_prep_multi_kernel(const long long* __restrict__ table) {
    const long long* e = table + (size_t)blockIdx.y * 8;
    const float* __restrict__ w = reinterpret_cast<const float*>(e[0]);
    __nv_bfloat16* __restrict__ w_fwd = reinterpret_cast<__nv_bfloat16*>(e[1]);
    __nv_bfloat16* __restrict__ w_flip = reinterpret_cast<__nv_bfloat16*>(e[2]);
    const int Cout = (int)e[3], Cin = (int)e[4], k = (int)e[5], Cin_pad = (int)e[6], kind = (int)e[7];
    const int taps = k * k;
    if (kind == 1) {
        for (int i = blockIdx.x * 256 + threadIdx.x; i < 3 * 64 * 64; i += gridDim.x * 256) {
            const int kk = i & 63, co = (i >> 6) & 63, r = i >> 12;
            const int q = kk >> 4, c = kk & 15;
            const int cr = c & 7;
            w_fwd[i] = __float2bfloat16_rn((q < 3 && cr < Cin) ? __ldg(w + ((size_t)co * Cin + cr) * 9 + r * 3 + q) : 0.0f);
        }
        return;
    }
    if (Cout % kPrepTile == 0 && Cin % kPrepTile == 0 && Cin_pad == Cin && taps <= 9) {
        // Tiled transposes: a (32 co x 32 ci x taps) block is read as 32 contiguous runs of 32 * taps floats, parked in
        // shared memory (row stride 32 * 9 + 1: both read-outs are bank-conflict free) and written as 64-byte runs of
        // both layouts.  The element-wise form below reads every 32-byte sector of the fp32 filter 8 times per layout
        // through L2; this form reads it once.
        __shared__ float tile[kPrepTile * (kPrepTile * 9 + 1)];
        constexpr int RS = kPrepTile * 9 + 1;
        const int run = kPrepTile * taps;
        const int tiles_ci = Cin / kPrepTile, n_tiles = (Cout / kPrepTile) * tiles_ci;
        for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
            const int co0 = (t / tiles_ci) * kPrepTile, ci0 = (t % tiles_ci) * kPrepTile;
            __syncthreads();
            for (int i = threadIdx.x; i < kPrepTile * run; i += 256) {
                const int co = i / run, r = i - co * run;
                tile[co * RS + r] = __ldg(w + ((size_t)(co0 + co) * Cin + ci0) * taps + r);
            }
            __syncthreads();
            for (int i = threadIdx.x; i < kPrepTile * run; i += 256) {
                const int ci = i % kPrepTile, tap = (i / kPrepTile) % taps, co = i / run;
                w_fwd[((size_t)(co0 + co) * taps + tap) * Cin_pad + ci0 + ci] = __float2bfloat16_rn(tile[co * RS + ci * taps + tap]);
            }
            if (w_flip) {
                for (int i = threadIdx.x; i < kPrepTile * run; i += 256) {
                    const int co = i % kPrepTile, tap = (i / kPrepTile) % taps, ci = i / run;
                    w_flip[((size_t)(ci0 + ci) * taps + tap) * Cout + co0 + co] =
                        __float2bfloat16_rn(tile[co * RS + ci * taps + (taps - 1 - tap)]);
                }
            }
        }
        return;
    }
    const size_t n_fwd = (size_t)Cout * taps * Cin_pad, n_flip = w_flip ? (size_t)Cin * taps * Cout : 0;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n_fwd + n_flip; i += (size_t)gridDim.x * 256) {
        if (i < n_fwd) {
            const int ci = (int)(i % Cin_pad), tap = (int)((i / Cin_pad) % taps), co = (int)(i / ((size_t)Cin_pad * taps));
            w_fwd[i] = __float2bfloat16_rn(ci < Cin ? __ldg(w + ((size_t)co * Cin + ci) * taps + tap) : 0.0f);
        } else {
            const size_t j = i - n_fwd;
            const int co = (int)(j % Cout), tap = (int)((j / Cout) % taps), ci = (int)(j / ((size_t)Cout * taps));
            w_flip[j] = __float2bfloat16_rn(__ldg(w + ((size_t)co * Cin + ci) * taps + (taps - 1 - tap)));
        }
    }
}

// the overlapping-stride view of the 16-channel input: (k, wo, hp, b) -> x16[b][hp][2 wo + k / 16][k % 16]
static int stem_encode_x_map(CUtensorMap* m, const void* x16, int B, int H, int W) {
    const int Hp = H + 2, Wp = W + 2, Wout = W / 2;
    const cuuint64_t dims[4] = {64, (cuuint64_t)Wout, (cuuint64_t)Hp, (cuuint64_t)B};
    const cuuint64_t strides[3] = {64, (cuuint64_t)Wp * 32, (cuuint64_t)Hp * Wp * 32};
    const cuuint32_t box[4] = {64, 128, 1, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    return tma_encode(m, x16, 4, dims, strides, box, estr, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

}  // namespace delora

using namespace delora;

extern "C" int delora_images_to_nhwc16_bf16(const float* image_1, const float* image_2, int B, int H, int W, void* x16,
                                            void* stream) {
    DELORA_CHECK_ARG(image_1 && image_2 && x16 && B > 0 && H > 0 && W > 0, "delora_images_to_nhwc16_bf16: bad argument");
    const size_t total = (size_t)B * (H + 2) * (W + 2);
    images_to_nhwc16_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(image_1, image_2, B, H, W,
                                                                                               (__nv_bfloat16*)x16);
    DELORA_CHECK_LAUNCH("images_to_nhwc16_kernel");
    return 0;
}

int delora::launch_images_to_nhwc16_dropout(const float* img1, const float* img2, int B, int H, int W, void* x16,
                                            DropoutCtr drop, cudaStream_t st) {
    const size_t total = (size_t)B * (H + 2) * (W + 2);
    images_to_nhwc16_dropout_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(img1, img2, B, H, W,
                                                                                   (__nv_bfloat16*)x16, drop);
    DELORA_CHECK_LAUNCH("images_to_nhwc16_dropout_kernel");
    return 0;
}

extern "C" int delora_stem_weight_prep_bf16(const float* w, int Cin, void* w_stem, void* stream) {
    DELORA_CHECK_ARG(w && w_stem && Cin >= 1 && Cin <= 8, "delora_stem_weight_prep_bf16: bad argument");
    stem_weight_prep_kernel<<<(3 * 64 * 64 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w, Cin, (__nv_bfloat16*)w_stem);
    DELORA_CHECK_LAUNCH("stem_weight_prep_kernel");
    return 0;
}

extern "C" int delora_conv_weight_prep_multi(const void* table, int n_layers, void* stream) {
    DELORA_CHECK_ARG(table && n_layers >= 1 && n_layers <= 65535, "delora_conv_weight_prep_multi: bad argument");
    weight_prep_multi_kernel<<<dim3(2 * num_sms(), (unsigned)n_layers), 256, 0, (cudaStream_t)stream>>>((const long long*)table);
    DELORA_CHECK_LAUNCH("weight_prep_multi_kernel");
    return 0;
}

extern "C" int delora_stem_fprop_bf16(const void* x16, const void* w_stem, void* y, int B, int H, int W, int act,
                                      int out_f16, void* stream) {
    DELORA_CHECK_ARG(x16 && w_stem && y, "delora_stem_fprop_bf16: null pointer");
    DELORA_CHECK_ARG(W % 2 == 0 && W >= 2 && H >= 1 && B >= 1, "delora_stem_fprop_bf16: needs an even image width (got %d)", W);
    DELORA_CHECK_ARG(act >= 0 && act <= 2, "delora_stem_fprop_bf16: act=%d", act);
    StemParams p;
    p.B = B; p.H = H; p.Wout = W / 2; p.segs = (p.Wout + 127) / 128; p.n_jobs = B * H * p.segs; p.act = act;
    p.out_f16 = out_f16 ? 1 : 0;
    CUtensorMap mx, mw;
    int rc = stem_encode_x_map(&mx, x16, B, H, W);
    DELORA_CHECK_ARG(rc == 0, "delora_stem_fprop_bf16: tensor map (x) failed: %d", rc);
    rc = tma_filter(&mw, w_stem, 64, 192, 64, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);     // [3 rows x 64 co][64 k]
    DELORA_CHECK_ARG(rc == 0, "delora_stem_fprop_bf16: tensor map (w) failed: %d", rc);
    const size_t smem = 3 * 8192 + (size_t)kStemStages * 3 * kStemTile + 2 * kAccTileBytes + 256 + 1024;
    const cudaError_t e = smem_opt_in<stem_fprop_tc_kernel>();
    DELORA_CHECK_ARG(e == cudaSuccess, "delora_stem_fprop_bf16: shared-memory opt-in failed: %s", cudaGetErrorString(e));
    const int grid = p.n_jobs < num_sms() ? p.n_jobs : num_sms();
    stem_fprop_tc_kernel<<<grid, kStemThreads, smem, (cudaStream_t)stream>>>(mx, mw, (__nv_bfloat16*)y, p);
    DELORA_CHECK_LAUNCH("stem_fprop_tc_kernel");
    return 0;
}

extern "C" int64_t delora_stem_wgrad_scratch_floats(int B, int H, int W) { return wgrad2_stem_scratch_floats(B, H, W / 2); }

extern "C" int delora_stem_wgrad_bf16(const void* x16, const void* dz, float* dw, float* scratch, int B, int H, int W,
                                      int Cin_true, void* stream) {
    DELORA_CHECK_ARG(x16 && dz && dw && scratch, "delora_stem_wgrad_bf16: null pointer");
    DELORA_CHECK_ARG(W % 2 == 0 && W >= 2 && Cin_true >= 1 && Cin_true <= 8, "delora_stem_wgrad_bf16: bad shape");
    CUtensorMap mx;
    const int rc = stem_encode_x_map(&mx, x16, B, H, W);
    DELORA_CHECK_ARG(rc == 0, "delora_stem_wgrad_bf16: tensor map (x) failed: %d", rc);
    return wgrad2_launch_stem(mx, dz, dw, scratch, B, H, W / 2, Cin_true, (cudaStream_t)stream);
}
