// The dropout masks of the training step (DELORA_TRAIN_DROPOUT; the contract is documented in include/delora_b200.h):
// a counter-based generator, so a mask is a pure function of (seed, step, tensor id, element index).  The forward and
// the backward regenerate the same masks instead of storing them, a CUDA-graph replay draws fresh masks because the
// step count lives on the device, and a resumed run draws the masks the uninterrupted run would have drawn.
#pragma once
#include <stdint.h>

#include "common.cuh"

namespace delora {

// Philox4x32-10 (Salmon et al., SC'11): 10 rounds of two 32x32 -> 64-bit products, with the key bumped by the Weyl
// constants between rounds.  The same arithmetic as curand's philox4x32_10, usable on the host too.
struct Philox4 {
    uint32_t x, y, z, w;
};

__host__ __device__ __forceinline__ Philox4 philox4x32_10(Philox4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c.x, p1 = (uint64_t)0xCD9E8D57u * c.z;
        c = Philox4{(uint32_t)(p1 >> 32) ^ c.y ^ k0, (uint32_t)p1, (uint32_t)(p0 >> 32) ^ c.w ^ k1, (uint32_t)p0};
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c;
}

// p = 0.2: keep iff u < 0.8f with u = (word >> 8) * 2^-24, i.e. (word >> 8) < 13421773 (0.8f is exactly
// 13421773 * 2^-24); a kept value is multiplied by 1/(1-p) = 1.25f, exact in fp32.
constexpr uint32_t kDropKeepBelow = 13421773u;
constexpr float kDropScale = 1.25f;

// Tensor ids of the three dropouts (the element index of each is per pair, independent of B and max_batch)
constexpr int kDropInput = 0;          // ((b * 8 + c) * H + h) * W + w over cat(image_1, image_2)
constexpr int kDropStage3 = 1;         // b * C3 + c, C3 = layer3's channel count
constexpr int kDropFc = 2;             // b * resnet_outputs + j

// The four words of counter (i >> 2, t, step) under key seed: elements 4q .. 4q+3 of tensor t
__host__ __device__ __forceinline__ Philox4 dropout_words(uint64_t seed, uint64_t step, int t, uint64_t q) {
    return philox4x32_10(Philox4{(uint32_t)q, (uint32_t)t, (uint32_t)step, (uint32_t)(step >> 32)}, (uint32_t)seed,
                         (uint32_t)(seed >> 32));
}

__host__ __device__ __forceinline__ bool dropout_word_keeps(uint32_t word) { return (word >> 8) < kDropKeepBelow; }

__host__ __device__ __forceinline__ uint32_t philox_word(const Philox4& r, int k) {
    return k == 0 ? r.x : k == 1 ? r.y : k == 2 ? r.z : r.w;
}

// Whether element i of tensor t is kept at (seed, step)
__host__ __device__ __forceinline__ bool dropout_keep(uint64_t seed, uint64_t step, int t, uint64_t i) {
    return dropout_word_keeps(philox_word(dropout_words(seed, step, t, i >> 2), (int)(i & 3)));
}

// Where a training-step kernel finds its masks: the workspace's counter slot (ctr[0] Adam's step count, ctr[2] the
// seed).  The forward runs before odometry_out_bwd_kernel advances the count, the backward after it, so bwd = 1 reads
// the count the step started with.  ctr == NULL: no dropout.
struct DropoutCtr {
    const long long* ctr;
    int bwd;
};

__device__ __forceinline__ void dropout_seed_step(const DropoutCtr& d, uint64_t& seed, uint64_t& step) {
    seed = (uint64_t)d.ctr[2];
    step = (uint64_t)(d.ctr[0] - d.bwd);
}

// The masked trunk-input conversions (conv_stem.cu, conv_tc.cu): delora_images_to_nhwc16_bf16 /
// delora_images_to_nhwc_bf16 with every element of cat(image_1, image_2) multiplied by keep * 1.25f in fp32 before the
// bf16 rounding.  Arguments are not checked.
int launch_images_to_nhwc16_dropout(const float* img1, const float* img2, int B, int H, int W, void* x16,
                                    DropoutCtr drop, cudaStream_t st);
int launch_images_to_nhwc_dropout(const float* img1, const float* img2, int B, int H, int W, int Cpad, void* x,
                                  DropoutCtr drop, cudaStream_t st);

}  // namespace delora
