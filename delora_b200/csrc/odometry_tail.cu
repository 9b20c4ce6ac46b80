// The odometry tail (sm_90a): resnet.fc and the heads in fp32 (reference: src/models/model.py:58-84, :103-116), their
// backward, and Adam on the training workspace's fp32 master blob.
//
// Forward:
//   odometry_linear_kernel: y = act(W x + b) for all B rows; one warp per output neuron, a float4 per lane per step.
//     The weight row is read from HBM once per call (batch rows after the first four hit L1), which is what bounds the
//     tail at small B: fc 512 x 1000 (2.05 MB) + heads (0.8 MB two heads / 1.7 MB single MLP).
//   odometry_out_kernel: the last Linear of each head (7 outputs per row), the division of the quaternion by the norm
//     of the WHOLE [B, 4] block (a quirk of the reference, :114) and quaternion -> T, in one CTA.
//   odometry_streams_out_kernel: the streams workspaces' form of it, each quaternion divided by its own row's norm.
// Backward (the training step's stage 4):
//   odometry_out_bwd_kernel (one CTA): grad_T / B -> quaternion -> T backward (quat_to_T_bwd_row, shared with
//     quat_to_T_bwd_kernel) -> backward of the division by the norm of the whole [B, 4] block (all rows coupled) ->
//     d(head outputs) [B, 7]; the last Linear of each head (dW, db) and d(hidden) * act'.  With
//     DELORA_LOSS_IDENTITY_FIT its dL/dT is the identity fit's, 2 (T - I) / (16 B) on the last row, taken from the
//     forward's T, and thread 0 writes that objective (an ordered sum over the 16 entries) to losses[B-1][5].
//   odometry_linear_bwd_kernel: y = act(W x + b) backward for up to two layers that read the same x (the heads'
//     hidden layers: their contributions to dx are summed in a fixed order), dW / db and dx * act'(x) in one launch.
//   odometry_adam_kernel: torch's Adam (fused formula, no weight decay) over the whole blob, float4 per thread; the
//     step count is read from the workspace, so the bias corrections need no host value.
//   DELORA_TRAIN_DROPOUT: the dropout variants of odometry_linear_kernel (the fc launch) and of
//     odometry_linear_bwd_kernel (into dz_fc) draw the fc mask of dropout.cuh, regenerated in the backward.
// Every sum has a fixed order (lane partials in k order, then an xor butterfly; the norm is one thread's loop), there
// are no atomics, so results are bit-identical from run to run and do not depend on B except through the norm.
#include <math.h>
#include <string.h>

#include "odometry.cuh"

namespace delora {

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

static TailLinear tail_args(const Linear& l, const float* w, const float* bias, const float* x, int ldx, float* y, int ldy) {
    TailLinear t;
    t.w = w;
    t.bias = bias;
    t.x = x; t.y = y; t.K = l.K; t.N = l.N; t.ldx = ldx; t.ldy = ldy;
    return t;
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
int run_tail(const Model& m, const TailIO& io, int act, const float* pooled, int B, float* T, cudaStream_t st,
             const float* factor, DropoutCtr drop) {
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

// The model at B = S on the trunk input of t: the trunk into pooled, the tail's hidden layers and
// odometry_streams_out_kernel, which reads io.raw (see the kernel for its other arguments); factor non-NULL selects
// its rescaling instantiation
int streams_forward(const Model& m, const TailIO& io, const TrunkActs& t, const TrunkWeights& w, char* ws, int act,
                    float* pooled, int S, const int32_t* active, int32_t* has_prev, float* T, int32_t* valid,
                    const float* factor, float* factor_out, int32_t* counts, int32_t* n_valid, cudaStream_t st) {
    int rc;
    if ((rc = trunk_forward(m.t, t, ws, w, ws, act, S, pooled, nullptr, st))) return rc;
    TailLinear rot, trans;
    if ((rc = run_tail_hidden(m, io, act, pooled, S, &rot, &trans, st))) return rc;
    const size_t smem = (size_t)S * 7 * sizeof(float);
    const int vec = tail_vec(rot) && tail_vec(trans);
    if (factor)
        odometry_streams_out_kernel<true><<<1, kTailWarps * 32, smem, st>>>(
            rot, trans, S, vec, active, has_prev, T, valid, factor, factor_out, counts, io.raw, n_valid);
    else
        odometry_streams_out_kernel<false><<<1, kTailWarps * 32, smem, st>>>(
            rot, trans, S, vec, active, has_prev, T, valid, factor, factor_out, counts, io.raw, n_valid);
    DELORA_CHECK_LAUNCH(factor ? "odometry_streams_out_kernel<true>" : "odometry_streams_out_kernel");
    return 0;
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
int train_tail_backward(const TrainPlan& tp, char* ws, int act, int B, bool identity, cudaStream_t st,
                        DropoutCtr drop, const int32_t* valid, const int32_t* n_valid) {
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

// Stage 5 of the step: Adam on the master blob (only where *run != 0, run non-NULL), then the bf16 filters from the
// master weights.  more (n > 0): Adam reads tp.grad plus those gradient slices and leaves their sum in tp.grad.
int adam_update(const TrainPlan& tp, char* ws, const delora_odometry_train_params* hp, const int32_t* run,
                cudaStream_t st, const GradSlices* more) {
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


}  // namespace delora
