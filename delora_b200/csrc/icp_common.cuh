// Shared pieces of the two ICP kernels (CSR lists: icp.cu, dense range-image grids: icp_dense.cu).
#pragma once
#include "common.cuh"

namespace delora {

constexpr float kHalfPiF = 1.57079632679489661923f;
constexpr int kIcpAcc = 38;

// Running nearest neighbour.  Ranking is EXACT in float64 (what cKDTree measures), but float64 is
// only touched when two candidates are closer than 1e-5 relative in fp32 (the fp32 squared
// distance of exact fp32 inputs is good to ~3e-7 relative): a candidate clearly below the best
// replaces it, one clearly above is dropped, and only the ambiguous band is re-measured.
struct NNBest {
    float d2f;         // fp32 squared distance of the current best
    float bx, by, bz;  // its coordinates (to re-measure in fp64 on demand)
    int pos;           // position of the best target in its array
    int tag;           // tie-break key (target .w bits)
};

constexpr float kNNBand = 1.0e-5f;

__device__ __forceinline__ void nn_init(NNBest& b) {
    b.d2f = 3.0e38f; b.bx = 0.f; b.by = 0.f; b.bz = 0.f; b.pos = -1; b.tag = 0x7fffffff;
}

__device__ __forceinline__ double nn_d2_exact(float sx, float sy, float sz, float tx, float ty, float tz) {
    const double ex = (double)sx - (double)tx, ey = (double)sy - (double)ty, ez = (double)sz - (double)tz;
    return ex * ex + ey * ey + ez * ez;
}

__device__ __forceinline__ void nn_eval(const float4 t, int j, float sx, float sy, float sz, NNBest& best) {
    const float dx = sx - t.x, dy = sy - t.y, dz = sz - t.z;
    const float d2f = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
    if (d2f <= best.d2f * (1.0f + kNNBand)) {
        bool take = d2f < best.d2f * (1.0f - kNNBand);
        if (!take) {                                   // ambiguous band: exact float64 order, lowest tag on ties
            const double dn = nn_d2_exact(sx, sy, sz, t.x, t.y, t.z);
            const double db = nn_d2_exact(sx, sy, sz, best.bx, best.by, best.bz);
            const int tag = __float_as_int(t.w);
            take = dn < db || (dn == db && tag < best.tag);
        }
        if (take) {
            best.d2f = d2f; best.bx = t.x; best.by = t.y; best.bz = t.z; best.pos = j;
            best.tag = __float_as_int(t.w);
        }
    }
}

// upper bound (fp32) of the distance to the current best, for the exactness guard
__device__ __forceinline__ float nn_best_dist_ub(const NNBest& best) {
    return sqrtf(best.d2f) * 1.00001f;
}

struct Rigid {
    float r00, r01, r02, tx, r10, r11, r12, ty, r20, r21, r22, tz;
};

__device__ __forceinline__ Rigid load_rigid(const float* __restrict__ t) {
    Rigid r;
    r.r00 = __ldg(t + 0); r.r01 = __ldg(t + 1); r.r02 = __ldg(t + 2); r.tx = __ldg(t + 3);
    r.r10 = __ldg(t + 4); r.r11 = __ldg(t + 5); r.r12 = __ldg(t + 6); r.ty = __ldg(t + 7);
    r.r20 = __ldg(t + 8); r.r21 = __ldg(t + 9); r.r22 = __ldg(t + 10); r.tz = __ldg(t + 11);
    return r;
}

// s = R p + t (R p first, + t afterwards: src/deploy/deployer.py:185-188), n_s = R m (:181-182)
__device__ __forceinline__ void apply_rigid(const Rigid& r, const float4 p, const float4 m, float& sx, float& sy,
                                            float& sz, float& nsx, float& nsy, float& nsz) {
    sx = fmaf(r.r02, p.z, fmaf(r.r01, p.y, r.r00 * p.x)) + r.tx;
    sy = fmaf(r.r12, p.z, fmaf(r.r11, p.y, r.r10 * p.x)) + r.ty;
    sz = fmaf(r.r22, p.z, fmaf(r.r21, p.y, r.r20 * p.x)) + r.tz;
    nsx = fmaf(r.r02, m.z, fmaf(r.r01, m.y, r.r00 * m.x));
    nsy = fmaf(r.r12, m.z, fmaf(r.r11, m.y, r.r10 * m.x));
    nsz = fmaf(r.r22, m.z, fmaf(r.r21, m.y, r.r20 * m.x));
}

// Per-pair accumulators (DELORA_ICP_PARTIAL = 40 floats per partial row):
//  0 sum r^2            1 sum pl2pl term      2 M
//  3..5   sum r*n_t                 6..14  sum (r*n_t) p^T
//  15..23 sum g_n m^T               24 sum |s-t|^2 (po2po)   25 M'
//  26..28 sum (s-t)                 29..37 sum (s-t) p^T      38,39 pad
// p, m: source point / normal before the transform; (sx..), (nsx..): after; t, q: matched target
// point and (normal, has-normal flag).  Masks: src/losses/icp_losses.py:48-52, :110-121, :83-99.
__device__ __forceinline__ void accumulate_pair(uint32_t flags, const float4 p, const float4 m, float sx, float sy,
                                                float sz, float nsx, float nsy, float nsz, const float4 t,
                                                const float4 q, float (&acc)[kIcpAcc], float4& pd, float4& nd) {
    const bool src_has = (nsx != 0.0f) | (nsy != 0.0f) | (nsz != 0.0f);
    const bool tgt_has = q.w != 0.0f;
    const float dx = sx - t.x, dy = sy - t.y, dz = sz - t.z;
    if (src_has && tgt_has) {
        acc[2] = 1.0f;
        if (flags & DELORA_LOSS_PO2PL) {
            const float r = fmaf(dz, q.z, fmaf(dy, q.y, dx * q.x));                      // icp_losses.py:197-199
            acc[0] = r * r;
            const float gx = r * q.x, gy = r * q.y, gz = r * q.z;
            acc[3] = gx; acc[4] = gy; acc[5] = gz;
            acc[6] = gx * p.x; acc[7] = gx * p.y; acc[8] = gx * p.z;
            acc[9] = gy * p.x; acc[10] = gy * p.y; acc[11] = gy * p.z;
            acc[12] = gz * p.x; acc[13] = gz * p.y; acc[14] = gz * p.z;
            pd = make_float4(gx, gy, gz, 1.0f);
        }
        if (flags & DELORA_LOSS_PL2PL) {
            float hx, hy, hz;
            if (flags & DELORA_NORMAL_LINEAR) {                                          // :226-231
                const float om = 1.0f - fmaf(nsz, q.z, fmaf(nsy, q.y, nsx * q.x));
                acc[1] = om * om;
                hx = -om * q.x; hy = -om * q.y; hz = -om * q.z;
            } else {                                                                     // :232-238
                hx = nsx - q.x; hy = nsy - q.y; hz = nsz - q.z;
                acc[1] = fmaf(hz, hz, fmaf(hy, hy, hx * hx));
            }
            acc[15] = hx * m.x; acc[16] = hx * m.y; acc[17] = hx * m.z;
            acc[18] = hy * m.x; acc[19] = hy * m.y; acc[20] = hy * m.z;
            acc[21] = hz * m.x; acc[22] = hz * m.y; acc[23] = hz * m.z;
            nd = make_float4(hx, hy, hz, 1.0f);
            pd.w = 1.0f;
        }
    } else if ((flags & DELORA_LOSS_PO2PO) && !src_has && !tgt_has) {                    // :168-179
        acc[24] = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
        acc[25] = 1.0f;
        acc[26] = dx; acc[27] = dy; acc[28] = dz;
        acc[29] = dx * p.x; acc[30] = dx * p.y; acc[31] = dx * p.z;
        acc[32] = dy * p.x; acc[33] = dy * p.y; acc[34] = dy * p.z;
        acc[35] = dz * p.x; acc[36] = dz * p.y; acc[37] = dz * p.z;
        pd = make_float4(dx, dy, dz, 2.0f);
    }
}

// Sum of `acc[k]` over the 32 lanes for every k < N, lane k keeping column k (keep0) and column 32 + k (keep1).
// Columns 0..31 go through a recursive-halving exchange: in the round with offset o the lanes whose bit o is clear
// keep the lower half of the live columns and receive the partner's contribution to them (31 shuffles for 32
// columns instead of 32 x 5 for per-column shuffle trees); after the five rounds lane L holds the total of column L.
// The (few) columns >= 32 use plain shuffle trees.
// Every round is its own instantiation so that all indices into v[] are compile-time constants: a `for (o = 16; o > 0;
// o >>= 1)` loop is not unrolled by nvcc, and its inner loop then indexes v[] at run time, i.e. in local memory.
template <int O>
__device__ __forceinline__ void halving_round(float (&v)[32], int lane) {
    const bool upper = (lane & O) != 0;
#pragma unroll
    for (int k = 0; k < O; ++k) {
        const float lo = v[k], hi = v[k + O];
        const float send = upper ? lo : hi;
        const float keep = upper ? hi : lo;
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, O);
    }
}

template <int N>
__device__ __forceinline__ void warp_column_sums(const float (&acc)[kIcpAcc], float& keep0, float& keep1) {
    const int lane = threadIdx.x & 31;
    float v[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) v[k] = (k < N) ? acc[k] : 0.0f;
    halving_round<16>(v, lane);
    halving_round<8>(v, lane);
    halving_round<4>(v, lane);
    halving_round<2>(v, lane);
    halving_round<1>(v, lane);
    keep0 = v[0];
    keep1 = 0.0f;
#pragma unroll
    for (int k = 32; k < N; ++k) {
        const float s = warp_sum(acc[k]);
        if (lane == k - 32) keep1 = s;
    }
}

// one partial row per warp, lane k writes column k (and k+32)
template <int N = kIcpAcc>   // columns >= N are known to be zero (e.g. the po2po block when it is off)
__device__ __forceinline__ void write_warp_partials(const float (&acc)[kIcpAcc], float* __restrict__ row) {
    const int lane = threadIdx.x & 31;
    float keep0, keep1;
    warp_column_sums<N>(acc, keep0, keep1);
    row[lane] = keep0;
    if (lane < DELORA_ICP_PARTIAL - 32) row[32 + lane] = keep1;
}

// same reduction, ADDED to a row that already holds the sums of the other lanes (second kernel of the dense path)
template <int N = kIcpAcc>
__device__ __forceinline__ void add_warp_partials(const float (&acc)[kIcpAcc], float* __restrict__ row) {
    const int lane = threadIdx.x & 31;
    float keep0, keep1;
    warp_column_sums<N>(acc, keep0, keep1);
    row[lane] += keep0;
    if (lane < DELORA_ICP_PARTIAL - 32) row[32 + lane] += keep1;
}

// scratch layout (floats): [B * rows * 40 partial rows][B * 40 column sums][B int32 counters]
struct IcpScratch {
    float* rows;
    float* colsum;
    int* counter;
};
inline IcpScratch icp_scratch(float* base, int B, int rows) {
    IcpScratch s;
    s.rows = base;
    s.colsum = base + (size_t)B * rows * DELORA_ICP_PARTIAL;
    s.counter = reinterpret_cast<int*>(s.colsum + (size_t)B * DELORA_ICP_PARTIAL);
    return s;
}

int launch_icp_finalize(float* scratch, int B, int rows, float lambda_po2pl, uint32_t flags, float* losses,
                        float* grad_T, cudaStream_t st);

}  // namespace delora
