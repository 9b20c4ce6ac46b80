// Shared pieces of the two ICP kernels (CSR lists: icp.cu, dense range-image grids: icp_dense.cu).
#pragma once
#include "common.cuh"

namespace delora {

constexpr float kHalfPiF = 1.57079632679489661923f;

// Columns of a partial row (DELORA_ICP_PARTIAL floats: sums over the pairs of one warp).  p, m: source point /
// normal before the transform; r = (s - t).n_t; g_n = d(pl2pl term)/d(n_s) / 2; 3 x 3 blocks are row-major.
constexpr int kColR2 = 0;       // sum r^2
constexpr int kColPl2pl = 1;    // sum of the pl2pl term
constexpr int kColM = 2;        // M: pairs with a normal on both sides
constexpr int kColRn = 3;       // 3: sum r n_t
constexpr int kColRnP = 6;      // 9: sum (r n_t) p^T
constexpr int kColGnM = 15;     // 9: sum g_n m^T
constexpr int kColPo2po = 24;   // the po2po block, last: a kernel without po2po reduces only the columns before it
constexpr int kColD2 = 24;      // sum |s - t|^2
constexpr int kColMp = 25;      // M': pairs with a normal on neither side
constexpr int kColD = 26;       // 3: sum (s - t)
constexpr int kColDP = 29;      // 9: sum (s - t) p^T
constexpr int kIcpAcc = 38;     // accumulated columns; the rest of the row is padding
static_assert(kColGnM + 9 == kColPo2po && kColDP + 9 == kIcpAcc, "the po2po block is the last one");
static_assert(kIcpAcc <= DELORA_ICP_PARTIAL, "the accumulators fit a partial row");

// Columns of a `losses` row (DELORA_LOSS_ROW floats)
constexpr int kLossPo2po = 0, kLossPo2pl = 1, kLossPl2pl = 2, kLossM = 3, kLossMp = 4;
static_assert(kLossMp < DELORA_LOSS_ROW, "the loss columns fit a losses row");

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

// acc[c + 3 i + j] = a_i v_j: the outer product (ax, ay, az) v^T into a 3 x 3 block of columns
__device__ __forceinline__ void acc_outer(float (&acc)[kIcpAcc], int c, float ax, float ay, float az, const float4 v) {
    acc[c + 0] = ax * v.x; acc[c + 1] = ax * v.y; acc[c + 2] = ax * v.z;
    acc[c + 3] = ay * v.x; acc[c + 4] = ay * v.y; acc[c + 5] = ay * v.z;
    acc[c + 6] = az * v.x; acc[c + 7] = az * v.y; acc[c + 8] = az * v.z;
}

// The columns of one (source, target) pair.  (sx..), (nsx..): source point / normal after the transform; t, q: matched
// target point and (normal, has-normal flag).  Masks: src/losses/icp_losses.py:48-52, :110-121, :83-99.
__device__ __forceinline__ void accumulate_pair(uint32_t flags, const float4 p, const float4 m, float sx, float sy,
                                                float sz, float nsx, float nsy, float nsz, const float4 t,
                                                const float4 q, float (&acc)[kIcpAcc], float4& pd, float4& nd) {
    const bool src_has = (nsx != 0.0f) | (nsy != 0.0f) | (nsz != 0.0f);
    const bool tgt_has = q.w != 0.0f;
    const float dx = sx - t.x, dy = sy - t.y, dz = sz - t.z;
    if (src_has && tgt_has) {
        acc[kColM] = 1.0f;
        if (flags & DELORA_LOSS_PO2PL) {
            const float r = fmaf(dz, q.z, fmaf(dy, q.y, dx * q.x));                      // icp_losses.py:197-199
            acc[kColR2] = r * r;
            const float gx = r * q.x, gy = r * q.y, gz = r * q.z;
            acc[kColRn + 0] = gx; acc[kColRn + 1] = gy; acc[kColRn + 2] = gz;
            acc_outer(acc, kColRnP, gx, gy, gz, p);
            pd = make_float4(gx, gy, gz, 1.0f);
        }
        if (flags & DELORA_LOSS_PL2PL) {
            float hx, hy, hz;
            if (flags & DELORA_NORMAL_LINEAR) {                                          // :226-231
                const float om = 1.0f - fmaf(nsz, q.z, fmaf(nsy, q.y, nsx * q.x));
                acc[kColPl2pl] = om * om;
                hx = -om * q.x; hy = -om * q.y; hz = -om * q.z;
            } else {                                                                     // :232-238
                hx = nsx - q.x; hy = nsy - q.y; hz = nsz - q.z;
                acc[kColPl2pl] = fmaf(hz, hz, fmaf(hy, hy, hx * hx));
            }
            acc_outer(acc, kColGnM, hx, hy, hz, m);
            nd = make_float4(hx, hy, hz, 1.0f);
            pd.w = 1.0f;
        }
    } else if ((flags & DELORA_LOSS_PO2PO) && !src_has && !tgt_has) {                    // :168-179
        acc[kColD2] = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
        acc[kColMp] = 1.0f;
        acc[kColD + 0] = dx; acc[kColD + 1] = dy; acc[kColD + 2] = dz;
        acc_outer(acc, kColDP, dx, dy, dz, p);
        pd = make_float4(dx, dy, dz, 2.0f);
    }
}

// The target id of a pair accumulate_pair keeps (a normal on both sides, or with po2po on neither), -1 otherwise.
// (nsx..): the rotated source normal; j: the NN of a paired lane in the target normals tn.
__device__ __forceinline__ int kept_nn(bool paired, bool po2po, float nsx, float nsy, float nsz,
                                       const float4* __restrict__ tn, int j) {
    if (!paired) return -1;
    const bool src_has = (nsx != 0.0f) | (nsy != 0.0f) | (nsz != 0.0f);
    const bool tgt_has = __ldg(tn + j).w != 0.0f;
    return (src_has == tgt_has && (src_has || po2po)) ? j : -1;
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

// The end of every ICP kernel.  The lane's pair (when `paired`: target tg[j], tn[j]) is accumulated, and the warp's
// column sums are written to (ADD = false) or added to (ADD = true, the dense path's block search adding to the row
// the window search wrote) partial row `warp_row` of pair b; lane k keeps column k and 32 + k.  N: the live
// columns, kIcpAcc or kColPo2po; below kIcpAcc the po2po flag is masked off, so the columns from N on stay zero.
template <int N, bool ADD>
__device__ __forceinline__ void accumulate_warp_row(bool paired, uint32_t flags, const float4 p, const float4 m,
                                                    float sx, float sy, float sz, float nsx, float nsy, float nsz,
                                                    const float4* __restrict__ tg, const float4* __restrict__ tn,
                                                    int j, float4* __restrict__ point_dir, float4* __restrict__ normal_dir, float* __restrict__ partial_rows,
                                                    int b, int rows_per_pair, int warp_row) {
    static_assert(N == kIcpAcc || N == kColPo2po, "all columns, or all but the po2po block");
    float acc[kIcpAcc];
#pragma unroll
    for (int k = 0; k < kIcpAcc; ++k) acc[k] = 0.0f;
    float4 pd = make_float4(0.f, 0.f, 0.f, 0.f), nd = make_float4(0.f, 0.f, 0.f, 0.f);
    if (paired)
        accumulate_pair(N == kIcpAcc ? flags : (flags & ~DELORA_LOSS_PO2PO), p, m, sx, sy, sz, nsx, nsy, nsz,
                        __ldg(tg + j), __ldg(tn + j), acc, pd, nd);
    if (point_dir) *point_dir = pd;
    if (normal_dir) *normal_dir = nd;
    if (warp_row >= rows_per_pair) return;
    float* __restrict__ row = partial_rows + ((size_t)b * rows_per_pair + warp_row) * DELORA_ICP_PARTIAL;
    const int lane = threadIdx.x & 31;
    float keep0, keep1;
    warp_column_sums<N>(acc, keep0, keep1);
    if (ADD) {
        row[lane] += keep0;
        if (lane < DELORA_ICP_PARTIAL - 32) row[32 + lane] += keep1;
    } else {
        row[lane] = keep0;
        if (lane < DELORA_ICP_PARTIAL - 32) row[32 + lane] = keep1;
    }
}

// Range extents of the dense path's target grids, per pair (target_extents_kernel):
//   blk[nbh * nbw]       [min, max] of |t| per 4 x 16-cell block (the block search's pyramid)
//   row_pre[H], row_suf[H]  [min, max] of |t| over the valid cells of the pixel rows <= k / >= k
// Every extent is widened by a relative 1e-6 so that bounds built on it stay conservative against the fp32 norm
// rounding; an empty block or row set has max < 0.
struct TargetExtents {
    float2* blk;
    float2* row_pre;
    float2* row_suf;
    int* counter;          // per pair: CTAs of the pre-pass that have finished (0 when idle)
};

// Work list of the dense path's block search (icp_dense_pending_kernel).  An ITEM is a warp of icp_dense_kernel that
// gave up on some of its lanes after `max_strips` window-growing steps; an ENTRY is one such lane.
struct PendingList {
    int* counters;          // [0] items, [1] CTAs of the second kernel that have finished, [2] entries; 0 when idle
    int4* items;            // (pair, warp in pair, mask of unfinished lanes, first entry)
    int* item_done;         // entries of the item already searched (0 when idle)
    float4* entries;        // (m1, m2, bits(j1), bits(item * 32 + lane)) of the window search so far
    int* result;            // per entry: pixel id of the nearest neighbour
};

// The scratch buffer of both ICP paths (delora_icp_scratch_floats floats), as element offsets in floats.  Every
// capacity follows from (B, src_stride) alone; the dense path uses src_stride = H * W.  Sections are ordered by the
// alignment they need (16-byte int4 / float4, then 8-byte float2, then 4-byte) and every size is a multiple of the
// next section's alignment, so no section needs padding.  The buffer is zeroed once; the kernels leave every counter
// at zero again.
struct IcpLayout {
    int rows;                  // partial rows per pair: one per warp of 32 source points
    int64_t blk_per_pair;      // range-pyramid blocks per pair
    int64_t partials;          // [B, rows, DELORA_ICP_PARTIAL] per-warp partial rows
    int64_t colsum;            // [B, DELORA_ICP_PARTIAL] column sums
    int64_t items;             // int4 [B * rows]: work-list items (at most one per warp)
    int64_t entries;           // float4 [B * rows * 32]: work-list entries (at most one per source point)
    int64_t blk;               // float2 [B, blk_per_pair]: range pyramid
    int64_t row_pre, row_suf;  // float2 [B, src_stride] each: row prefix / suffix extents (H <= src_stride)
    int64_t result;            // int [B * rows * 32]: per entry
    int64_t item_done;         // int [B * rows]: per item
    int64_t counter;           // int [B + 2]: finalize counters, one per pair
    int64_t ext_counter;       // int [B]: extents counters, one per pair
    int64_t pend_counters;     // int [8]: work-list counters
    int64_t total;
};
static_assert(sizeof(int4) == 16 && sizeof(float4) == 16 && sizeof(float2) == 8, "element sizes the layout assumes");
static_assert(DELORA_ICP_PARTIAL % 4 == 0, "the partial rows and column sums keep the int4 / float4 sections 16-byte aligned");

inline IcpLayout icp_layout(int B, int src_stride) {
    IcpLayout L;
    const int64_t b = B, s = src_stride;
    L.rows = (int)((s + 31) / 32);
    L.blk_per_pair = s / 16 + 4096;
    int64_t off = 0;
    auto take = [&off](int64_t n) { const int64_t o = off; off += n; return o; };
    L.partials = take(b * L.rows * DELORA_ICP_PARTIAL);
    L.colsum = take(b * DELORA_ICP_PARTIAL);
    L.items = take(4 * b * L.rows);
    L.entries = take(4 * b * L.rows * 32);
    L.blk = take(2 * b * L.blk_per_pair);
    L.row_pre = take(2 * b * s);
    L.row_suf = take(2 * b * s);
    L.result = take(b * L.rows * 32);
    L.item_done = take(b * L.rows);
    L.counter = take(b + 2);
    L.ext_counter = take(b);
    L.pend_counters = take(8);
    L.total = off;
    return L;
}

// device views of a scratch buffer laid out by icp_layout
struct IcpScratch {
    float* rows;
    float* colsum;
    int* counter;
    TargetExtents ext;
    PendingList pend;
};

inline IcpScratch icp_scratch(float* base, const IcpLayout& L) {
    IcpScratch s;
    s.rows = base + L.partials;
    s.colsum = base + L.colsum;
    s.counter = reinterpret_cast<int*>(base + L.counter);
    s.ext.blk = reinterpret_cast<float2*>(base + L.blk);
    s.ext.row_pre = reinterpret_cast<float2*>(base + L.row_pre);
    s.ext.row_suf = reinterpret_cast<float2*>(base + L.row_suf);
    s.ext.counter = reinterpret_cast<int*>(base + L.ext_counter);
    s.pend.counters = reinterpret_cast<int*>(base + L.pend_counters);
    s.pend.items = reinterpret_cast<int4*>(base + L.items);
    s.pend.item_done = reinterpret_cast<int*>(base + L.item_done);
    s.pend.entries = reinterpret_cast<float4*>(base + L.entries);
    s.pend.result = reinterpret_cast<int*>(base + L.result);
    return s;
}

// The caller buffer of delora_icp_dense_information (delora_icp_information_scratch_floats floats), as element offsets:
// the NN id of every source pixel (int32 [B, HW], first: the header documents it), then the per-warp partial rows of
// the information pass (fp32 [B, rows, kInfoPartial]).  Every section is written before it is read, on every call.
constexpr int kInfoSums = 21;                       // upper triangle of a symmetric 6 x 6, row by row
constexpr int kInfoPartial = 64;                    // po2pl, pl2pl, po2po sums (3 x 21), one column of padding
struct IcpInfoLayout {
    int rows;
    int64_t ids, partials, total;
};

inline IcpInfoLayout icp_info_layout(int B, int HW) {
    IcpInfoLayout L;
    L.rows = (HW + 31) / 32;
    L.ids = 0;
    L.partials = (int64_t)B * HW;
    L.total = L.partials + (int64_t)B * L.rows * kInfoPartial;
    return L;
}

// icp_info.cu: the information pass after the dense search (which wrote the NN ids) and the finalize (losses); factor
// [B] or NULL: H in metres for pairs whose clouds were divided by factor[b] (delora_icp_dense_information_scaled)
int launch_icp_information(const float4* src_grid, const float4* src_ngrid, const float* T, const float4* tgt_ngrid, int B, int HW, float lambda_po2pl, uint32_t flags,
                           const float* losses, float* info_scratch, float* info, const float* factor, cudaStream_t st);

int launch_icp_finalize(const IcpScratch& sc, int B, int rows, float lambda_po2pl, float* losses, float* grad_T,
                        cudaStream_t st);

}  // namespace delora
