// The Gauss-Newton information of the ICP objective at T (delora_icp_dense_information, sm_90a).
//
// After the dense search has written every source pixel's kept NN (icp_dense_kernel / icp_dense_pending_kernel with
// IDS) and the finalize its losses row, two launches:
//   icp_info_rows_kernel      one thread per source pixel: the pair's Jacobian rows in the right-perturbation
//                             xi = (rho, phi) of T(xi) = T Exp(xi), their J^T J upper triangles per term (po2pl, pl2pl,
//                             po2po: 63 fp32 FMAs at most), and the warp's sums into its partial row;
//   icp_info_finalize_kernel  one CTA per pair: fixed-order float64 sums of the partial rows, the weighted 6 x 6 H, a
//                             float64 cyclic Jacobi eigen-solve, the information row.
// Each pair's arithmetic reads only that pair's rows, in a fixed order: the row is bit-identical from run to run and
// does not depend on B or on the other pairs.
#include "icp_common.cuh"

namespace delora {

constexpr int kInfoThreads = 128;
constexpr int kInfoFinThreads = 256;
constexpr int kInfoGroups = kInfoFinThreads / kInfoPartial;   // row groups of the finalize's column sums
static_assert(kInfoPartial == 64 && 3 * kInfoSums < kInfoPartial, "three terms and padding: two 32-column halves");
static_assert(DELORA_INFO_ROW == 80, "H 36, eigenvalues 6, eigenvectors 36, M, M'");
constexpr int kRowH = 0, kRowEval = 36, kRowEvec = 42, kRowM = 78, kRowMp = 79;

// acc[off + k] += J_i J_j over the upper triangle i <= j (k in row-major order)
__device__ __forceinline__ void add_jtj(float (&acc)[kInfoPartial], int off, const float (&J)[6]) {
    int k = off;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
        for (int j = i; j < 6; ++j, ++k) acc[k] = fmaf(J[i], J[j], acc[k]);
    }
}

__device__ __forceinline__ void cross3(float ax, float ay, float az, float bx, float by, float bz, float& cx, float& cy,
                                       float& cz) {
    cx = fmaf(ay, bz, -az * by);
    cy = fmaf(az, bx, -ax * bz);
    cz = fmaf(ax, by, -ay * bx);
}

// Per pair (source p, m; matched target normal q = n_t; R the rotation of T, R_k its row k; u = R^T n_t):
//   po2pl               J = [u, p x u]
//   pl2pl, squared      J_k = [0, m x R_k], k = 0..2      (rows of -R [m]x)
//   pl2pl, linear       J = [0, u x m]                      (n_t^T R [m]x)
//   po2po               J_k = [R_k, p x R_k], k = 0..2      (rows of [R, -R [p]x])
// The masks are accumulate_pair's: the ids are -1 for every pair it does not keep.
__global__ void __launch_bounds__(kInfoThreads)
icp_info_rows_kernel(const float4* __restrict__ src_grid, const float4* __restrict__ src_ngrid,
                     const float* __restrict__ T, const float4* __restrict__ tgt_ngrid, int HW, int rows, uint32_t flags,
                     const int* __restrict__ nn_ids, float* __restrict__ partials) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * kInfoThreads + threadIdx.x;
    const int lane = threadIdx.x & 31, warp_row = i >> 5;
    float acc[kInfoPartial];
#pragma unroll
    for (int k = 0; k < kInfoPartial; ++k) acc[k] = 0.0f;
    const int j = i < HW ? __ldg(nn_ids + (size_t)b * HW + i) : -1;
    if (j >= 0) {
        const float4 p = __ldg(src_grid + (size_t)b * HW + i), m = __ldg(src_ngrid + (size_t)b * HW + i);
        const float4 q = __ldg(tgt_ngrid + (size_t)b * HW + j);
        const Rigid r = load_rigid(T + (size_t)b * 12);
        const bool both = (q.w != 0.0f);                   // kept: a normal on both sides, or on neither (po2po)
        const float Rk[3][3] = {{r.r00, r.r01, r.r02}, {r.r10, r.r11, r.r12}, {r.r20, r.r21, r.r22}};
        if (both) {
            const float ux = fmaf(r.r20, q.z, fmaf(r.r10, q.y, r.r00 * q.x));
            const float uy = fmaf(r.r21, q.z, fmaf(r.r11, q.y, r.r01 * q.x));
            const float uz = fmaf(r.r22, q.z, fmaf(r.r12, q.y, r.r02 * q.x));
            if (flags & DELORA_LOSS_PO2PL) {
                float J[6] = {ux, uy, uz, 0.f, 0.f, 0.f};
                cross3(p.x, p.y, p.z, ux, uy, uz, J[3], J[4], J[5]);
                add_jtj(acc, 0, J);
            }
            if (flags & DELORA_LOSS_PL2PL) {
                if (flags & DELORA_NORMAL_LINEAR) {
                    float J[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                    cross3(ux, uy, uz, m.x, m.y, m.z, J[3], J[4], J[5]);
                    add_jtj(acc, kInfoSums, J);
                } else {
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        float J[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                        cross3(m.x, m.y, m.z, Rk[k][0], Rk[k][1], Rk[k][2], J[3], J[4], J[5]);
                        add_jtj(acc, kInfoSums, J);
                    }
                }
            }
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                float J[6] = {Rk[k][0], Rk[k][1], Rk[k][2], 0.f, 0.f, 0.f};
                cross3(p.x, p.y, p.z, Rk[k][0], Rk[k][1], Rk[k][2], J[3], J[4], J[5]);
                add_jtj(acc, 2 * kInfoSums, J);
            }
        }
    }
    // the warp's column sums: two recursive-halving exchanges (warp_column_sums), lane L keeps columns L and 32 + L
    float lo[32], hi[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) { lo[k] = acc[k]; hi[k] = acc[32 + k]; }
    halving_round<16>(lo, lane); halving_round<16>(hi, lane);
    halving_round<8>(lo, lane); halving_round<8>(hi, lane);
    halving_round<4>(lo, lane); halving_round<4>(hi, lane);
    halving_round<2>(lo, lane); halving_round<2>(hi, lane);
    halving_round<1>(lo, lane); halving_round<1>(hi, lane);
    if (warp_row < rows) {
        float* __restrict__ row = partials + ((size_t)b * rows + warp_row) * kInfoPartial;
        row[lane] = lo[0];
        row[32 + lane] = hi[0];
    }
}

// One cyclic Jacobi rotation of (p, q) on the symmetric a and the eigenvector columns v (compile-time indices)
template <int P, int Q>
__device__ __forceinline__ void jacobi_rotate(double (&a)[6][6], double (&v)[6][6]) {
    const double apq = a[P][Q];
    if (apq == 0.0) return;
    const double theta = (a[Q][Q] - a[P][P]) / (2.0 * apq);
    const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(fma(theta, theta, 1.0)));
    const double c = 1.0 / sqrt(fma(t, t, 1.0)), s = t * c;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const double akp = a[k][P], akq = a[k][Q];
        a[k][P] = c * akp - s * akq;
        a[k][Q] = s * akp + c * akq;
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const double apk = a[P][k], aqk = a[Q][k];
        a[P][k] = c * apk - s * aqk;
        a[Q][k] = s * apk + c * aqk;
    }
    a[P][Q] = 0.0;
    a[Q][P] = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const double vkp = v[k][P], vkq = v[k][Q];
        v[k][P] = c * vkp - s * vkq;
        v[k][Q] = s * vkp + c * vkq;
    }
}

template <int P, int Q>
__device__ __forceinline__ void jacobi_row(double (&a)[6][6], double (&v)[6][6]) {
    if constexpr (Q < 6) {
        jacobi_rotate<P, Q>(a, v);
        jacobi_row<P, Q + 1>(a, v);
    } else if constexpr (P + 2 < 6) {
        jacobi_row<P + 1, P + 2>(a, v);
    }
}

// Eigen-decomposition of the symmetric a (destroyed): sweeps of the 15 rotations in a fixed order until the
// off-diagonal part is below 1e-30 of the whole (or 50 sweeps); eigenvalues on the diagonal, eigenvectors in v's columns
__device__ void jacobi6(double (&a)[6][6], double (&v)[6][6]) {
    double total = 0.0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
        for (int j = 0; j < 6; ++j) { v[i][j] = (i == j) ? 1.0 : 0.0; total = fma(a[i][j], a[i][j], total); }
    }
    for (int sweep = 0; sweep < 50; ++sweep) {
        double off = 0.0;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
#pragma unroll
            for (int j = i + 1; j < 6; ++j) off = fma(a[i][j], a[i][j], off);
        }
        if (!(off > 1e-30 * total)) break;
        jacobi_row<0, 1>(a, v);
    }
}

// One CTA per pair.  Thread (column c = tid % 64, group g = tid / 64) sums rows g, g + 4, ... of column c in float64,
// the groups are added in order; thread 0 then weights the three terms into H (float64), solves it and writes the row.
// kScaled (delora_icp_dense_information_scaled): the pair's clouds were divided by factor[b], so H is taken in xi =
// (rho / f, phi); H_m = D H D, D = diag(1/f, 1/f, 1/f, 1, 1, 1), is H in metres and radians.  D is applied to the
// float64 H before it is stored and solved, so the eigen-pairs are H_m's; with f = 1 every product is by 1.0, exact.
template <bool kScaled>
__global__ void __launch_bounds__(kInfoFinThreads)
icp_info_finalize_kernel(const float* __restrict__ partials, int rows, float lambda_po2pl, uint32_t flags,
                         const float* __restrict__ losses, float* __restrict__ info, const float* __restrict__ factor) {
    __shared__ double red[kInfoGroups][kInfoPartial];
    __shared__ double sum[kInfoPartial];
    __shared__ double evec[6][6], eval[6];
    const int b = blockIdx.x;
    const int c = threadIdx.x % kInfoPartial, grp = threadIdx.x / kInfoPartial;
    const float* __restrict__ p = partials + (size_t)b * rows * kInfoPartial + c;
    double s = 0.0;
#pragma unroll 8
    for (int r = grp; r < rows; r += kInfoGroups) s += (double)__ldg(p + (size_t)r * kInfoPartial);
    red[grp][c] = s;
    __syncthreads();
    if (threadIdx.x < kInfoPartial) {
        double tot = red[0][c];
#pragma unroll
        for (int g = 1; g < kInfoGroups; ++g) tot += red[g][c];
        sum[c] = tot;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const float* __restrict__ lrow = losses + (size_t)b * DELORA_LOSS_ROW;
    const float M = lrow[kLossM], Mp = lrow[kLossMp];
    // the objective's means: po2pl and pl2pl over the M (normal, normal) pairs, po2po over the 3 M' coordinates
    const double w_pl = (M > 0.0f && (flags & DELORA_LOSS_PO2PL)) ? 2.0 * (double)lambda_po2pl / (double)M : 0.0;
    const double w_nn = (M > 0.0f && (flags & DELORA_LOSS_PL2PL)) ? 2.0 / (double)M : 0.0;
    const double w_pp = (Mp > 0.0f && (flags & DELORA_LOSS_PO2PO)) ? 2.0 / (3.0 * (double)Mp) : 0.0;
    const double inv_f = kScaled ? 1.0 / (double)factor[b] : 1.0;
    double a[6][6], v[6][6];
    int k = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
        for (int j = i; j < 6; ++j, ++k) {
            double h = w_pl * sum[k] + w_nn * sum[kInfoSums + k] + w_pp * sum[2 * kInfoSums + k];
            if constexpr (kScaled) {
                if (i < 3) h *= inv_f;
                if (j < 3) h *= inv_f;
            }
            a[i][j] = h;
            a[j][i] = h;
        }
    }
    float* __restrict__ o = info + (size_t)b * DELORA_INFO_ROW;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
        for (int j = 0; j < 6; ++j) o[kRowH + 6 * i + j] = (float)a[i][j];
    }
    jacobi6(a, v);
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        eval[i] = a[i][i];
#pragma unroll
        for (int j = 0; j < 6; ++j) evec[i][j] = v[i][j];
    }
    // ascending eigenvalues (stable selection: the lower column first on equal values); each eigenvector's
    // largest-magnitude component (the first of equals) is positive
    int order[6] = {0, 1, 2, 3, 4, 5};
#pragma unroll
    for (int x = 0; x < 6; ++x) {
#pragma unroll
        for (int y = x + 1; y < 6; ++y) {
            if (eval[order[y]] < eval[order[x]]) { const int t = order[x]; order[x] = order[y]; order[y] = t; }
        }
    }
    for (int x = 0; x < 6; ++x) {
        const int col = order[x];
        o[kRowEval + x] = (float)eval[col];
        int big = 0;
        for (int y = 1; y < 6; ++y) if (fabs(evec[y][col]) > fabs(evec[big][col])) big = y;
        const double sign = evec[big][col] < 0.0 ? -1.0 : 1.0;
        for (int y = 0; y < 6; ++y) o[kRowEvec + 6 * x + y] = (float)(sign * evec[y][col]);
    }
    o[kRowM] = M;
    o[kRowMp] = Mp;
}

int launch_icp_information(const float4* src_grid, const float4* src_ngrid, const float* T, const float4* tgt_ngrid, int B, int HW, float lambda_po2pl, uint32_t flags,
                           const float* losses, float* info_scratch, float* info, const float* factor, cudaStream_t st) {
    const IcpInfoLayout L = icp_info_layout(B, HW);
    const int* nn_ids = reinterpret_cast<const int*>(info_scratch + L.ids);
    float* partials = info_scratch + L.partials;
    icp_info_rows_kernel<<<dim3((HW + kInfoThreads - 1) / kInfoThreads, B), kInfoThreads, 0, st>>>(
        src_grid, src_ngrid, T, tgt_ngrid, HW, L.rows, flags, nn_ids, partials);
    DELORA_CHECK_LAUNCH("icp_info_rows_kernel");
    if (factor) {
        icp_info_finalize_kernel<true><<<B, kInfoFinThreads, 0, st>>>(partials, L.rows, lambda_po2pl, flags, losses, info,
                                                                      factor);
        DELORA_CHECK_LAUNCH("icp_info_finalize_kernel<true>");
    } else {
        icp_info_finalize_kernel<false><<<B, kInfoFinThreads, 0, st>>>(partials, L.rows, lambda_po2pl, flags, losses, info,
                                                                       nullptr);
        DELORA_CHECK_LAUNCH("icp_info_finalize_kernel<false>");
    }
    return 0;
}

}  // namespace delora
