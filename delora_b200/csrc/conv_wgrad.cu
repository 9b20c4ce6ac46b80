// Encoder weight gradient, second-generation kernel (round 2).
//
//   dW[co][tap][ci] = sum over output pixels of dZ[pix][co] * X[pix * stride + tap][ci]
// (autograd's backward of the reference's nn.Conv2d layers w.r.t. their weights, src/models/resnet_modified.py:40,
// :126-134).  GEMM with K = PIXELS, both operands pixel-major NHWC tiles (MN-major for the tensor core).
//
// The first-generation kernel (conv_tc.cu) streams a dZ tile AND one X tile per filter tap through shared memory.  Here
// a K-row (one image row segment of NS pixels) is loaded ONCE and the taps are formed in the MMA descriptors: tap q of
// a row = the same X tile starting q pixels (q * 128 B) later (MN-major operands may start at any 128-byte offset).
// The GEMM is cut into 64 x 64 fp32 accumulators ("units", each one wgmma chain: A = 64 rows of one operand, B = 64
// rows of the other, K = pixels):
//   mode 0 (Cout % 128 == 0): A = 64 output channels of dZ, B = the X tile of tap q; filter row r per CTA, 2 x 3 units;
//   mode 1 (Cout == 64):      A = the X tile of tap (r, q), B = the 64 output channels of dZ; all 9 taps in one CTA;
//   mode 2 (stem):            A = the X window of filter row r (conv_stem.cu), B = dZ; 3 units;
//   strided layers read X through an element-strided tensor map (even / odd columns as separate tiles).
// The unit list ("plan") is built on the host; three consumer warpgroups take every third unit.  Split-K over pixel
// rows: grid = tiles x splits <= #SMs, fp32 partials, a coalesced fixed-order reduction (deterministic) into the torch
// layout.  Warp roles: 0..11 MMA + epilogue (three warpgroups), 12 TMA producer.
#include <string.h>
#include "conv_internal.cuh"

namespace delora {

// dynamic shared memory of one CTA: stages + accumulator hand-off tiles + barriers, under the 227 KB opt-in limit
constexpr int kWgSmemBudget = 225 * 1024;
constexpr int kWgConsumers = 3;                          // consumer warpgroups
constexpr int kWgThreads = kWgConsumers * 128 + 32;
constexpr int kWgSlots = 3;                              // units per warpgroup (3 x 32 accumulator registers)
constexpr int kWgMaxLoads = 6, kWgMaxUnits = kWgConsumers * kWgSlots, kWgMaxStages = 8;

struct WgLoad { int is_x, ch_blk, dw, dh, smem_off, bytes; };
// a_off / b_off: byte offsets of the two operands in a stage; tap: filter tap (mode 0: column q, mode 1: r * 3 + q,
// mode 2: filter row); co_base / ci_base: first output / input channel of the unit inside the CTA's tile
struct WgUnit { int a_off, b_off, tap, co_base, ci_base; };

struct Wg2Params {
    int B, Hout, Wout, Cin, Cout, taps;
    int sh, sw;
    int NS, segs, k_rows;
    int mode;
    int co_tiles, ci_tiles, n_tiles, splits;
    int ci_per_tile, co_per_tile;
    int stage_bytes, stages, stage_tx;
    int n_loads, n_units;
    WgLoad loads[kWgMaxLoads];
    WgUnit units[kWgMaxUnits];
};

__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad2_tc_kernel(const __grid_constant__ CUtensorMap map_dz, const __grid_constant__ CUtensorMap map_x,
                      float* __restrict__ partial, const __grid_constant__ Wg2Params p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = DELORA_ALIGNED_SMEM(smem_raw);
    float* acc_tiles = reinterpret_cast<float*>(smem + p.stages * p.stage_bytes);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(acc_tiles) + kWgConsumers * kAccTileBytes);
    uint64_t* empty_bar = full_bar + kWgMaxStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x % p.n_tiles, split = blockIdx.x / p.n_tiles;
    const int ci_t = tile % p.ci_tiles, co_t = (tile / p.ci_tiles) % p.co_tiles, r = tile / (p.ci_tiles * p.co_tiles);
    const int co0 = co_t * p.co_per_tile, ci0 = ci_t * p.ci_per_tile;
    const int per = (p.k_rows + p.splits - 1) / p.splits;
    const int k_begin = split * per, k_end = min(p.k_rows, k_begin + per);
    const int n_iter = max(0, k_end - k_begin);
    const int S = p.stages;

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) { mbar_init(full_bar + s, 1); mbar_init(empty_bar + s, 4 * kWgConsumers); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 4 * kWgConsumers) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            tma_prefetch_desc(&map_dz);
            tma_prefetch_desc(&map_x);
            uint32_t s = 0, ph = 0;
            for (int it = 0; it < n_iter; ++it) {
                int kt = k_begin + it;
                const int seg = kt % p.segs; kt /= p.segs;
                const int h = kt % p.Hout;
                const int b = kt / p.Hout;
                const int w0 = seg * p.NS;
                mbar_wait(empty_bar + s, ph ^ 1);
                mbar_expect_tx(full_bar + s, (uint32_t)p.stage_tx);
                uint8_t* st = smem + s * p.stage_bytes;
                for (int l = 0; l < p.n_loads; ++l) {
                    const WgLoad& ld = p.loads[l];
                    if (ld.is_x)
                        tma_load_4d(st + ld.smem_off, &map_x, full_bar + s, ci0 + 64 * ld.ch_blk, w0 * p.sw + ld.dw,
                                    h * p.sh + ld.dh + (p.mode == 0 ? r : 0), b);
                    else
                        tma_load_4d(st + ld.smem_off, &map_dz, full_bar + s, co0 + 64 * ld.ch_blk, w0 + 1, h + 1, b);
                }
                if (++s == (uint32_t)S) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    // ===================== MMA: warpgroup wg runs units wg, wg + 3, wg + 6 =====================
    const int wg = warp >> 2;
    const int ksteps = p.NS >> 4;                          // 16 pixels = 16 rows of 128 B = 2 KB per wgmma
    float acc[kWgSlots][32];
#pragma unroll
    for (int u = 0; u < kWgSlots; ++u)
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[u][j] = 0.0f;
    uint32_t a_off[kWgSlots], b_off[kWgSlots];
#pragma unroll
    for (int u = 0; u < kWgSlots; ++u) {
        const int e = u * kWgConsumers + wg;
        a_off[u] = e < p.n_units ? (uint32_t)p.units[e].a_off : 0u;
        b_off[u] = e < p.n_units ? (uint32_t)p.units[e].b_off : 0u;
    }
    const uint32_t st0 = smem_u32(smem);
    uint32_t s = 0, ph = 0;
    for (int it = 0; it < n_iter; ++it) {
        mbar_wait(full_bar + s, ph);
        const uint32_t st = st0 + s * (uint32_t)p.stage_bytes;
        wgmma_fence();
        for (int k = 0; k < ksteps; ++k) {
#pragma unroll
            for (int u = 0; u < kWgSlots; ++u)
                if (u * kWgConsumers + wg < p.n_units)
                    wgmma_64x64x16<1, 1>(acc[u], make_smem_desc_mn(st + a_off[u] + k * 2048),
                                         make_smem_desc_mn(st + b_off[u] + k * 2048));
        }
        wgmma_commit();
        wgmma_wait_all();
        if (lane == 0) mbar_arrive(empty_bar + s);
        if (++s == (uint32_t)S) { s = 0; ph ^= 1; }
    }
    // ===================== epilogue: fp32 partial of this (tile, split) =====================
    float* tl = acc_tiles + wg * (kAccTileBytes / 4);
    float* __restrict__ out_split = partial + (size_t)split * p.taps * p.Cout * p.Cin;
    const int m = threadIdx.x & 63, half = (threadIdx.x >> 6) & 1;   // accumulator row, 32-column half
#pragma unroll
    for (int u = 0; u < kWgSlots; ++u) {
        const int e = u * kWgConsumers + wg;
        if (e < p.n_units) {
            wg_sync(wg);
            acc_stage(acc[u], tl);
            wg_sync(wg);
            float v[32];
            acc_row32(tl, m, half * 32, v);
            const WgUnit& un = p.units[e];
            const int n0 = half * 32;
            if (p.mode == 0) {
                // rows = output channels, columns = input channels of tap (r, un.tap): 128 contiguous bytes
                const int tap = 3 * r + un.tap;
                float4* o4 = reinterpret_cast<float4*>(out_split + ((size_t)tap * p.Cout + co0 + un.co_base + m) * p.Cin +
                                                       ci0 + un.ci_base + n0);
#pragma unroll
                for (int j = 0; j < 8; ++j) o4[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            } else if (p.mode == 2) {
                // stem: rows = k = q * 16 + c of filter row un.tap, columns = output channels
                const int q = m >> 4, c = m & 15;
                if (q < 3) {
                    float* o = out_split + ((size_t)(un.tap * 3 + q) * p.Cout + co0 + n0) * p.Cin + c;
#pragma unroll
                    for (int j = 0; j < 32; ++j) o[(size_t)j * p.Cin] = v[j];
                }
            } else {
                // rows = input channels of tap un.tap, columns = output channels: a warp's 32 lanes are 32
                // consecutive input channels of one (tap, co) -> coalesced 128-byte stores
                float* o = out_split + ((size_t)un.tap * p.Cout + co0 + n0) * p.Cin + ci0 + un.ci_base + m;
#pragma unroll
                for (int j = 0; j < 32; ++j) o[(size_t)j * p.Cin] = v[j];
            }
        }
    }
}

// sum the split-K slices in a fixed order (deterministic) and write the torch layout dW[co][ci][r][s].
// blockDim = (32, 8): thread (x, y) owns 4 consecutive input channels of one (tap, co) and the slices y, y + 8, ...;
// the 8 partial sums are combined through shared memory in y order.  Reads are 512 contiguous bytes per warp.
__global__ void __launch_bounds__(256)
wgrad2_reduce_kernel(const float* __restrict__ partial, int splits, int taps, int Cout, int Cin, int Cin_true,
                     float* __restrict__ dw) {
    __shared__ float4 sm[8][32];
    const size_t total4 = (size_t)taps * Cout * Cin / 4;
    const size_t q = (size_t)blockIdx.x * 32 + threadIdx.x;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q < total4) {
        const float4* src = reinterpret_cast<const float4*>(partial) + q;
        for (int s = threadIdx.y; s < splits; s += 8) {
            const float4 v = __ldg(src + (size_t)s * total4);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
    }
    sm[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && q < total4) {
#pragma unroll
        for (int y = 1; y < 8; ++y) {
            const float4 v = sm[y][threadIdx.x];
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        const size_t i = q * 4;
        const int ci = (int)(i % Cin);
        const int co = (int)((i / Cin) % Cout);
        const int tap = (int)(i / ((size_t)Cin * Cout));
        const float vals[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (ci + j < Cin_true) dw[((size_t)co * Cin_true + ci + j) * taps + tap] = vals[j];
    }
}

// stem: dW[co][c][tap] = sum over slices of (partial[tap][co][c] + partial[tap][co][c + 8]) -- channels c and c + 8
// of the 16-channel input are bf16(x) and its rounding residual, which share one weight (conv_stem.cu)
__global__ void __launch_bounds__(256)
stem_reduce_kernel(const float* __restrict__ partial, int splits, int Cin_true, float* __restrict__ dw) {
    const int i = blockIdx.x * 256 + threadIdx.x;            // (tap, co, c < 8)
    if (i >= 9 * 64 * 8) return;
    const int c = i & 7, co = (i >> 3) & 63, tap = i >> 9;
    if (c >= Cin_true) return;
    const size_t total = (size_t)9 * 64 * 16, o = ((size_t)tap * 64 + co) * 16 + c;
    float acc = 0.0f;
    for (int s = 0; s < splits; ++s) acc += __ldg(partial + (size_t)s * total + o) + __ldg(partial + (size_t)s * total + o + 8);
    dw[((size_t)co * Cin_true + c) * 9 + tap] = acc;
}

bool wgrad2_eligible(int Cin, int Cout, int ksize, int stride_h, int stride_w) {
    if (ksize != 3 || Cin % 64 != 0) return false;
    if (Cout % 128 == 0) return true;
    return Cout == 64 && stride_h == 1 && stride_w == 1;
}

static void wgrad2_shape(int B, int Hout, int Wout, int Cin, int Cout, int sw, Wg2Params* p) {
    p->mode = (Cout % 128 == 0) ? 0 : 1;
    const int ns_cap = (sw == 2) ? 64 : 128;
    p->NS = Wout >= ns_cap ? ns_cap : (Wout + 15) / 16 * 16;
    p->segs = (Wout + p->NS - 1) / p->NS;
    p->k_rows = B * Hout * p->segs;
    if (p->mode == 0) {
        p->ci_per_tile = 64; p->co_per_tile = 128;
        p->ci_tiles = Cin / p->ci_per_tile; p->co_tiles = Cout / 128;
        p->n_tiles = 3 * p->ci_tiles * p->co_tiles;
    } else {
        p->ci_per_tile = 64; p->co_per_tile = 64;
        p->ci_tiles = Cin / 64; p->co_tiles = Cout / 64;
        p->n_tiles = p->ci_tiles * p->co_tiles;
    }
    int splits = num_sms() / p->n_tiles;
    if (splits < 1) splits = 1;
    if (splits > p->k_rows) splits = p->k_rows > 0 ? p->k_rows : 1;
    p->splits = splits;
}

int64_t wgrad2_scratch_floats(int B, int Hout, int Wout, int Cin, int Cout, int sw) {
    Wg2Params p;
    wgrad2_shape(B, Hout, Wout, Cin, Cout, sw, &p);
    return (int64_t)p.splits * 9 * Cout * Cin;
}

int wgrad2_launch(const void* x, const void* dz, float* dw, float* scratch, int B, int Hin, int Win, int Cin, int Cin_true,
                  int Cout, int stride_h, int stride_w, cudaStream_t st) {
    Wg2Params p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.Cin = Cin; p.Cout = Cout; p.taps = 9; p.sh = stride_h; p.sw = stride_w;
    p.Hout = (Hin - 1) / stride_h + 1; p.Wout = (Win - 1) / stride_w + 1;
    wgrad2_shape(B, p.Hout, p.Wout, Cin, Cout, stride_w, &p);
    const int NS = p.NS;
    const int DB = NS * 128;                                        // one 64-channel block of dZ
    const int xpix = (stride_w == 2) ? NS + 1 : NS + 2;             // pixels per X tile
    const int TS = (xpix * 128 + 1023) / 1024 * 1024;
    int nl = 0, nu = 0;
    if (p.mode == 0) {
        p.loads[nl++] = WgLoad{0, 0, 0, 0, 0, DB};
        p.loads[nl++] = WgLoad{0, 1, 0, 0, DB, DB};
        const int xo = 2 * DB;
        // (X tile offset, tap q): stride 1 -- taps q = 0, 1, 2 one pixel apart in one tile; stride 2 -- even columns
        // (q = 0 and, one pixel later, q = 2), odd columns (q = 1)
        const int xt[3][2] = {{xo, 0}, {xo + 128, stride_w == 1 ? 1 : 2}, {stride_w == 1 ? xo + 256 : xo + TS, stride_w == 1 ? 2 : 1}};
        p.loads[nl++] = WgLoad{1, 0, 0, 0, xo, xpix * 128};
        if (stride_w == 2) p.loads[nl++] = WgLoad{1, 0, 1, 0, xo + TS, xpix * 128};
        for (int ab = 0; ab < 2; ++ab)
            for (int t = 0; t < 3; ++t) p.units[nu++] = WgUnit{ab * DB, xt[t][0], xt[t][1], 64 * ab, 0};
        p.stage_bytes = xo + (stride_w == 2 ? 2 : 1) * TS;
    } else {
        p.loads[nl++] = WgLoad{0, 0, 0, 0, 0, DB};
        const int xo = DB;
        for (int rr = 0; rr < 3; ++rr) p.loads[nl++] = WgLoad{1, 0, 0, rr, xo + rr * TS, xpix * 128};
        // A = the X view of tap (rr, q): row rr's tile, q pixels in
        for (int t = 0; t < 9; ++t) p.units[nu++] = WgUnit{xo + (t / 3) * TS + (t % 3) * 128, 0, t, 0, 0};
        p.stage_bytes = xo + 3 * TS;
    }
    p.n_loads = nl; p.n_units = nu;
    p.stage_tx = 0;
    for (int l = 0; l < nl; ++l) p.stage_tx += p.loads[l].bytes;
    int stages = (kWgSmemBudget - kWgConsumers * kAccTileBytes) / p.stage_bytes;
    if (stages > kWgMaxStages) stages = kWgMaxStages;
    DELORA_CHECK_ARG(stages >= 2, "conv_wgrad2: stage of %d bytes does not fit twice", p.stage_bytes);
    p.stages = stages;

    CUtensorMap map_dz, map_x;
    int rc = tma_nhwc(&map_dz, dz, B, p.Hout, p.Wout, Cout, NS, 1, 1, 1, true);
    DELORA_CHECK_ARG(rc == 0, "conv_wgrad2: tensor map (dz) failed: %d", rc);
    rc = tma_nhwc(&map_x, x, B, Hin, Win, Cin, xpix * stride_w, 1, stride_w, 1, false);
    DELORA_CHECK_ARG(rc == 0, "conv_wgrad2: tensor map (x) failed: %d", rc);
    const size_t smem = (size_t)p.stages * p.stage_bytes + kWgConsumers * kAccTileBytes + 2 * kWgMaxStages * 8 + 1024;
    const cudaError_t e = smem_opt_in<conv_wgrad2_tc_kernel>();
    DELORA_CHECK_ARG(e == cudaSuccess, "conv_wgrad2: shared-memory opt-in failed: %s", cudaGetErrorString(e));
    conv_wgrad2_tc_kernel<<<p.n_tiles * p.splits, kWgThreads, smem, st>>>(map_dz, map_x, scratch, p);
    DELORA_CHECK_LAUNCH("conv_wgrad2_tc_kernel");
    const size_t total4 = (size_t)9 * Cout * Cin / 4;
    wgrad2_reduce_kernel<<<(unsigned)((total4 + 31) / 32), dim3(32, 8), 0, st>>>(scratch, p.splits, 9, Cout, Cin, Cin_true, dw);
    DELORA_CHECK_LAUNCH("wgrad2_reduce_kernel");
    return 0;
}

// stem (conv_stem.cu): X tiles come from the overlapping-stride map (one 128-byte row = the 4 x 16-channel window of
// an output pixel); a unit = one filter row: M = 64 k = 4 pixels x 16 channels, N = 64 output channels
static void wgrad2_stem_shape(int B, int H, int Wout, Wg2Params* p) {
    p->mode = 2;
    p->NS = 128; p->segs = (Wout + 127) / 128; p->k_rows = B * H * p->segs;
    p->ci_per_tile = 16; p->co_per_tile = 64; p->ci_tiles = 1; p->co_tiles = 1; p->n_tiles = 1;
    p->splits = p->k_rows < num_sms() ? (p->k_rows > 0 ? p->k_rows : 1) : num_sms();
}

int64_t wgrad2_stem_scratch_floats(int B, int H, int Wout) {
    Wg2Params p;
    wgrad2_stem_shape(B, H, Wout, &p);
    return (int64_t)p.splits * 9 * 64 * 16;
}

int wgrad2_launch_stem(const CUtensorMap& map_x, const void* dz, float* dw, float* scratch, int B, int H, int Wout,
                       int Cin_true, cudaStream_t st) {
    Wg2Params p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.Cin = 16; p.Cout = 64; p.taps = 9; p.sh = 1; p.sw = 1; p.Hout = H; p.Wout = Wout;
    wgrad2_stem_shape(B, H, Wout, &p);
    const int T = 16384;
    p.loads[0] = WgLoad{0, 0, 0, 0, 0, T};
    for (int rr = 0; rr < 3; ++rr) p.loads[1 + rr] = WgLoad{1, 0, 0, rr, T + rr * T, T};
    for (int rr = 0; rr < 3; ++rr) p.units[rr] = WgUnit{T + rr * T, 0, rr, 0, 0};     // filter row rr
    p.n_loads = 4; p.n_units = 3; p.stage_bytes = 4 * T; p.stage_tx = 4 * T;
    p.stages = (kWgSmemBudget - kWgConsumers * kAccTileBytes) / p.stage_bytes;
    CUtensorMap map_dz;
    const int rc = tma_nhwc(&map_dz, dz, B, H, Wout, 64, 128, 1, 1, 1, true);
    DELORA_CHECK_ARG(rc == 0, "stem wgrad: tensor map (dz) failed: %d", rc);
    const size_t smem = (size_t)p.stages * p.stage_bytes + kWgConsumers * kAccTileBytes + 2 * kWgMaxStages * 8 + 1024;
    const cudaError_t e = smem_opt_in<conv_wgrad2_tc_kernel>();
    DELORA_CHECK_ARG(e == cudaSuccess, "stem wgrad: shared-memory opt-in failed: %s", cudaGetErrorString(e));
    conv_wgrad2_tc_kernel<<<p.n_tiles * p.splits, kWgThreads, smem, st>>>(map_dz, map_x, scratch, p);
    DELORA_CHECK_LAUNCH("conv_wgrad2_tc_kernel (stem)");
    stem_reduce_kernel<<<(9 * 64 * 8 + 255) / 256, 256, 0, st>>>(scratch, p.splits, Cin_true, dw);
    DELORA_CHECK_LAUNCH("stem_reduce_kernel");
    return 0;
}

}  // namespace delora
