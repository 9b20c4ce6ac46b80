// Encoder convolutions, second-generation kernel: row-block implicit GEMM with the filter taps issued from ONE halo tile
// in shared memory.
//
// Same operator as conv_tc.cu (the reference's nn.Conv2d layers, src/models/resnet_modified.py:126-134 used at
// :159-177; circular padding in W, zero padding in H, materialised in the padded NHWC bf16 layout) for the layers
// that carry the FLOPs: 3x3 (and 1x1) stride-1 convolutions with Cout % 128 == 0, and the data gradient of the
// strided 3x3 convolutions by PHASE DECOMPOSITION (each output phase (h % sh, w % sw) is a small convolution of the
// un-upsampled output gradient with a subset of the flipped taps: no zero-upsampled tensor, no MMAs on zeros).
//
// Why a second kernel: conv_tc.cu loads every (tap, 64-channel chunk) as its own TMA box, so an activation tile is
// fetched 9x from L2.  Here
//   * M = 128 OUTPUT CHANNELS (A operand = filter tile [128 co][64 ci], K-major; each of the two consumer warpgroups
//     owns 64 of them), N = the NS pixels of one output-row segment (B operand = activation rows, K-major), R rows
//     per job, so ANY image width maps onto the N dimension (multiples of 16);
//   * per job and 64-channel chunk ONE TMA box brings the (R + 2) x (NS + 2) pixel halo tile; the B descriptor of
//     tap (r, q), row i starts at byte ((i + r) * (NS + 2) + q) * 128 of that tile -- the 128-byte swizzle follows the
//     absolute shared-memory address, so 128-byte-granular start offsets need no re-layout.  Activation traffic per
//     MMA drops ~6x;
//   * CTAs are persistent (grid = min(jobs, SMs)); separate producer warps stream halo tiles (2 stages) and filter
//     tiles (a ring of 2-8 stages), so the next job's tiles arrive while the current job's epilogue runs;
//   * the accumulators of a job are up to four 64 x 64 fp32 register tiles per warpgroup (row i x 64-pixel chunk);
//     the epilogue reads each through shared memory as one pixel x 32 channels (64 contiguous bytes of NHWC), then
//     residual / activation / act' / store as in conv_tc.cu.
// Warp roles: 0..7 MMA + epilogue (two warpgroups), 8 halo-tile producer, 9 filter producer.
#include <string.h>
#include <stdlib.h>
#include "tc_common.cuh"

namespace delora {

constexpr int kRowsThreads = 320;                 // two consumer warpgroups + two producer warps
constexpr int kRowsMaxUnits = 4;                  // 64 x 64 accumulators per warpgroup and job
constexpr int kRowsMaxTaps = 9;
constexpr int kRowsMaxPhases = 4;
constexpr int kWTileBytes = 128 * 64 * 2;          // filter tile: 128 output channels x 64 input channels
// Dynamic shared memory of one persistent CTA: 226 KB, not the 227 KB maximum -- 228 KB per SM minus this and the 1 KB
// the system reserves per CTA leaves room for ONE more (shared-memory-free) CTA on the SM, which is what lets the
// gradient all-reduce kernel (grad_allreduce.cu) run beside the convolutions instead of between them.
constexpr int kRowsSmemBudget = 226 * 1024;

struct RowsPhase {
    int ntaps;
    int oh, ow;                                    // output pixel = (out_sh * h + oh, out_sw * w + ow)
    signed char drow[kRowsMaxTaps], dcol[kRowsMaxTaps], wtap[kRowsMaxTaps];
};

struct RowsParams {
    int B, Cin, Cout;
    int Hout, Wout;                                // output tensor (unpadded) size
    int Hg, Wg;                                    // job grid extent in phase coordinates (= Hout, Wout for stride 1)
    int out_sh, out_sw;
    int NS, R;                                     // pixels per row segment, rows per job
    int nch;                                       // 64-wide chunks of N per row: ceil(NS / 64), or n_tile / 64 (PIXM)
    int segs_w, blocks_h, co_tiles, kchunks;
    int n_phases;
    int n_jobs;
    int act;
    int w_stages;
    int a_stage_bytes;
    int n_tile;                                    // pixel-on-M mode: output channels per job (MMA N) = Cout <= 128
    int w_tile_bytes;                              // bytes of one filter tile in the ring
    int res_grid;                                  // 1: `residual` is given on the job grid [B, Hg+2, Wg+2, Cout] and belongs
                                                   //    to phase (0, 0) only (data gradient of a 1x1 strided downsample)
    RowsPhase phase[kRowsMaxPhases];
};

struct RowsJob { int ct, ph, b, h0, w0; };

// job -> (co tile, phase, image, first row, first column)
__device__ __forceinline__ RowsJob rows_decode(const RowsParams& p, int job) {
    RowsJob j;
    j.ct = job % p.co_tiles; job /= p.co_tiles;
    j.w0 = (job % p.segs_w) * p.NS; job /= p.segs_w;
    j.h0 = (job % p.blocks_h) * p.R; job /= p.blocks_h;
    j.b = job % p.B; job /= p.B;
    j.ph = job;                                    // phase-major: the phases with the most taps come first (host order)
    return j;
}

// PIXM (layers with Cout = 64 / 128, where M = 128 output channels cannot be filled): the roles are swapped --
//         M = the 128 PIXELS of a row segment (A operand = halo-tile rows, same shifted descriptors; warpgroup wg takes
//         pixels 64 wg ..), N = all Cout output channels (B operand = filter tile [Cout][64]).
// Unit u of a job = (row i = u / nch, 64-wide N chunk c = u % nch).
template <bool PIXM>
__global__ void __launch_bounds__(kRowsThreads, 1)
conv_rows_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                    const __nv_bfloat16* __restrict__ residual, const __nv_bfloat16* __restrict__ saved,
                    __nv_bfloat16* __restrict__ y, const __grid_constant__ RowsParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = DELORA_ALIGNED_SMEM(smem_raw);
    uint8_t* smem_a = smem;                                        // 2 halo-tile stages
    uint8_t* smem_w = smem_a + 2 * p.a_stage_bytes;                // filter ring
    float* acc_tiles = reinterpret_cast<float*>(smem_w + p.w_stages * p.w_tile_bytes);
    uint64_t* a_full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(acc_tiles) + 2 * kAccTileBytes);
    uint64_t* a_empty = a_full + 2;
    uint64_t* w_full = a_empty + 2;
    uint64_t* w_empty = w_full + 8;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int S = p.w_stages;
    const int pitch = p.NS + 2;                                    // pixels per halo-tile row

    if (threadIdx.x == 0) {
        for (int s = 0; s < 2; ++s) { mbar_init(a_full + s, 1); mbar_init(a_empty + s, 8); }
        for (int s = 0; s < S; ++s) { mbar_init(w_full + s, 1); mbar_init(w_empty + s, 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ===================== halo-tile producer =====================
        if (lane == 0) {
            tma_prefetch_desc(&map_x);
            const uint32_t a_bytes = (uint32_t)(pitch * (p.R + 2) * 128);
            uint32_t it = 0;
            for (int job = blockIdx.x; job < p.n_jobs; job += gridDim.x) {
                const RowsJob j = rows_decode(p, job);
                for (int kc = 0; kc < p.kchunks; ++kc, ++it) {
                    const uint32_t s = it & 1;
                    mbar_wait(a_empty + s, ((it >> 1) & 1) ^ 1);
                    // local (row j, pixel c) = padded input pixel (h0 + j, w0 + c)
                    mbar_expect_tx(a_full + s, a_bytes);
                    tma_load_4d(smem_a + s * p.a_stage_bytes, &map_x, a_full + s, kc * 64, j.w0, j.h0, j.b);
                }
            }
        }
        return;
    }
    if (warp == 9) {
        // ===================== filter producer =====================
        if (lane == 0) {
            tma_prefetch_desc(&map_w);
            uint32_t it = 0;
            for (int job = blockIdx.x; job < p.n_jobs; job += gridDim.x) {
                const RowsJob j = rows_decode(p, job);
                const RowsPhase& ph = p.phase[j.ph];
                const int co0 = PIXM ? j.ct * p.n_tile : j.ct * 128;
                const uint32_t wb = (uint32_t)p.w_tile_bytes;
                for (int kc = 0; kc < p.kchunks; ++kc)
                    for (int t = 0; t < ph.ntaps; ++t, ++it) {
                        const uint32_t s = it % S;
                        mbar_wait(w_empty + s, ((it / S) & 1) ^ 1);
                        mbar_expect_tx(w_full + s, wb);
                        tma_load_2d(smem_w + s * wb, &map_w, w_full + s, (int)ph.wtap[t] * p.Cin + kc * 64, co0);
                    }
            }
        }
        return;
    }
    // ===================== MMA + epilogue (warpgroup wg) =====================
    const int wg = warp >> 2;
    const int row = threadIdx.x & 63, half = (threadIdx.x >> 6) & 1;
    float* tile = acc_tiles + wg * (kAccTileBytes / 4);
    const int n_units = p.R * p.nch;
    const uint32_t row_bytes = (uint32_t)pitch * 128u;
    const uint32_t a_base = smem_u32(smem_a), w_base = smem_u32(smem_w);
    const int Wp = p.Wout + 2, Hp = p.Hout + 2;
    uint32_t as = 0, aph = 0, ws = 0, wph = 0;                     // ring slots and phase bits
    // One wgmma group stays in flight: the stages a group reads are released once the NEXT group has been issued and
    // this one has completed (wait_group 1), so the tensor core does not idle while a stage is handed back.
    int pend_ws = -1, pend_as = -1;                                // stages read by the group still in flight
    for (int job = blockIdx.x; job < p.n_jobs; job += gridDim.x) {
        const RowsJob j = rows_decode(p, job);
        const RowsPhase& ph = p.phase[j.ph];
        float acc[kRowsMaxUnits][32];
#pragma unroll
        for (int u = 0; u < kRowsMaxUnits; ++u)
#pragma unroll
            for (int e = 0; e < 32; ++e) acc[u][e] = 0.0f;
        for (int kc = 0; kc < p.kchunks; ++kc) {
            mbar_wait(a_full + as, aph);
            const uint32_t x_stage = a_base + as * (uint32_t)p.a_stage_bytes;
            for (int t = 0; t < ph.ntaps; ++t) {
                mbar_wait(w_full + ws, wph);
                const uint32_t x_tap = x_stage + (uint32_t)(((int)ph.drow[t] * pitch + (int)ph.dcol[t]) * 128);
                const uint32_t w_addr = w_base + ws * (uint32_t)p.w_tile_bytes;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {                   // 64 channels = 4 x K16; +32 bytes = +2 in 16-byte units
#pragma unroll
                    for (int u = 0; u < kRowsMaxUnits; ++u) {
                        if (u < n_units) {
                            const int i = u / p.nch, c = u - i * p.nch;
                            if (PIXM) {
                                const uint64_t da = make_smem_desc(x_tap + i * row_bytes + wg * 64 * 128) + (uint64_t)(k * 2);
                                const uint64_t db = make_smem_desc(w_addr + c * 8192) + (uint64_t)(k * 2);
                                wgmma_64x64x16<0, 0>(acc[u], da, db);
                            } else {
                                // The last chunk always spans 64 pixel rows: with NS < 64 * nch it reads up to
                                // (64 * nch - NS) * 128 B past this row's pixels -- into the next halo row, the other
                                // halo stage or the filter ring, possibly while TMA writes there.  Such a B row only
                                // feeds its own accumulator column, i.e. pixels wl >= NS, which the epilogue never
                                // stores (`wl < p.NS`).  The smem layout must keep that over-read inside the allocation:
                                // the halo stages are followed by the filter ring and the accumulator tiles.
                                const uint64_t da = make_smem_desc(w_addr + wg * 8192) + (uint64_t)(k * 2);
                                const uint64_t db = make_smem_desc(x_tap + i * row_bytes + c * 64 * 128) + (uint64_t)(k * 2);
                                wgmma_64x64x16<0, 0>(acc[u], da, db);
                            }
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait_one();
                if (lane == 0 && pend_ws >= 0) {
                    mbar_arrive(w_empty + pend_ws);               // filter tile of the previous group consumed
                    if (pend_as >= 0) mbar_arrive(a_empty + pend_as);   // halo tile free after a chunk's last tap
                }
                pend_ws = (int)ws;
                pend_as = (t == ph.ntaps - 1) ? (int)as : -1;
                if (++ws == (uint32_t)S) { ws = 0; wph ^= 1; }
            }
            as ^= 1; aph ^= (as == 0);
        }
        wgmma_wait_all();                                           // accumulators of this job complete
        if (lane == 0 && pend_ws >= 0) {
            mbar_arrive(w_empty + pend_ws);
            if (pend_as >= 0) mbar_arrive(a_empty + pend_as);
        }
        pend_ws = -1; pend_as = -1;
        // epilogue: unit (row i, chunk c) -> one pixel x 32 channels per thread
#pragma unroll
        for (int u = 0; u < kRowsMaxUnits; ++u) {
            if (u < n_units) {
                const int i = u / p.nch, c = u - i * p.nch;
                wg_sync(wg);
                acc_stage(acc[u], tile);
                wg_sync(wg);
                float v[32];
                int wl, c_first;
                if (PIXM) {
                    acc_row32(tile, row, half * 32, v);            // rows = pixels, columns = output channels
                    wl = wg * 64 + row;
                    c_first = j.ct * p.n_tile + c * 64 + half * 32;
                } else {
                    acc_col32(tile, row, half * 32, v);            // rows = output channels, columns = pixels
                    wl = c * 64 + row;
                    c_first = j.ct * 128 + wg * 64 + half * 32;
                }
                const int hg = j.h0 + i, wgx = j.w0 + wl;
                const int ho = hg * p.out_sh + ph.oh, wo = wgx * p.out_sw + ph.ow;
                if (wl < p.NS && hg < p.Hg && wgx < p.Wg && ho < p.Hout && wo < p.Wout) {
                    const bool use_res = residual != nullptr && (!p.res_grid || (ph.oh | ph.ow) == 0);
                    const size_t off = (((size_t)j.b * Hp + (ho + 1)) * Wp + (wo + 1)) * p.Cout + c_first;
                    const size_t roff = p.res_grid ? (((size_t)j.b * (p.Hg + 2) + (hg + 1)) * (p.Wg + 2) + (wgx + 1)) * p.Cout + c_first
                                                   : off;
                    EpiloguePrefetch pf;
                    epilogue_prefetch32(pf, use_res ? residual + roff : nullptr, saved + (p.act >= 3 ? off : 0), 0, p.act);
                    epilogue_finish32(v, pf, use_res, y, off, p.act, wo == 0, wo == p.Wout - 1, (size_t)p.Wout * p.Cout);
                }
            }
        }
    }
}

// ---------------------------------------------------------------- host side
static int rows_encode_maps(CUtensorMap* mx, CUtensorMap* mw, const void* x, const void* w, int B, int Hin, int Win,
                            int Cin, int Cout, int wtaps, int NS, int R, int w_rows) {
    PFN_cuTensorMapEncodeTiled_v12000 encode = get_tensor_map_encoder();
    if (!encode) return 1;
    const int Hp = Hin + 2, Wp = Win + 2;
    {
        cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)Wp, (cuuint64_t)Hp, (cuuint64_t)B};
        cuuint64_t strides[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)Wp * Cin * 2, (cuuint64_t)Hp * Wp * Cin * 2};
        cuuint32_t box[4] = {64, (cuuint32_t)(NS + 2), (cuuint32_t)(R + 2), 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        if (encode(mx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return 2;
    }
    {
        cuuint64_t dims[2] = {(cuuint64_t)wtaps * Cin, (cuuint64_t)Cout};
        cuuint64_t strides[1] = {(cuuint64_t)wtaps * Cin * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)w_rows};
        cuuint32_t estr[2] = {1, 1};
        if (encode(mw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return 3;
    }
    return 0;
}

// Tensor maps depend only on (pointers, shapes); the encoder's activations, filters and gradients live in
// persistent buffers, so a small per-thread cache removes the encode cost from the 40 launches of a step.
struct RowsMapKey { const void* x; const void* w; int B, Hin, Win, Cin, Cout, wtaps, NS, R, w_rows; };
struct RowsMapEntry { RowsMapKey k; CUtensorMap mx, mw; };

static const RowsMapEntry* rows_get_maps(const RowsMapKey& key) {
    static thread_local RowsMapEntry cache[128];
    static thread_local int used = 0, next = 0;
    for (int i = 0; i < used; ++i) {
        const RowsMapKey& c = cache[i].k;
        if (c.x == key.x && c.w == key.w && c.B == key.B && c.Hin == key.Hin && c.Win == key.Win && c.Cin == key.Cin &&
            c.Cout == key.Cout && c.wtaps == key.wtaps && c.NS == key.NS && c.R == key.R && c.w_rows == key.w_rows)
            return &cache[i];
    }
    RowsMapEntry& e = cache[next];
    if (rows_encode_maps(&e.mx, &e.mw, key.x, key.w, key.B, key.Hin, key.Win, key.Cin, key.Cout, key.wtaps, key.NS,
                         key.R, key.w_rows) != 0)
        return nullptr;
    e.k = key;
    const RowsMapEntry* out = &e;
    next = (next + 1) % 128;
    if (used < 128) ++used;
    return out;
}

// segment width for a job grid Hg x Wg: NS = multiple of 16 covering the row in equal segments of at most 128 pixels
static int rows_pick_ns(int Wg) {
    const int segs = (Wg + 127) / 128;
    const int ns = ((Wg + segs - 1) / segs + 15) / 16 * 16;
    return ns < 16 ? 16 : ns;
}

// pixel-on-M mode: Cout = 64 or 128 and a job grid at least one full 128-pixel segment wide
static bool rows_pixm(int Cout, int Wg) { return (Cout == 64 || Cout == 128) && Wg >= 128; }

// Wg = width of the job grid (the output width for a stride-1 convolution, ceil(Wout / stride_w) for a data gradient)
bool conv_rows_eligible(int Cin, int Cout, int ksize, int Wg) {
    if (Cin % 64 != 0 || !(ksize == 3 || ksize == 1)) return false;
    return Cout % 128 == 0 || rows_pixm(Cout, Wg);
}

// stride-1 convolution (up_h = up_w = 1) or data gradient of a stride-(up_h, up_w) 3x3 convolution (x = output
// gradient of that convolution, w = its flipped / transposed filter [Cout][9][Cin], y = input gradient Hout x Wout)
int conv_rows_launch(const void* x, const void* w, const void* residual, const void* saved, void* y, int B, int Hout,
                     int Wout, int Cin, int Cout, int ksize, int up_h, int up_w, int act, cudaStream_t stream,
                     int residual_on_grid) {
    RowsParams p;
    memset(&p, 0, sizeof(p));
    p.res_grid = (residual_on_grid && (up_h > 1 || up_w > 1)) ? 1 : 0;
    p.B = B; p.Cin = Cin; p.Cout = Cout; p.Hout = Hout; p.Wout = Wout; p.act = act;
    p.out_sh = up_h; p.out_sw = up_w;
    p.Hg = (Hout + up_h - 1) / up_h; p.Wg = (Wout + up_w - 1) / up_w;
    const int Hin = (Hout - 1) / up_h + 1, Win = (Wout - 1) / up_w + 1;      // size of x (unpadded)
    if (ksize == 1) {
        p.n_phases = 1;
        p.phase[0].ntaps = 1; p.phase[0].drow[0] = 1; p.phase[0].dcol[0] = 1; p.phase[0].wtap[0] = 0;
    } else if (up_h == 1 && up_w == 1) {
        p.n_phases = 1;
        p.phase[0].ntaps = 9;
        for (int t = 0; t < 9; ++t) { p.phase[0].drow[t] = (signed char)(t / 3); p.phase[0].dcol[t] = (signed char)(t % 3); p.phase[0].wtap[t] = (signed char)t; }
    } else {
        // out[h][w] = sum_{r', q'} U[h + r' - 1][w + q' - 1] * Wf[r'][q'],  U = zero-upsampled x: only taps with
        // (h + r' - 1) % up_h == 0 and (w + q' - 1) % up_w == 0 contribute.  Phase (fh, fw): h = up_h * jh + fh.
        // Local halo-tile coordinates: padded x row jh0 + drow, drow = (fh + r' - 1) / up_h + 1 (same for columns).
        int np = 0;
        // phases ordered by decreasing tap count (static round-robin over CTAs: expensive jobs first)
        for (int pass = 9; pass >= 1; --pass)
            for (int fh = 0; fh < up_h; ++fh)
                for (int fw = 0; fw < up_w; ++fw) {
                    RowsPhase ph;
                    memset(&ph, 0, sizeof(ph));
                    ph.oh = fh; ph.ow = fw;
                    for (int r = 0; r < 3; ++r) {
                        if ((fh + r - 1 + up_h) % up_h != 0) continue;
                        for (int q = 0; q < 3; ++q) {
                            if ((fw + q - 1 + up_w) % up_w != 0) continue;
                            // floor division of (fh + r - 1) by up_h, values -1 .. 2
                            const int dr = (fh + r - 1 + up_h) / up_h - 1, dq = (fw + q - 1 + up_w) / up_w - 1;
                            ph.drow[ph.ntaps] = (signed char)(dr + 1); ph.dcol[ph.ntaps] = (signed char)(dq + 1);
                            ph.wtap[ph.ntaps] = (signed char)(r * 3 + q);
                            ++ph.ntaps;
                        }
                    }
                    if (ph.ntaps == pass) p.phase[np++] = ph;
                }
        p.n_phases = np;
    }
    const bool pixm = rows_pixm(Cout, p.Wg);
    if (pixm) {
        p.NS = 128;                                    // 128 pixels on M, Cout columns per row
        p.n_tile = Cout; p.w_tile_bytes = Cout * 128;
        p.nch = Cout / 64;
        p.co_tiles = 1;
    } else {
        p.NS = rows_pick_ns(p.Wg);
        p.n_tile = 0; p.w_tile_bytes = kWTileBytes;
        p.nch = (p.NS + 63) / 64;
        p.co_tiles = Cout / 128;
    }
    p.kchunks = Cin / 64;
    // rows per job: as many as the accumulator registers hold (R x nch <= 4 units), no more than the image has, and
    // small enough that two halo tiles and two filter tiles fit next to the accumulator hand-off tiles
    const int fixed_other = 2 * kAccTileBytes + 256 + 1024;
    int R = kRowsMaxUnits / p.nch;
    if (R > p.Hg) R = p.Hg;
    if (R < 1) R = 1;
    auto a_stage = [&](int r) { return (((p.NS + 2) * (r + 2) * 128) + 1023) / 1024 * 1024; };
    while (R > 1 && 2 * a_stage(R) + fixed_other + 2 * p.w_tile_bytes > kRowsSmemBudget) --R;
    p.R = R;
    p.segs_w = (p.Wg + p.NS - 1) / p.NS;
    p.blocks_h = (p.Hg + p.R - 1) / p.R;
    p.n_jobs = p.n_phases * B * p.blocks_h * p.segs_w * p.co_tiles;
    p.a_stage_bytes = a_stage(p.R);
    const int fixed = 2 * p.a_stage_bytes + fixed_other;
    int ws = (kRowsSmemBudget - fixed) / p.w_tile_bytes;
    if (ws > 8) ws = 8;
    DELORA_CHECK_ARG(ws >= 2, "conv_rows: tile %dx%d leaves no room for the filter ring", p.NS, p.R);
    p.w_stages = ws;
    const RowsMapKey key = {x, w, B, Hin, Win, Cin, Cout, ksize * ksize, p.NS, p.R, p.w_tile_bytes / 128};
    const RowsMapEntry* maps = rows_get_maps(key);
    DELORA_CHECK_ARG(maps != nullptr, "conv_rows: cuTensorMapEncodeTiled failed or is unavailable");
    const size_t smem = (size_t)fixed + (size_t)ws * p.w_tile_bytes;
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_set[64] = {};
    if (dev < 64 && !attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(conv_rows_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(conv_rows_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        DELORA_CHECK_ARG(e == cudaSuccess, "conv_rows: shared-memory opt-in failed: %s", cudaGetErrorString(e));
        attr_set[dev] = true;
    }
    const int grid = p.n_jobs < num_sms() ? p.n_jobs : num_sms();
    const __nv_bfloat16* res_p = (const __nv_bfloat16*)residual;
    const __nv_bfloat16* sav_p = (const __nv_bfloat16*)saved;
    __nv_bfloat16* y_p = (__nv_bfloat16*)y;
    if (pixm)
        conv_rows_tc_kernel<true><<<grid, kRowsThreads, smem, stream>>>(maps->mx, maps->mw, res_p, sav_p, y_p, p);
    else
        conv_rows_tc_kernel<false><<<grid, kRowsThreads, smem, stream>>>(maps->mx, maps->mw, res_p, sav_p, y_p, p);
    cudaError_t le = cudaGetLastError();
    DELORA_CHECK_ARG(le == cudaSuccess, "conv_rows: launch failed: %s", cudaGetErrorString(le));
    DELORA_CHECK_LAUNCH("conv_rows_tc_kernel");
    return 0;
}

}  // namespace delora

using namespace delora;

extern "C" int delora_conv2d_dgrad_bf16(const void* dz, const void* w_flip, const void* residual, const void* saved,
                                        void* dx, int B, int Hin, int Win, int Cin, int Cout, int stride_h, int stride_w,
                                        int act, int residual_strided, void* stream) {
    // Cin / Cout are those of the FORWARD convolution: dz has Cout channels, dx has Cin channels
    DELORA_CHECK_ARG(dz && w_flip && dx, "delora_conv2d_dgrad_bf16: null pointer");
    DELORA_CHECK_ARG(act >= 0 && act <= 4 && (act < 3 || saved), "delora_conv2d_dgrad_bf16: act=%d (3/4 need `saved`)", act);
    DELORA_CHECK_ARG((stride_h == 1 || stride_h == 2) && (stride_w == 1 || stride_w == 2) && Hin >= 1 && Win >= 1,
                     "delora_conv2d_dgrad_bf16: stride (%d,%d) unsupported", stride_h, stride_w);
    DELORA_CHECK_ARG(stride_w == 1 || Win % 2 == 0, "delora_conv2d_dgrad_bf16: stride_w = 2 needs an even Win (got %d)", Win);
    DELORA_CHECK_ARG(conv_rows_eligible(Cout, Cin, 3, (Win + stride_w - 1) / stride_w),
                     "delora_conv2d_dgrad_bf16: needs Cout %% 64 == 0 and Cin %% 128 == 0 (or Cin = 64 / 128 with at least "
                     "128 columns per phase); got Cin=%d, Cout=%d, Win=%d", Cin, Cout, Win);
    return conv_rows_launch(dz, w_flip, residual, saved, dx, B, Hin, Win, Cout, Cin, 3, stride_h, stride_w, act,
                            (cudaStream_t)stream, residual_strided);
}
