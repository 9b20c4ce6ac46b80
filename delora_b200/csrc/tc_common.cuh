// PTX wrappers shared by the wgmma convolution kernels (conv_tc.cu, conv_rows.cu, conv_wgrad.cu, conv_stem.cu):
// mbarrier, TMA (cp.async.bulk.tensor), wgmma, shared-memory matrix descriptors, the accumulator hand-off; and the host
// side of their launchers: the tensor-map encoder with its cache, the shared-memory opt-in.
//
// With SWIZZLE_128B the swizzle phase of a row follows from its ABSOLUTE shared-memory address (TMA writes and the
// tensor core reads alike), so an operand may start at any multiple of 128 B inside a 1024-byte-aligned TMA-written
// tile with the descriptor's base offset left at 0.  This is what lets one halo tile serve all filter taps.
#pragma once
#include <string.h>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cudaTypedefs.h>
#include "common.cuh"

namespace delora {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!done);
}
// dynamic shared memory base rounded up to 1024 B WITHOUT leaving the shared address space (pointer arithmetic on the
// extern array; a round trip through uintptr_t makes every later access a generic LD/ST)
#define DELORA_ALIGNED_SMEM(raw) ((raw) + ((1024u - (smem_u32(raw) & 1023u)) & 1023u))
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// wgmma shared-memory matrix descriptors (128-byte swizzle): start address >> 4 (bits 0..13), leading byte offset >> 4
// (16..29), stride byte offset >> 4 (32..45), layout type 1 = SWIZZLE_128B (bits 62..63), base offset 0.
// K-major: rows of 64 K elements (128 B), SBO = 1024 B between groups of 8 rows (LBO unused).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// MN-major: rows of 64 M/N elements (128 B), K runs across rows; SBO = 1024 B between groups of 8 K rows.  Every
// operand here is 64 wide along M/N, so the leading byte offset (distance between 64-element blocks) is never used.
__device__ __forceinline__ uint64_t make_smem_desc_mn(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// ---- warpgroup MMA (wgmma): one warpgroup = 4 consecutive warps, warp index a multiple of 4.
// The kernels tile every GEMM into 64 x 64 fp32 accumulators ("units"): M = 64 rows of the A operand, N = 64 rows of
// B, K = 16 per instruction, both operands in shared memory.  TA / TB = 1: the operand is MN-major (transposed).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// all but the most recently committed group have completed (their shared-memory operands may be released)
__device__ __forceinline__ void wgmma_wait_one() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
template <int TA, int TB>
__device__ __forceinline__ void wgmma_64x64x16(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b), "r"(1), "n"(TA), "n"(TB)
        : "memory");
}
// barrier over the 128 threads of warpgroup `wg` (ids 1.. ; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory"); }

// Accumulator hand-off to the epilogue.  Fragment of thread t of a warpgroup (warp w4 = t / 32 in the group, lane l):
// d[4j + {0,1,2,3}] = rows 16 w4 + l / 4 (+ 8 for {2,3}), columns 8 j + 2 (l % 4) (+ 1 for {1,3}).  acc_stage writes
// it to a 64 x kAccPitch fp32 tile; after wg_sync a thread reads 32 consecutive values of one row (acc_row32) or of
// one column (acc_col32) -- one output pixel's 32 channels whichever operand carried the pixels.
constexpr int kAccPitch = 65;
constexpr int kAccTileBytes = 64 * kAccPitch * 4;
__device__ __forceinline__ void acc_stage(const float (&d)[32], float* tile) {
    const int t = threadIdx.x & 127, w4 = t >> 5, l = t & 31;
    const int r = 16 * w4 + (l >> 2), c = 2 * (l & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        tile[r * kAccPitch + 8 * j + c] = d[4 * j];
        tile[r * kAccPitch + 8 * j + c + 1] = d[4 * j + 1];
        tile[(r + 8) * kAccPitch + 8 * j + c] = d[4 * j + 2];
        tile[(r + 8) * kAccPitch + 8 * j + c + 1] = d[4 * j + 3];
    }
}
__device__ __forceinline__ void acc_row32(const float* tile, int row, int c0, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = tile[row * kAccPitch + c0 + j];
}
__device__ __forceinline__ void acc_col32(const float* tile, int col, int r0, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = tile[(r0 + j) * kAccPitch + col];
}

__device__ __forceinline__ float apply_act(float v, int act) {
    if (act == 1) return fmaxf(v, 0.0f);
    if (act == 2) {           // MUFU.TANH: 2^-11 relative error, far below the bf16 output rounding
        float t;
        asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(v));
        return t;
    }
    return v;
}

// ---- host: TMA tensor maps.  Every map of the convolution kernels is bf16 with the 128-byte swizzle the smem
// descriptors above assume, no interleave and zero out-of-bounds fill; what differs is the request below.
struct TmaRequest {
    const void* ptr;
    cuuint64_t dims[4], strides[3];               // strides in bytes, of dims 1 .. rank - 1
    cuuint32_t box[4], estr[4];
    int rank;
    CUtensorMapL2promotion promo;
};
static_assert(sizeof(TmaRequest) == 104, "TmaRequest is compared with memcmp: it must have no padding");

// Encodes a map (cuTensorMapEncodeTiled through the runtime's driver entry point: no -lcuda link dependency) behind a
// per-thread cache keyed on the complete request.  Activations, filters and gradients live in persistent buffers, so
// the cache takes the encode cost (microseconds of host time per map) out of the convolution launches; it holds 512
// maps: the 384 of the two caches it replaced, plus room for the weight-gradient and stem maps.
// Returns 0, the encoder's CUresult, or CUDA_ERROR_NOT_FOUND when the driver has no encoder.
inline int tma_encode(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                      const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapL2promotion promo) {
    constexpr int kCap = 512;
    struct Cache { TmaRequest keys[kCap]; CUtensorMap maps[kCap]; int used, next; };
    static thread_local Cache cache;
    TmaRequest req;
    memset(&req, 0, sizeof(req));
    req.ptr = ptr; req.rank = rank; req.promo = promo;
    for (int i = 0; i < rank; ++i) {
        req.dims[i] = dims[i]; req.box[i] = box[i]; req.estr[i] = estr[i];
        if (i > 0) req.strides[i - 1] = strides[i - 1];
    }
    for (int i = 0; i < cache.used; ++i)          // the pointer first: most entries differ there
        if (cache.keys[i].ptr == ptr && memcmp(&cache.keys[i], &req, sizeof(req)) == 0) {
            *map = cache.maps[i];
            return 0;
        }
    static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
    if (!encode) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            encode = (PFN_cuTensorMapEncodeTiled_v12000)p;
    }
    if (!encode) return CUDA_ERROR_NOT_FOUND;
    const CUresult rc = encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), req.dims,
                               req.strides, req.box, req.estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (rc != CUDA_SUCCESS) return (int)rc;
    cache.keys[cache.next] = req;
    cache.maps[cache.next] = *map;
    cache.next = (cache.next + 1) % kCap;
    if (cache.used < kCap) ++cache.used;
    return 0;
}

// Padded NHWC activation [B, H+2, W+2, C] as the map (channel, column, row, image), box (64, box_w, box_h, 1).
// sw / sh: traversal strides -- the box spans box_w (box_h) elements and loads every sw-th (sh-th) one.
// clip: the extents stop at the last REAL pixel (padded index W / H), so a ragged tile reads zeros from the
// out-of-bounds fill instead of the circular halo column (output-gradient maps of the weight gradients: the halo
// would add to the sum).
inline int tma_nhwc(CUtensorMap* map, const void* x, int B, int H, int W, int C, int box_w, int box_h, int sw, int sh,
                    bool clip) {
    const cuuint64_t Hp = (cuuint64_t)H + 2, Wp = (cuuint64_t)W + 2, pixel = (cuuint64_t)C * 2;
    const cuuint64_t dims[4] = {(cuuint64_t)C, clip ? Wp - 1 : Wp, clip ? Hp - 1 : Hp, (cuuint64_t)B};
    const cuuint64_t strides[3] = {pixel, Wp * pixel, Hp * Wp * pixel};
    const cuuint32_t box[4] = {64, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    const cuuint32_t estr[4] = {1, (cuuint32_t)sw, (cuuint32_t)sh, 1};
    return tma_encode(map, x, 4, dims, strides, box, estr, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

// Row-major bf16 filter matrix [rows][cols] as the map (column, row), box (64, box_rows).
inline int tma_filter(CUtensorMap* map, const void* w, int cols, int rows, int box_rows, CUtensorMapL2promotion promo) {
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return tma_encode(map, w, 2, dims, strides, box, estr, promo);
}

// Lets `kernel` use the full 227 KB of dynamic shared memory a CTA may have on sm_90, once per (kernel, device).  The
// flags are per template instance, i.e. per kernel ADDRESS: two instances of one kernel template share a function
// type but not their flags.
template <auto kernel>
inline cudaError_t smem_opt_in() {
    static bool done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 64 && done[dev]) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e == cudaSuccess && dev < 64) done[dev] = true;
    return e;
}

// Epilogue of one output pixel's 32 consecutive channels (fp32 accumulators in v[32]): residual add, activation or
// activation derivative of the saved forward output (dgrad modes 3 = tanh', 4 = relu'), bf16 conversion, NHWC store
// and the circular halo copies of the padded layout.  `off` = element offset of the pixel's first channel of this
// group in y / residual / saved; halo_right / halo_left: also store at pixel + Wout / pixel - Wout.
struct EpiloguePrefetch { uint4 r[4]; uint4 s[4]; };
// issue the residual / saved loads of one pixel's 32 channels early (before the accumulator hand-off)
__device__ __forceinline__ void epilogue_prefetch32(EpiloguePrefetch& pf, const __nv_bfloat16* __restrict__ residual,
                                                    const __nv_bfloat16* __restrict__ saved, size_t off, int act) {
    if (residual) {
        const uint4* rp = reinterpret_cast<const uint4*>(residual + off);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) pf.r[j4] = __ldg(rp + j4);
    }
    if (act >= 3) {
        const uint4* sp = reinterpret_cast<const uint4*>(saved + off);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) pf.s[j4] = __ldg(sp + j4);
    }
}
// same as epilogue_store32 with the residual / saved values already in registers
__device__ __forceinline__ void epilogue_finish32(float (&v)[32], const EpiloguePrefetch& pf, bool has_residual,
                                                  __nv_bfloat16* __restrict__ y, size_t off, int act, bool halo_right,
                                                  bool halo_left, size_t halo_elems) {
    if (has_residual) {
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&pf.r[j4]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __bfloat1622float2(h[e]);
                v[j4 * 8 + e * 2] += f.x; v[j4 * 8 + e * 2 + 1] += f.y;
            }
        }
    }
    if (act >= 3) {
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&pf.s[j4]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 a = __bfloat1622float2(h[e]);
                const float d0 = (act == 3) ? fmaf(-a.x, a.x, 1.0f) : (a.x > 0.0f ? 1.0f : 0.0f);
                const float d1 = (act == 3) ? fmaf(-a.y, a.y, 1.0f) : (a.y > 0.0f ? 1.0f : 0.0f);
                v[j4 * 8 + e * 2] *= d0; v[j4 * 8 + e * 2 + 1] *= d1;
            }
        }
    }
    uint4 out[4];
#pragma unroll
    for (int j4 = 0; j4 < 4; ++j4) {
        __nv_bfloat162 h[4];
#pragma unroll
        for (int e = 0; e < 4; ++e)
            h[e] = __floats2bfloat162_rn(apply_act(v[j4 * 8 + e * 2], act), apply_act(v[j4 * 8 + e * 2 + 1], act));
        out[j4] = *reinterpret_cast<uint4*>(h);
    }
    uint4* yp = reinterpret_cast<uint4*>(y + off);
#pragma unroll
    for (int j4 = 0; j4 < 4; ++j4) yp[j4] = out[j4];
    if (halo_right) {
        uint4* hp = reinterpret_cast<uint4*>(y + off + halo_elems);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) hp[j4] = out[j4];
    }
    if (halo_left) {
        uint4* hp = reinterpret_cast<uint4*>(y + off - halo_elems);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) hp[j4] = out[j4];
    }
}

__device__ __forceinline__ void epilogue_store32(float (&v)[32], const __nv_bfloat16* __restrict__ residual,
                                                 const __nv_bfloat16* __restrict__ saved, __nv_bfloat16* __restrict__ y,
                                                 size_t off, int act, bool halo_right, bool halo_left, size_t halo_elems) {
    if (residual) {
        const uint4* rp = reinterpret_cast<const uint4*>(residual + off);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
            const uint4 rv = __ldg(rp + j4);
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&rv);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __bfloat1622float2(h[e]);
                v[j4 * 8 + e * 2] += f.x; v[j4 * 8 + e * 2 + 1] += f.y;
            }
        }
    }
    if (act >= 3) {
        const uint4* sp = reinterpret_cast<const uint4*>(saved + off);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
            const uint4 sv = __ldg(sp + j4);
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&sv);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 a = __bfloat1622float2(h[e]);
                const float d0 = (act == 3) ? fmaf(-a.x, a.x, 1.0f) : (a.x > 0.0f ? 1.0f : 0.0f);
                const float d1 = (act == 3) ? fmaf(-a.y, a.y, 1.0f) : (a.y > 0.0f ? 1.0f : 0.0f);
                v[j4 * 8 + e * 2] *= d0; v[j4 * 8 + e * 2 + 1] *= d1;
            }
        }
    }
    uint4 out[4];
#pragma unroll
    for (int j4 = 0; j4 < 4; ++j4) {
        __nv_bfloat162 h[4];
#pragma unroll
        for (int e = 0; e < 4; ++e)
            h[e] = __floats2bfloat162_rn(apply_act(v[j4 * 8 + e * 2], act), apply_act(v[j4 * 8 + e * 2 + 1], act));
        out[j4] = *reinterpret_cast<uint4*>(h);
    }
    uint4* yp = reinterpret_cast<uint4*>(y + off);
#pragma unroll
    for (int j4 = 0; j4 < 4; ++j4) yp[j4] = out[j4];
    if (halo_right) {
        uint4* hp = reinterpret_cast<uint4*>(y + off + halo_elems);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) hp[j4] = out[j4];
    }
    if (halo_left) {
        uint4* hp = reinterpret_cast<uint4*>(y + off - halo_elems);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) hp[j4] = out[j4];
    }
}

}  // namespace delora
