// Stable LSD radix sort of each scan's points by fp32 range (sm_90a).
//
// The reference orders the cloud with `torch.argsort(range)` (src/utility/projection.py:63-67)
// and returns (u, v) and the surviving point indices in that order (:105-106).  The projection
// itself does not need the order (see projection.cu); this sort exists so that the drop-in
// ImageProjectionLayer can hand back the reference-shaped, range-ordered outputs.  Stable LSD
// passes over the 32 bits of sort_key_bits leave equal ranges in index order, i.e. the deterministic
// version of the reference's unstable argsort: torch.argsort(range, stable=True), on any fp32 keys.
//
// Per 8-bit pass: tile histograms -> per-digit exclusive scan over tiles -> stable scatter
// (warp `match_any` ranking).  Integer work, bound by L2/HBM bandwidth: 16 B moved per key and pass.
#include "common.cuh"

namespace delora {

constexpr int kSortThreads = 256;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kSortItersPerWarp = 8;
constexpr int kSortTile = kSortThreads * kSortItersPerWarp;   // 2048 keys per block

// The radix key of a range, in torch.argsort's order: -0 is +0, every NaN (either sign, any payload) is one key above
// +inf, and the sign flip (negative: all bits inverted; otherwise: the sign bit set) makes the unsigned order the
// order of the values.  Both first passes read keys through here only.
__device__ __forceinline__ unsigned sort_key_bits(const float* __restrict__ rng, int i) {
    unsigned b = __float_as_uint(__ldg(rng + i));
    if ((b & 0x7fffffffu) > 0x7f800000u) return 0xffffffffu;
    if (b == 0x80000000u) b = 0u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

template <bool FIRST>
__global__ void __launch_bounds__(kSortThreads)
sort_hist_kernel(const float* __restrict__ rng, const unsigned* __restrict__ keys_in,
                 const int32_t* __restrict__ n_points, int n_stride, int shift, int ntiles,
                 int32_t* __restrict__ tile_hist) {
    __shared__ int hist[256];
    const int b = blockIdx.y, tile = blockIdx.x;
    const int n = n_points[b];
    hist[threadIdx.x] = 0;
    __syncthreads();
    const size_t off = (size_t)b * n_stride;
#pragma unroll
    for (int k = 0; k < kSortItersPerWarp; ++k) {
        const int i = tile * kSortTile + k * kSortThreads + threadIdx.x;
        if (i < n) {
            const unsigned key = FIRST ? sort_key_bits(rng + off, i) : keys_in[off + i];
            atomicAdd(&hist[(key >> shift) & 255u], 1);
        }
    }
    __syncthreads();
    tile_hist[((size_t)b * ntiles + tile) * 256 + threadIdx.x] = hist[threadIdx.x];
}

// one block per scan: exclusive offsets of (digit, tile) in digit-major order
__global__ void __launch_bounds__(256)
sort_scan_kernel(int32_t* __restrict__ tile_hist, int ntiles) {
    __shared__ int warp_tot[8];
    int32_t* __restrict__ h = tile_hist + (size_t)blockIdx.x * ntiles * 256;
    const int d = threadIdx.x;
    int running = 0;
    for (int t = 0; t < ntiles; ++t) {
        const int c = h[(size_t)t * 256 + d];
        h[(size_t)t * 256 + d] = running;
        running += c;
    }
    // exclusive scan of the digit totals across the 256 threads
    const int lane = d & 31, w = d >> 5;
    int inc = running;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) warp_tot[w] = inc;
    __syncthreads();
    int base = 0;
    for (int i = 0; i < w; ++i) base += warp_tot[i];
    const int digit_base = base + inc - running;
    for (int t = 0; t < ntiles; ++t) h[(size_t)t * 256 + d] += digit_base;
}

template <bool FIRST>
__global__ void __launch_bounds__(kSortThreads)
sort_scatter_kernel(const float* __restrict__ rng, const unsigned* __restrict__ keys_in,
                    const int32_t* __restrict__ idx_in, const int32_t* __restrict__ n_points, int n_stride,
                    int shift, int ntiles, const int32_t* __restrict__ tile_off, unsigned* __restrict__ keys_out,
                    int32_t* __restrict__ idx_out) {
    __shared__ int cnt[kSortWarps][256];
    const int b = blockIdx.y, tile = blockIdx.x;
    const int n = n_points[b];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const size_t off = (size_t)b * n_stride;
    for (int i = threadIdx.x; i < kSortWarps * 256; i += kSortThreads) (&cnt[0][0])[i] = 0;
    __syncthreads();
    // warp w owns the contiguous keys [tile*TILE + w*256, +256), 32 at a time, in order
    unsigned key[kSortItersPerWarp];
    int idx[kSortItersPerWarp];
    const int wbase = tile * kSortTile + w * (32 * kSortItersPerWarp);
#pragma unroll
    for (int k = 0; k < kSortItersPerWarp; ++k) {
        const int i = wbase + k * 32 + lane;
        const bool ok = i < n;
        key[k] = ok ? (FIRST ? sort_key_bits(rng + off, i) : keys_in[off + i]) : 0u;
        idx[k] = ok ? (FIRST ? i : idx_in[off + i]) : -1;
    }
    const unsigned lt = (1u << lane) - 1u;
#pragma unroll
    for (int k = 0; k < kSortItersPerWarp; ++k) {
        const bool ok = idx[k] >= 0;
        const int d = ok ? (int)((key[k] >> shift) & 255u) : 256 + lane;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        if (ok && (peers & lt) == 0u) cnt[w][d] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    {
        const int d = threadIdx.x;
        int base = tile_off[((size_t)b * ntiles + tile) * 256 + d];
#pragma unroll
        for (int j = 0; j < kSortWarps; ++j) {
            const int c = cnt[j][d];
            cnt[j][d] = base;
            base += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kSortItersPerWarp; ++k) {
        const bool ok = idx[k] >= 0;
        const int d = ok ? (int)((key[k] >> shift) & 255u) : 256 + lane;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        if (ok) {
            const int pos = cnt[w][d] + __popc(peers & lt);
            keys_out[off + pos] = key[k];
            idx_out[off + pos] = idx[k];
        }
        __syncwarp();
        if (ok && (peers & lt) == 0u) cnt[w][d] += __popc(peers);
        __syncwarp();
    }
}

}  // namespace delora

using namespace delora;

static inline int sort_tiles(int n_stride) { return (n_stride + kSortTile - 1) / kSortTile; }
static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" int64_t delora_sort_scratch_bytes(int B, int n_stride) {
    const size_t arr = align256(sizeof(uint32_t) * (size_t)B * n_stride);
    const size_t hist = align256(sizeof(int32_t) * (size_t)B * sort_tiles(n_stride) * 256);
    return (int64_t)(3 * arr + hist);
}

extern "C" int delora_sort_by_range(const float* range, const int32_t* n_points, int B, int n_stride,
                                    int32_t* order, void* scratch, void* stream) {
    DELORA_CHECK_ARG(range && n_points && order && scratch, "delora_sort_by_range: null pointer");
    DELORA_CHECK_ARG(B > 0 && B <= 65535 && n_stride > 0, "delora_sort_by_range: bad shape");
    const size_t arr = align256(sizeof(uint32_t) * (size_t)B * n_stride);
    char* base = (char*)scratch;
    unsigned* keys_a = (unsigned*)base;
    unsigned* keys_b = (unsigned*)(base + arr);
    int32_t* idx_b = (int32_t*)(base + 2 * arr);
    int32_t* hist = (int32_t*)(base + 3 * arr);
    const int ntiles = sort_tiles(n_stride);
    dim3 grid(ntiles, B);
    cudaStream_t st = (cudaStream_t)stream;
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 8 * pass;
        const unsigned* kin = (pass & 1) ? keys_b : keys_a;
        const int32_t* iin = (pass & 1) ? idx_b : order;
        unsigned* kout = (pass & 1) ? keys_a : keys_b;
        int32_t* iout = (pass & 1) ? order : idx_b;
        if (pass == 0) {
            sort_hist_kernel<true><<<grid, kSortThreads, 0, st>>>(range, nullptr, n_points, n_stride, shift, ntiles, hist);
        } else {
            sort_hist_kernel<false><<<grid, kSortThreads, 0, st>>>(range, kin, n_points, n_stride, shift, ntiles, hist);
        }
        DELORA_CHECK_LAUNCH("sort_hist_kernel");
        sort_scan_kernel<<<B, 256, 0, st>>>(hist, ntiles);
        DELORA_CHECK_LAUNCH("sort_scan_kernel");
        if (pass == 0) {
            sort_scatter_kernel<true><<<grid, kSortThreads, 0, st>>>(range, nullptr, nullptr, n_points, n_stride, shift,
                                                                     ntiles, hist, kout, iout);
        } else {
            sort_scatter_kernel<false><<<grid, kSortThreads, 0, st>>>(range, kin, iin, n_points, n_stride, shift,
                                                                      ntiles, hist, kout, iout);
        }
        DELORA_CHECK_LAUNCH("sort_scatter_kernel");
    }
    return 0;
}
