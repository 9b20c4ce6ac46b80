// Gradient all-reduce over NVLink / NVSwitch peer memory for the data-parallel training step (sm_90a).
//
// SURVEY.md 8(e): the reference is single-process (src/deploy/trainer.py:23-24 steps one optimizer on one
// device); the data-parallel step averages the weight gradients of equal per-rank batches, which reproduces
// the reference's `loss / batch_size` (src/deploy/deployer.py:329-342) over the global batch.
//
// Why not NCCL here: the row-block convolution kernels are persistent, one 320-thread CTA with ~226 KB of shared
// memory per SM.  An NCCL CTA (640 threads, tens of KB of shared memory) cannot share an SM with them, so a
// collective issued during the backward only runs in the gaps between convolution kernels and then delays the next
// one.  This kernel is built
// to be CO-RESIDENT with them instead: 128 threads, no shared memory, < 64 registers, so its CTAs are placed next
// to the running convolution CTAs and the reduction proceeds while the backward continues.
//
// Data path (every gradient lives in ONE flat fp32 buffer that is symmetric memory, i.e. mapped at every peer and,
// where the fabric offers it, bound to an NVSwitch multicast object):
//   rank r owns elements [r * per, (r + 1) * per) of the bucket.
//   multicast:  v = multimem.ld_reduce.add.v4.f32 [mc + i]   -- the switch adds the 8 copies in flight
//               multimem.st.v4.f32 [mc + i] = v * scale       -- and writes the average back to all 8
//   peer (no multicast):  v = sum over ranks q (fixed order) of ld [peer_q + i];  st [peer_q + i] = v * scale
// so every element crosses the links once in each direction and all ranks end up with bit-identical averages.
// Ordering between ranks: one flag word per (phase, CTA, source rank) in symmetric memory, written with
// st.release.sys and polled with ld.acquire.sys; CTA c of every rank synchronises only with CTA c of the peers
// (start: all gradients of the bucket are written; end: all slices are stored), monotonically increasing
// sequence numbers, no reset.  A wait that exceeds kArTimeoutNs sets *status and carries on: a lost peer shows
// up as an error on the host, never as a hung GPU.
//
// Sequence numbers: delora_grad_allreduce_f32 takes `seq` from the host.  The group training step
// (delora_odometry_train_step_group) launches the device-seq variant instead, which reads a step counter in device
// memory at the start of the kernel, seq = step * seq_stride + seq_add: a CUDA graph that captured it replays a new
// number every step, where a captured host value would repeat and every wait after the first replay would pass at once.
#include "common.cuh"

namespace delora {

static_assert(kArMaxWorld == DELORA_GRAD_ALLREDUCE_MAX_WORLD, "the header's world limit is the kernel's");
constexpr unsigned long long kArTimeoutNs = 20ull * 1000ull * 1000ull * 1000ull;

struct ArParams {
    unsigned long long peer_buf[kArMaxWorld];     // unicast address of the flat buffer at every rank
    unsigned long long peer_flag[kArMaxWorld];    // unicast address of the flag words at every rank
    float* mc;                                    // multicast address of the flat buffer (nullptr: peer path)
    int rank, world;
    long long off, count;                         // bucket = elements [off, off + count) of the flat buffer
    float scale;
    unsigned seq;                                 // the host's sequence number, or seq_add of the device-seq variant
    const long long* seq_step;                    // device-seq variant: seq = *seq_step * seq_stride + seq
    unsigned seq_stride;
    int* status;
};

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 multimem_ld_reduce_add(const float4* p) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void multimem_st(float4* p, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
                 ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 ld_relaxed_sys(const float4* p) {
    float4 v;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys(float4* p, float4 v) {
    asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
                 ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Flag word of (phase, cta, source rank) inside one rank's flag array.
__device__ __forceinline__ int ar_flag_index(int phase, int cta, int src) {
    return (phase * kArMaxCtas + cta) * kArMaxWorld + src;
}

// All ranks' CTA `cta` meet: thread q tells rank q "rank `rank` reached `seq`", then waits for rank q's word here.
__device__ __forceinline__ void ar_meet(const ArParams& p, unsigned seq, int phase, int cta) {
    const int q = threadIdx.x;
    if (q < p.world) {
        unsigned* theirs = reinterpret_cast<unsigned*>(p.peer_flag[q]) + ar_flag_index(phase, cta, p.rank);
        st_release_sys(theirs, seq);
        const unsigned* mine = reinterpret_cast<const unsigned*>(p.peer_flag[p.rank]) + ar_flag_index(phase, cta, q);
        const unsigned long long t0 = global_timer_ns();
        while ((int)(ld_acquire_sys(mine) - seq) < 0) {
            if (global_timer_ns() - t0 > kArTimeoutNs) { atomicExch(p.status, 1 + q); break; }
            __nanosleep(64);
        }
    }
    __syncthreads();
}

template <bool MC, bool kDevSeq>
__global__ void __launch_bounds__(kArMaxThreads)
grad_allreduce_kernel(ArParams p) {
    const int cta = blockIdx.x;
    const unsigned seq = kDevSeq ? (unsigned)*p.seq_step * p.seq_stride + p.seq : p.seq;
    ar_meet(p, seq, 0, cta);                                        // every rank's bucket is complete

    const long long n4 = p.count >> 2;
    const long long per = (n4 + p.world - 1) / p.world;
    const long long lo = (p.off >> 2) + (long long)p.rank * per;
    const long long hi_raw = (p.off >> 2) + ((long long)(p.rank + 1) * per < n4 ? (long long)(p.rank + 1) * per : n4);
    const long long hi = hi_raw > lo ? hi_raw : lo;
    constexpr int U = 4;                                            // independent 16-byte requests in flight per thread
    const int nt = blockDim.x;
    const long long step = (long long)gridDim.x * nt * U;
    for (long long i0 = lo + (long long)cta * nt * U + threadIdx.x; i0 < hi; i0 += step) {
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long i = i0 + (long long)u * nt;
            if (i < hi) {
                if (MC) {
                    v[u] = multimem_ld_reduce_add(reinterpret_cast<const float4*>(p.mc) + i);
                } else {
                    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
                    for (int q = 0; q < p.world; ++q) {
                        const float4 t = ld_relaxed_sys(reinterpret_cast<const float4*>(p.peer_buf[q]) + i);
                        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
                    }
                    v[u] = s;
                }
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long i = i0 + (long long)u * nt;
            if (i < hi) {
                const float4 o = make_float4(v[u].x * p.scale, v[u].y * p.scale, v[u].z * p.scale, v[u].w * p.scale);
                if (MC) {
                    multimem_st(reinterpret_cast<float4*>(p.mc) + i, o);
                } else {
                    for (int q = 0; q < p.world; ++q) st_relaxed_sys(reinterpret_cast<float4*>(p.peer_buf[q]) + i, o);
                }
            }
        }
    }
    __threadfence_system();                                         // this thread's stores before the CTA's flag
    __syncthreads();
    ar_meet(p, seq, 1, cta);                                        // every rank's slice has landed everywhere
}

__device__ __forceinline__ void st_relaxed_sys(int* p, int v) {
    asm volatile("st.relaxed.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_relaxed_sys(const int* p) {
    int v;
    asm volatile("ld.relaxed.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// The adapting streams' valid-count exchange (delora_odometry_streams_push_adapt_group), one CTA.  p.peer_buf[q] is
// rank q's exchange slots, int32 [2][kArMaxWorld].  The tick counter advances to t; thread q stores this rank's count in
// slot [t & 1][rank] of rank q, before its flag store in ar_meet (CTA 0, phase 0, seq = t * seq_stride), whose release
// orders it; after the meet, thread q's acquire of rank q's flag makes rank q's count of tick t visible in this rank's
// slot [t & 1][q].  The counts are summed in rank order into *n_out.  The parity of t double-buffers the slots: a rank
// writes the slots of tick t + 2 only after passing the meet of tick t + 1, i.e. after every peer has finished the
// kernel of tick t, which read them.  A meet that times out sets *status and carries on with the slot as it is.
__global__ void __launch_bounds__(kArMaxThreads)
count_allreduce_kernel(ArParams p, long long* __restrict__ tick, const int32_t* __restrict__ n_local,
                       int32_t* __restrict__ n_out) {
    __shared__ int s_n[kArMaxWorld];
    const long long t = *tick + 1;
    const int par = (int)(t & 1);
    const int q = threadIdx.x;
    if (q < p.world) st_relaxed_sys(reinterpret_cast<int*>(p.peer_buf[q]) + par * kArMaxWorld + p.rank, *n_local);
    ar_meet(p, (unsigned)t * p.seq_stride, 0, 0);
    if (q < p.world) s_n[q] = ld_relaxed_sys(reinterpret_cast<const int*>(p.peer_buf[p.rank]) + par * kArMaxWorld + q);
    __syncthreads();
    if (q == 0) {
        int n = 0;
        for (int r = 0; r < p.world; ++r) n += s_n[r];
        *n_out = n;
        *tick = t;
    }
}

int count_allreduce_launch(const uint64_t* peer_slots, const uint64_t* peer_flags, int rank, int world,
                           unsigned seq_stride, long long* tick, const int32_t* n_local, int32_t* n_out, int32_t* status,
                           cudaStream_t st) {
    ArParams p;
    memset(&p, 0, sizeof(p));
    for (int q = 0; q < world; ++q) {
        p.peer_buf[q] = peer_slots[q];
        p.peer_flag[q] = peer_flags[q];
    }
    p.rank = rank; p.world = world; p.seq_stride = seq_stride; p.status = status;
    count_allreduce_kernel<<<1, kArMaxThreads, 0, st>>>(p, tick, n_local, n_out);
    DELORA_CHECK_LAUNCH("count_allreduce_kernel");
    return 0;
}

// Loads the collective kernels of a group tick on the current device now.  Under lazy module loading (CUDA's default)
// a kernel is loaded at its first launch, and the load waits for the kernels running on the device.  If that device
// runs a rank that spins in a meet while the peer it waits for is still to be enqueued by the same host thread, the
// load would hold both until the meet's timeout.
int collective_kernels_preload(const char* who) {
    cudaFuncAttributes a;
    cudaError_t e = cudaFuncGetAttributes(&a, count_allreduce_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&a, grad_allreduce_kernel<true, true>);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&a, grad_allreduce_kernel<false, true>);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

// Both entry points validate their arguments before they get here; count > 0.
int grad_allreduce_launch(const uint64_t* peer_bufs, const uint64_t* peer_flags, uint64_t multicast_ptr, int rank,
                          int world, long long offset, long long count, float scale, unsigned seq,
                          const long long* seq_step, unsigned seq_stride, int n_ctas, int n_threads, int32_t* status,
                          cudaStream_t st) {
    ArParams p;
    for (int q = 0; q < kArMaxWorld; ++q) {
        p.peer_buf[q] = q < world ? peer_bufs[q] : 0ull;
        p.peer_flag[q] = q < world ? peer_flags[q] : 0ull;
    }
    p.mc = reinterpret_cast<float*>(multicast_ptr);
    p.rank = rank; p.world = world; p.off = offset; p.count = count; p.scale = scale; p.seq = seq;
    p.seq_step = seq_step; p.seq_stride = seq_stride; p.status = status;
    if (seq_step) {
        if (p.mc)
            grad_allreduce_kernel<true, true><<<n_ctas, n_threads, 0, st>>>(p);
        else
            grad_allreduce_kernel<false, true><<<n_ctas, n_threads, 0, st>>>(p);
    } else if (p.mc) {
        grad_allreduce_kernel<true, false><<<n_ctas, n_threads, 0, st>>>(p);
    } else {
        grad_allreduce_kernel<false, false><<<n_ctas, n_threads, 0, st>>>(p);
    }
    DELORA_CHECK_LAUNCH("grad_allreduce_kernel");
    return 0;
}

}  // namespace delora

using namespace delora;

extern "C" int delora_grad_allreduce_flag_words(void) { return 2 * kArMaxCtas * kArMaxWorld; }

extern "C" int delora_grad_allreduce_f32(const uint64_t* peer_bufs, const uint64_t* peer_flags, uint64_t multicast_ptr,
                                         int rank, int world, long long offset, long long count, float scale,
                                         uint32_t seq, int n_ctas, int n_threads, int32_t* status, void* stream) {
    DELORA_CHECK_ARG(peer_bufs && peer_flags && status, "delora_grad_allreduce_f32: null pointer");
    DELORA_CHECK_ARG(world >= 1 && world <= kArMaxWorld && rank >= 0 && rank < world,
                     "delora_grad_allreduce_f32: bad rank %d / world %d (max %d)", rank, world, kArMaxWorld);
    DELORA_CHECK_ARG(offset >= 0 && count >= 0 && (offset & 3) == 0 && (count & 3) == 0,
                     "delora_grad_allreduce_f32: offset %lld / count %lld must be multiples of 4 floats", offset, count);
    DELORA_CHECK_ARG(n_ctas >= 1 && n_ctas <= kArMaxCtas, "delora_grad_allreduce_f32: n_ctas %d outside [1, %d]", n_ctas,
                     kArMaxCtas);
    DELORA_CHECK_ARG(n_threads >= 32 && n_threads <= kArMaxThreads && n_threads % 32 == 0,
                     "delora_grad_allreduce_f32: n_threads %d must be 32, 64, 96 or 128", n_threads);
    if (count == 0) return 0;
    for (int q = 0; q < world; ++q)
        DELORA_CHECK_ARG(peer_bufs[q] && peer_flags[q] && (peer_bufs[q] & 15) == 0,
                         "delora_grad_allreduce_f32: peer %d has a null or unaligned mapping", q);
    DELORA_CHECK_ARG((multicast_ptr & 15) == 0, "delora_grad_allreduce_f32: unaligned multicast address");
    return grad_allreduce_launch(peer_bufs, peer_flags, multicast_ptr, rank, world, offset, count, scale, seq, nullptr, 0,
                                 n_ctas, n_threads, status, (cudaStream_t)stream);
}
