// Gradient all-reduce over NVLink 5 / NVSwitch peer memory (SURVEY section 8e: one exchange per step = the SUM of the
// parameter gradients over the data-parallel ranks, main.py:786-802), written against SYMMETRIC memory instead of a
// library collective: every rank's flat gradient buffer sits at the same offset of a buffer that all ranks have mapped
// (peer pointers) and that the switch exposes as one multicast address.
//
//   two-shot, in place:  rank r owns slice r of the range.  For each 16-byte vector of its slice it issues ONE
//   multimem.ld_reduce (the switch reads the vector from all ranks and returns the sum: NVLS in-switch reduction) and ONE
//   multimem.st (the switch writes the sum back into every rank's buffer).  Per GPU 2 * n / world floats cross the link.
//   No rank reads an element after another rank may have overwritten it: element e is read and written by its owner only.
//
// Cross-GPU ordering uses monotonically increasing epoch flags in the same symmetric buffer (no reset races):
//   A: "my gradients of this bucket are complete"  (every rank -> every rank, before any ld_reduce)
//   B: "my slice has been written everywhere"      (every rank -> every rank, before the optimizer reads the sums)
// nn_allreduce_wait (1 warp) waits for B and advances the epoch; it is launched on the stream that consumes the sums, so
// the reduction itself can run on a side stream under the backward pass (CUDA-graph capturable, no host involvement).
// Without a multicast mapping the same schedule runs on plain peer loads / stores (8 loads + 8 stores per vector).
#include "nn_common.cuh"

namespace {

constexpr int AR_MAX_WORLD = 16;
constexpr int AR_MAX_BUCKETS = 8;
constexpr long long AR_TIMEOUT = 20000000000LL;          // ~10 s of SM clocks

struct ArP {
    unsigned long long peer_base[AR_MAX_WORLD];           // every rank's mapping of the symmetric buffer (this rank's view)
    unsigned long long mc_base;                           // multicast mapping of the same buffer (0: none)
    int rank, world, bucket;
    long long data_off;                                   // byte offset of the gradient range inside the buffer
    long long n_vec;                                      // float4 vectors in the range (multiple of world)
};

// control block at the start of every rank's symmetric buffer
struct ArCtl {
    unsigned int flag_a[AR_MAX_BUCKETS][AR_MAX_WORLD];
    unsigned int flag_b[AR_MAX_BUCKETS][AR_MAX_WORLD];
    unsigned int epoch[AR_MAX_BUCKETS];                   // local: completed exchanges of the bucket
    unsigned int done_ctas[AR_MAX_BUCKETS];               // local: CTAs of the running kernel that have finished their stores
};

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 mc_ld_reduce(const void* mc) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
    return v;
}
__device__ __forceinline__ void mc_st(void* mc, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 peer_ld(const void* p) {
    float4 v;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void peer_st(void* p, float4 v) {
    asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__device__ __forceinline__ bool wait_flags(const unsigned int* flags, int world, unsigned int target) {
    // lanes 0..world-1 of the calling warp poll one flag each
    const int lane = threadIdx.x & 31;
    bool ok = true;
    if (lane < world) {
        const long long t0 = clock64();
        while ((int)(ld_acquire_sys(flags + lane) - target) < 0) {
            if (clock64() - t0 > AR_TIMEOUT) { ok = false; break; }
        }
    }
    return __all_sync(0xffffffffu, ok);
}

__global__ void __launch_bounds__(512)
k_allreduce_twoshot(const ArP p) {
    ArCtl* const ctl = reinterpret_cast<ArCtl*>(p.peer_base[p.rank]);
    const unsigned int target = ctl->epoch[p.bucket] + 1u;        // stable for the whole launch (nn_allreduce_wait advances it)
    // ---- A: every rank's gradients of this bucket are complete (they were written by earlier kernels of its stream)
    if (blockIdx.x == 0 && threadIdx.x < p.world) {
        __threadfence_system();
        ArCtl* peer = reinterpret_cast<ArCtl*>(p.peer_base[threadIdx.x]);
        st_release_sys(&peer->flag_a[p.bucket][p.rank], target);
    }
    if (threadIdx.x < 32) {
        if (!wait_flags(ctl->flag_a[p.bucket], p.world, target)) {
            if (threadIdx.x == 0) printf("noisynet_b200: gradient all-reduce timed out waiting for the peers (rank %d, bucket %d)\n", p.rank, p.bucket);
            __trap();
        }
    }
    __syncthreads();
    // ---- reduce my slice, broadcast the sums
    const long long per = p.n_vec / p.world, v0 = (long long)p.rank * per;
    if (p.mc_base) {
        // four independent switch round trips in flight per thread: the loop is bound by the ld_reduce latency (~2-3 us), not
        // by bandwidth
        char* mc = reinterpret_cast<char*>(p.mc_base) + p.data_off + v0 * 16;
        const long long stride = (long long)gridDim.x * blockDim.x;
        long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
        for (; i + 3 * stride < per; i += 4 * stride) {
            const float4 s0 = mc_ld_reduce(mc + i * 16), s1 = mc_ld_reduce(mc + (i + stride) * 16);
            const float4 s2 = mc_ld_reduce(mc + (i + 2 * stride) * 16), s3 = mc_ld_reduce(mc + (i + 3 * stride) * 16);
            mc_st(mc + i * 16, s0); mc_st(mc + (i + stride) * 16, s1);
            mc_st(mc + (i + 2 * stride) * 16, s2); mc_st(mc + (i + 3 * stride) * 16, s3);
        }
        for (; i < per; i += stride) {
            const float4 s0 = mc_ld_reduce(mc + i * 16);
            mc_st(mc + i * 16, s0);
        }
    } else {
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < per; i += (long long)gridDim.x * blockDim.x) {
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < p.world; ++r) {       // fixed rank order: every rank computes bit-identical sums
                const float4 v = peer_ld(reinterpret_cast<const char*>(p.peer_base[r]) + p.data_off + (v0 + i) * 16);
                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
            }
            for (int r = 0; r < p.world; ++r) peer_st(reinterpret_cast<char*>(p.peer_base[r]) + p.data_off + (v0 + i) * 16, s);
        }
    }
    // ---- B: my slice has landed everywhere (the last CTA of this launch tells every rank)
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        if (atomicAdd(&ctl->done_ctas[p.bucket], 1u) == gridDim.x - 1) {
            ctl->done_ctas[p.bucket] = 0u;
            __threadfence_system();
            for (int r = 0; r < p.world; ++r) st_release_sys(&reinterpret_cast<ArCtl*>(p.peer_base[r])->flag_b[p.bucket][p.rank], target);
        }
    }
}

__global__ void k_allreduce_wait(unsigned long long local_base, int world, int bucket) {
    ArCtl* const ctl = reinterpret_cast<ArCtl*>(local_base);
    const unsigned int target = ctl->epoch[bucket] + 1u;
    if (!wait_flags(ctl->flag_b[bucket], world, target)) {
        if (threadIdx.x == 0) printf("noisynet_b200: gradient all-reduce timed out waiting for the reduced slices (bucket %d)\n", bucket);
        __trap();
    }
    __syncwarp();
    if (threadIdx.x == 0) { ctl->epoch[bucket] = target; __threadfence(); }
}

}  // namespace

extern "C" int64_t nn_allreduce_ctl_bytes(void) { return (int64_t)((sizeof(ArCtl) + 1023) / 1024 * 1024); }

// SUM all-reduce, in place, of `count` floats at byte offset `data_off` of the symmetric buffer (count * 4 a multiple of
// 16 * world; data_off a multiple of 16).  peer_ptrs[world]: this process's mappings of every rank's buffer (own included);
// mc_ptr: multicast mapping or NULL.  The buffers start with nn_allreduce_ctl_bytes() of zero-initialised control words.
// Enqueues the exchange on `stream`; the sums are complete on a stream once nn_allreduce_wait has run there.
extern "C" int nn_allreduce_start(const void* const* peer_ptrs, const void* mc_ptr, int rank, int world, int bucket, int64_t data_off,
                                  int64_t count, int ctas, int device, void* stream) {
    if (!peer_ptrs || world < 2 || world > AR_MAX_WORLD || rank < 0 || rank >= world || bucket < 0 || bucket >= AR_MAX_BUCKETS)
        return nn_fail("nn_allreduce_start: bad arguments%s", "");
    if ((count * 4) % (16 * world) || data_off % 16 || data_off < nn_allreduce_ctl_bytes())
        return nn_fail("nn_allreduce_start: the range must be a multiple of 16 * world bytes behind the control block%s", "");
    NN_SET_DEVICE(device);
    ArP p;
    memset(&p, 0, sizeof(p));
    for (int r = 0; r < world; ++r) p.peer_base[r] = (unsigned long long)(uintptr_t)peer_ptrs[r];
    p.mc_base = (unsigned long long)(uintptr_t)mc_ptr;
    p.rank = rank; p.world = world; p.bucket = bucket; p.data_off = data_off; p.n_vec = count / 4;
    if (ctas < 1) ctas = 32;
    const long long per = p.n_vec / world;
    if ((long long)ctas * 512 * 2 > per) ctas = (int)((per + 1023) / 1024);      // at least two vectors per thread
    if (ctas < 1) ctas = 1;
    k_allreduce_twoshot<<<ctas, 512, 0, (cudaStream_t)stream>>>(p);
    NN_LAUNCH_OK();
    return 0;
}

extern "C" int nn_allreduce_wait(const void* local_ptr, int world, int bucket, int device, void* stream) {
    if (!local_ptr || world < 2 || world > AR_MAX_WORLD || bucket < 0 || bucket >= AR_MAX_BUCKETS)
        return nn_fail("nn_allreduce_wait: bad arguments%s", "");
    NN_SET_DEVICE(device);
    k_allreduce_wait<<<1, 32, 0, (cudaStream_t)stream>>>((unsigned long long)(uintptr_t)local_ptr, world, bucket);
    NN_LAUNCH_OK();
    return 0;
}
