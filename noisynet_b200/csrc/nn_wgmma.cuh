// PTX wrappers shared by the tensor-core kernels (sm_90a): mbarrier, bulk / tensor-map TMA copies, warpgroup MMA
// (wgmma) with shared-memory matrix descriptors, and the fp32 accumulator tile that hands a warpgroup's wgmma
// fragments to epilogue threads that own one output row each.  Every mbarrier wait is bounded by a clock64 watchdog;
// a kernel whose watchdog fires records a code and traps (nn_pipeline_abort).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

namespace {

constexpr long long UM_TIMEOUT = 4000000000LL;       // ~2 s of SM clocks

// A pipeline watchdog fired (a barrier did not complete within UM_TIMEOUT clocks): record the code and TRAP.  The
// accumulators are incomplete, so letting the epilogue and the optimizer run on them would silently corrupt the
// model; the trap turns the failure into a launch error that the next CUDA call of the process reports, and the code
// stays readable through nn_debug_error_flag.  (No printf: a function call anywhere in a kernel makes ptxas serialize
// every wgmma of it.)
__device__ __forceinline__ void nn_pipeline_abort(int* err_flag, int code) {
    if (err_flag) atomicExch(err_flag, code);
    __threadfence_system();
    __trap();
}

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok;
}
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return true;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > UM_TIMEOUT) return false;
    }
    return true;
}
// waiting roles that are not on the critical path (producers waiting for a free stage): sleep between polls instead of
// competing with the MMA warpgroups for issue slots and the barrier unit
__device__ __forceinline__ bool mbar_wait_backoff(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return true;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        __nanosleep(64);
        if (clock64() - t0 > UM_TIMEOUT) return false;
    }
    return true;
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void st_global_f32(float* ptr, float v) {
    asm volatile("st.global.f32 [%0], %1;" ::"l"(ptr), "f"(v) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// im2col-mode tensor-map copy (cuTensorMapEncodeIm2col): `pixelsPerColumn` output pixels x `channelsPerPixel` channels
// of one filter tap land as rows of the swizzled K-major tile.  Coordinates: first channel, then the INPUT position of
// the tile's first output pixel for tap (0, 0) -- (ow * stride - pad, oh * stride - pad, image) -- and the tap as offsets.
__device__ __forceinline__ void tma_im2col_4d(uint32_t dst, const void* map, uint32_t bar, int c, int w, int h, int n,
                                              uint16_t off_w, uint16_t off_h) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h) : "memory");
}
__device__ __forceinline__ void tma_tile_2d(uint32_t dst, const void* map, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// One lane of a CONVERGED warp.  The single-thread instructions of this file (TMA copies, barrier arrivals) take
// their operands from uniform registers; issued under `if (lane == 0)` inside divergent code the compiler cannot prove the
// operands warp-uniform and moves every one of them through R2UR in an ELECT loop on each use (5 per MMA, ~250 cycles per
// copy).  Role loops therefore run on the whole warp with warp-uniform control flow and elect the issuing lane.
__device__ __forceinline__ bool elect_one_sync() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xFFFFFFFF;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void tma_prefetch_desc(const void* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ------------------------------------------------------------------ shared-memory matrix descriptors (wgmma)
// start address, leading / stride byte offsets (16-byte units), layout: 0 none (core matrices of 8 rows x 16 B),
// 1 SWIZZLE_128B, 2 SWIZZLE_64B, 3 SWIZZLE_32B.  Only the 14-bit start field changes between stages and k-steps, so
// issue loops add to a descriptor template.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_units, uint32_t sbo_units, uint32_t layout) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | ((uint64_t)(lbo_units & 0x3FFFu) << 16) |
           ((uint64_t)(sbo_units & 0x3FFFu) << 32) | ((uint64_t)layout << 62);
}
// K-major tile whose rows are `sw_bytes` (32 / 64 / 128) wide, 8-row atoms of 8 * sw_bytes: advancing 16 bf16 along K
// = +32 bytes = +2 units inside a row
__device__ __forceinline__ uint64_t gmma_desc_kmajor(uint32_t smem_addr, uint32_t sw_bytes) {
    return gmma_desc(smem_addr, 1u, (8u * sw_bytes) >> 4, sw_bytes == 128u ? 1u : (sw_bytes == 64u ? 2u : 3u));
}
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) { return gmma_desc_kmajor(smem_addr, 128u); }
// SWIZZLE_NONE: K-major -- lbo = distance between the two 8-column K halves of one MMA, sbo = between 8-row groups;
// MN-major -- lbo = between 8-row reduction groups, sbo = between 8-element MN atoms
__device__ __forceinline__ uint64_t gmma_desc_none(uint32_t smem_addr, uint32_t lbo_units, uint32_t sbo_units) {
    return gmma_desc(smem_addr, lbo_units, sbo_units, 0u);
}

// ------------------------------------------------------------------ warpgroup MMA: D[64 x N] (+)= A[64 x 16] B[16 x N]
// bf16 operands from shared memory, fp32 accumulators in registers.  TA / TB = 1: the operand is MN-major.
// Fragment of thread t of the warpgroup (warp w = t / 32, lane l): register 4 i + j holds row 16 w + l / 4 + 8 (j / 2),
// column 8 i + 2 (l % 4) + j % 2 -- the first N / 2 registers of a wider fragment are the narrower one.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wg_fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_n8(float* d, uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0,%1,%2,%3}, %4, %5, p, 1, 1, %7, %8;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float* d, uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n24(float* d, uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %14, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n24k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11}, %12, %13, p, 1, 1, %15, %16;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n40(float* d, uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %22, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n40k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19}, %20, %21, p, 1, 1, %23, %24;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n48(float* d, uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, %27, %28;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n56(float* d, uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %30, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n56k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27}, %28, %29, p, 1, 1, %31, %32;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}

// one wgmma of compile-time width N
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_c(float* d, uint64_t a, uint64_t b, int scale_d) {
    static_assert(N % 8 == 0 && N >= 8 && N <= 64, "wgmma_c: N = 8 .. 64");
    if constexpr (N == 64) wgmma_n64<TA, TB>(d, a, b, scale_d);
    else if constexpr (N == 56) wgmma_n56<TA, TB>(d, a, b, scale_d);
    else if constexpr (N == 48) wgmma_n48<TA, TB>(d, a, b, scale_d);
    else if constexpr (N == 40) wgmma_n40<TA, TB>(d, a, b, scale_d);
    else if constexpr (N == 32) wgmma_n32<TA, TB>(d, a, b, scale_d);
    else if constexpr (N == 24) wgmma_n24<TA, TB>(d, a, b, scale_d);
    else if constexpr (N == 16) wgmma_n16<TA, TB>(d, a, b, scale_d);
    else wgmma_n8<TA, TB>(d, a, b, scale_d);
}
// one wgmma of runtime width n (a multiple of 8, <= 64) into the chunk registers d[32]
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n(float* d, uint64_t a, uint64_t b, int n, int scale_d) {
    if (n >= 64) wgmma_n64<TA, TB>(d, a, b, scale_d);
    else if (n == 56) wgmma_n56<TA, TB>(d, a, b, scale_d);
    else if (n == 48) wgmma_n48<TA, TB>(d, a, b, scale_d);
    else if (n == 40) wgmma_n40<TA, TB>(d, a, b, scale_d);
    else if (n == 32) wgmma_n32<TA, TB>(d, a, b, scale_d);
    else if (n == 24) wgmma_n24<TA, TB>(d, a, b, scale_d);
    else if (n == 16) wgmma_n16<TA, TB>(d, a, b, scale_d);
    else if (n == 8) wgmma_n8<TA, TB>(d, a, b, scale_d);
}
// D[64 x n] (+)= A B for n <= 64 NCH: one wgmma per 64-column chunk, the chunks' B operands `b_step` descriptor units apart
template <int NCH, int TA, int TB>
__device__ __forceinline__ void wg_mma(float (&acc)[NCH][32], uint64_t ad, uint64_t bd, uint32_t b_step, int n, int scale_d) {
#pragma unroll
    for (int c = 0; c < NCH; ++c)
        if (n > 64 * c) wgmma_n<TA, TB>(acc[c], ad, bd + (uint64_t)(c * b_step), n - 64 * c, scale_d);
}
template <int NCH>
__device__ __forceinline__ void wg_fence_acc(float (&acc)[NCH][32]) {
#pragma unroll
    for (int c = 0; c < NCH; ++c) wg_fence_regs<32>(acc[c]);
}

// ------------------------------------------------------------------ fp32 accumulator tile in shared memory
// Row r of a 128-row tile at p + r * stride floats (stride % 8 == 4: the float4 reads of 8 consecutive rows and the
// float2 fragment writes spread over the banks).  Epilogue threads own one row each; the "address" of a read is
// (first row of the warp << 16) | column, and lane l of the warp reads row (first row + l).
struct AccTile {
    float* p;
    int stride;
};
__device__ __forceinline__ const float* acc_at(const AccTile& t, uint32_t taddr) {
    return t.p + (size_t)((taddr >> 16) + (threadIdx.x & 31u)) * t.stride + (taddr & 0xFFFFu);
}
__device__ __forceinline__ void acc_ld4(const AccTile& t, uint32_t taddr, float v[4]) {
    const float4 a = *reinterpret_cast<const float4*>(acc_at(t, taddr));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}
__device__ __forceinline__ void acc_ld16(const AccTile& t, uint32_t taddr, float v[16]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) acc_ld4(t, taddr + 4u * i, v + 4 * i);
}
__device__ __forceinline__ void acc_ld4x2(const AccTile& t, uint32_t ta, uint32_t tb, float a[4], float b[4]) {
    acc_ld4(t, ta, a); acc_ld4(t, tb, b);
}
__device__ __forceinline__ void acc_ld4x4(const AccTile& t, uint32_t ta, uint32_t tb, uint32_t tc, uint32_t td, float a[4], float b[4],
                                          float c[4], float d[4]) {
    acc_ld4(t, ta, a); acc_ld4(t, tb, b); acc_ld4(t, tc, c); acc_ld4(t, td, d);
}
// a warpgroup's fragments of rows row0 .. row0 + 63, columns col0 .. col0 + n - 1, into the tile
template <int NCH>
__device__ __forceinline__ void wg_acc_store(const float (&acc)[NCH][32], const AccTile& t, int row0, int col0, int n) {
    const int wt = threadIdx.x & 127, l = wt & 31;
    float* r0 = t.p + (size_t)(row0 + 16 * (wt >> 5) + (l >> 2)) * t.stride + col0 + 2 * (l & 3);
    float* r1 = r0 + 8 * t.stride;
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (64 * c + 8 * i < n) {
                *reinterpret_cast<float2*>(r0 + 64 * c + 8 * i) = make_float2(acc[c][4 * i], acc[c][4 * i + 1]);
                *reinterpret_cast<float2*>(r1 + 64 * c + 8 * i) = make_float2(acc[c][4 * i + 2], acc[c][4 * i + 3]);
            }
        }
}

}  // namespace
