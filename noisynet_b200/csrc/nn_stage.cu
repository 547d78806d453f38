// Between-layer stages of the NoisyNet step, fused (SURVEY.md section 8f.1):
//   conv stage : MaxPool2d(2,2) -> BatchNorm2d (batch statistics) -> ReLU -> clamp(max=act_max) -> 4-bit
//                quantize (stochastic rounding) -> NHWC bf16 code pack for the next tensor-core contraction
//                (noisynet.py:419-460, 483-520), and its backward (STE + clamp + ReLU masks, BN backward,
//                max-pool routing) emitting the NHWC bf16 gradient the wgrad/dgrad kernels consume.
//   fc stage   : BatchNorm1d -> ReLU -> clamp -> quantize -> pack (noisynet.py:540-569) and backward.
//   head       : BatchNorm1d(10) -> cross-entropy (mean) -> gradient (noisynet.py:594, :1278).
// All HBM-bound elementwise/reduction work; per-channel reductions use fixed-order partials (deterministic).
#include <cooperative_groups.h>
#include <cuda_bf16.h>

#include "nn_common.cuh"

namespace cg = cooperative_groups;

namespace {

#ifndef ST_CHUNK_FAST
#define ST_CHUNK_FAST 1   // thread index: 16-byte channel chunk fastest (coalesced NHWC stores) vs pixel fastest
#endif
constexpr int ST_SPLITS = 16;   // MAX batch slices per channel for the deterministic partial sums (gridDim.y <= ST_SPLITS)

// slices actually used: enough blocks to fill the GPU, but at least ~2048 elements per block (the fc stages have 512
// elements per channel: 16 slices of 32 elements are pure launch overhead)
static inline int stage_splits(int64_t per_channel) {
    int64_t s = per_channel / 2048;
    if (s < 1) s = 1;
    if (s > ST_SPLITS) s = ST_SPLITS;
    return (int)s;
}

__device__ __forceinline__ float quant_code(float v, float s, float qmax, float u) {
    // hardware_model.py:154-166 with min_value = 0: rne(clamp(v / s + u, 0, qmax))
    float t = __fadd_rn(__fdiv_rn(v, s), u);
    return rintf(fminf(fmaxf(t, 0.f), qmax));
}

// Scratch (nn_stage_scratch_bytes): one record per channel, [ST_SPLITS][2] double partial sums (slice s: sum, sum of
// squares) and then the channel's arrival counter, padded to 16 bytes.  Channel c's record lies at the same address
// whatever the calling stage's C, so stages of different widths can share one scratch: a wider stage's partials never
// cover a narrower stage's counters.
constexpr int ST_REC = ST_SPLITS * 2 + 2;       // doubles per channel record
__device__ __forceinline__ double* stage_rec(double* scratch, int c) { return scratch + (int64_t)c * ST_REC; }

// The per-channel reductions end in the LAST slice's block of each channel (a self-resetting arrival counter behind the
// partials): it adds the slices in fixed order -- deterministic whichever block happens to be last -- and writes the
// statistics, so no separate finalize launch sits on the step's critical path.
__device__ __forceinline__ bool stage_last_slice(double* rec, int slices) {
    unsigned* counter = reinterpret_cast<unsigned*>(rec + ST_SPLITS * 2);
    __threadfence();                                   // this block's partial is visible before its arrival
    const unsigned done = atomicAdd(counter, 1u);
    if (done != (unsigned)slices - 1u) return false;
    *counter = 0u;                                     // ready for the next launch that uses this scratch
    __threadfence();
    return true;
}

// ------------------------------------------------------------------ F1: 2x2 max pool + per-channel partial sums
// grid (C, slices); block 256.  y [B,C,OH,OW] -> pooled [B,C,PH,PW], argmax (0..3), partial sums in the channel records
__global__ void __launch_bounds__(256)
k_pool_stats(const float* __restrict__ y, float* __restrict__ pooled, uint8_t* __restrict__ amax, double* __restrict__ scratch,
             const BnFinP fin, int B, int C, int OH, int OW) {
    const int c = blockIdx.x, sp = blockIdx.y;
    if (c == 0 && sp == 0 && threadIdx.x == 0 && fin.xmax_out) *fin.xmax_out = 0.f;      // the pack kernel that follows maxes into it
    const int PH = OH >> 1, PW = OW >> 1, PHW = PH * PW;
    const int b0 = (int)((int64_t)B * sp / (int)gridDim.y), b1 = (int)((int64_t)B * (sp + 1) / (int)gridDim.y);
    const int n = (b1 - b0) * PHW;
    double s1 = 0.0, s2 = 0.0;
    // no divisions in the element loop (the kernel is issue-bound): (sample, position) advance incrementally and the
    // window origin of a position comes from a shared table
    __shared__ unsigned short s_org[1024];                     // 2*ph*OW + 2*pw for positions < 1024
    const bool tab = PHW <= 1024 && 2 * OH * OW < 65536;
    if (tab) {
        for (int r = threadIdx.x; r < PHW; r += blockDim.x) { const int ph = r / PW; s_org[r] = (unsigned short)(2 * ph * OW + 2 * (r - ph * PW)); }
        __syncthreads();
    }
    const unsigned step_b = blockDim.x / (unsigned)PHW, step_r = blockDim.x - step_b * (unsigned)PHW;
    unsigned bi = threadIdx.x / (unsigned)PHW, r = threadIdx.x - bi * (unsigned)PHW;
    for (unsigned i = threadIdx.x; i < (unsigned)n; i += blockDim.x) {
        const int b = b0 + (int)bi;
        unsigned org;
        if (tab) org = s_org[r];
        else { const unsigned ph = r / (unsigned)PW; org = 2 * ph * OW + 2 * (r - ph * (unsigned)PW); }
        const float* src = y + ((int64_t)b * C + c) * OH * OW + org;
        const float2 t0 = *reinterpret_cast<const float2*>(src);
        const float2 t1 = *reinterpret_cast<const float2*>(src + OW);
        float m = t0.x; int a = 0;
        if (t0.y > m) { m = t0.y; a = 1; }
        if (t1.x > m) { m = t1.x; a = 2; }
        if (t1.y > m) { m = t1.y; a = 3; }
        const int64_t o = ((int64_t)b * C + c) * PHW + r;
        pooled[o] = m;
        amax[o] = (uint8_t)a;
        bi += step_b; r += step_r;
        if (r >= (unsigned)PHW) { r -= (unsigned)PHW; ++bi; }
        s1 += m; s2 += (double)m * m;
    }
    __shared__ double sh[2][8];
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s1; sh[1][threadIdx.x >> 5] = s2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, b = 0;
        for (int w = 0; w < 8; ++w) { a += sh[0][w]; b += sh[1][w]; }
        double* rec = stage_rec(scratch, c);
        rec[sp * 2 + 0] = a;
        rec[sp * 2 + 1] = b;
        if (stage_last_slice(rec, (int)gridDim.y)) bn_finalize_channel(rec, (int)gridDim.y, 2, c, fin);
    }
}

// statistics only (fc stages / no pooling): x [B,C,HW]
__global__ void __launch_bounds__(256)
k_chan_stats(const float* __restrict__ x, double* __restrict__ scratch, const BnFinP fin, int B, int C, int HW) {
    const int c = blockIdx.x, sp = blockIdx.y;
    if (c == 0 && sp == 0 && threadIdx.x == 0 && fin.xmax_out) *fin.xmax_out = 0.f;
    const int b0 = (int)((int64_t)B * sp / (int)gridDim.y), b1 = (int)((int64_t)B * (sp + 1) / (int)gridDim.y);
    const int n = (b1 - b0) * HW;
    double s1 = 0.0, s2 = 0.0;
    const unsigned step_b = blockDim.x / (unsigned)HW, step_r = blockDim.x - step_b * (unsigned)HW;
    unsigned bi = threadIdx.x / (unsigned)HW, r = threadIdx.x - bi * (unsigned)HW;
    unsigned i = threadIdx.x;
    for (; i + 3 * blockDim.x < (unsigned)n; i += 4 * blockDim.x) {         // four loads in flight, sums in element order
        float m[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            m[k] = __ldg(x + ((int64_t)(b0 + (int)bi) * C + c) * HW + r);
            bi += step_b; r += step_r;
            if (r >= (unsigned)HW) { r -= (unsigned)HW; ++bi; }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) { s1 += m[k]; s2 += (double)m[k] * m[k]; }
    }
    for (; i < (unsigned)n; i += blockDim.x) {
        const int b = b0 + (int)bi;
        const float m = __ldg(x + ((int64_t)b * C + c) * HW + r);
        s1 += m; s2 += (double)m * m;
        bi += step_b; r += step_r;
        if (r >= (unsigned)HW) { r -= (unsigned)HW; ++bi; }
    }
    __shared__ double sh[2][8];
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s1; sh[1][threadIdx.x >> 5] = s2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, b = 0;
        for (int w = 0; w < 8; ++w) { a += sh[0][w]; b += sh[1][w]; }
        double* rec = stage_rec(scratch, c);
        rec[sp * 2 + 0] = a;
        rec[sp * 2 + 1] = b;
        if (stage_last_slice(rec, (int)gridDim.y)) bn_finalize_channel(rec, (int)gridDim.y, 2, c, fin);
    }
}

// ------------------------------------------------------------------ F2: BN + ReLU + clamp + quantize + NHWC pack
// one thread = (pixel, 8-channel chunk).  pooled [B,C,PH,PW] fp32 -> xp [B,PH,PW,Cp] bf16 codes; optional act
// (dequantised fp32, NCHW) for callers that want the reference-layout tensor; xmax_out = max value (for the
// external-DAC sigma of the next layer, hardware_model.py:45).
struct BnActP {
    const float *x, *mean, *invstd, *gamma, *beta, *u_inject;
    __nv_bfloat16* xp;
    float* act;
    float* xmax_out;
    int B, C, HW, Cp;
    float act_max, q_scale, q_max, stoch;
    int quant;
    nn_rng rng;
    // dropout (DROP instantiations only): keep mask out [B,C,HW] uint8, optional injected mask, rate, 1/(1-p), stream
    uint8_t* keep;
    const uint8_t* keep_inject;
    float drop_p, drop_k;
    nn_rng drop_rng;
};

// Dropout between the clamp and the quantizer (noisynet.py:456, :512, :565): torch's x * (bernoulli(1-p) / (1-p)) in fp32,
// k = fl(1 / fl(1 - p)).  The keep decisions of a (pixel, 8-channel chunk) thread i come from their own Philox stream
// (drop_rng): groups 2i and 2i + 1 -- the group indices of the rounding draws, so those stay the same draws whether dropout
// is on or off -- word j for channel j of the chunk; keep iff u01 >= p.  The mask is stored (BN-input layout) for the backward.
__device__ __forceinline__ float stage_drop(float v, bool keep, float k) { return keep ? __fmul_rn(v, k) : 0.f; }

// keep bits of one (pixel, chunk) thread, bit j = channel j of the chunk (one register instead of eight words)
__device__ __forceinline__ unsigned stage_keep_bits(const NnRng& ds, unsigned i, float p) {
    const uint4 k0 = nn_philox(ds, (uint64_t)i * 2), k1 = nn_philox(ds, (uint64_t)i * 2 + 1);
    const uint32_t kr[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
    unsigned bits = 0u;
#pragma unroll
    for (int j = 0; j < 8; ++j) bits |= (nn_u01(kr[j]) >= p ? 1u : 0u) << j;
    return bits;
}

template <bool DROP>
__global__ void __launch_bounds__(256)
k_bn_act_pack(const BnActP p) {
    const NnRng rs = nn_rng_load(p.rng);
    NnRng ds{};
    if (DROP) ds = nn_rng_load(p.drop_rng);
    const int chunks = p.Cp >> 3;
    const unsigned npix = (unsigned)p.B * p.HW, total = npix * chunks;      // 32-bit index arithmetic
    float vmax = 0.f;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const unsigned pixel = ST_CHUNK_FAST ? i / chunks : i % npix;
        const int chunk = (int)(ST_CHUNK_FAST ? i % chunks : i / npix);
        const int b = (int)(pixel / p.HW), r = (int)(pixel - (unsigned)b * p.HW);
        __align__(16) __nv_bfloat16 out[8];
        uint4 rnd[2];
        if (p.quant && p.stoch > 0.f && !p.u_inject) {
            // Philox group = (NCHW element index of channel c) / 4 is not chunk aligned; use one group per
            // (pixel, chunk, half): 8 uniforms for 8 channels
            rnd[0] = nn_philox(rs, (uint64_t)i * 2);
            rnd[1] = nn_philox(rs, (uint64_t)i * 2 + 1);
        }
        const uint32_t* rr = reinterpret_cast<const uint32_t*>(rnd);
        uint4 krnd[2];
        if (DROP && !p.keep_inject) {
            krnd[0] = nn_philox(ds, (uint64_t)i * 2);
            krnd[1] = nn_philox(ds, (uint64_t)i * 2 + 1);
        }
        const uint32_t* kr = reinterpret_cast<const uint32_t*>(krnd);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = chunk * 8 + j;
            float code = 0.f;
            if (c < p.C) {
                const int64_t o = ((int64_t)b * p.C + c) * p.HW + r;
                float v = (__ldg(p.x + o) - __ldg(p.mean + c)) * __ldg(p.invstd + c) * __ldg(p.gamma + c) + __ldg(p.beta + c);
                v = fmaxf(v, 0.f);                                          // ReLU
                if (p.act_max > 0.f) v = fminf(v, p.act_max);               // clamp(max=act_max)
                if (DROP) {
                    const bool keep = p.keep_inject ? __ldg(p.keep_inject + o) != 0 : nn_u01(kr[j]) >= p.drop_p;
                    p.keep[o] = (uint8_t)keep;
                    v = stage_drop(v, keep, p.drop_k);
                }
                float val = v;
                if (p.quant) {
                    const float u = p.stoch > 0.f ? (p.u_inject ? __ldg(p.u_inject + o) : nn_usym(rr[j], p.stoch)) : 0.f;
                    code = quant_code(v, p.q_scale, p.q_max, u);
                    val = __fmul_rn(code, p.q_scale);
                } else {
                    code = v;
                }
                if (p.act) p.act[o] = val;
                vmax = fmaxf(vmax, val);
            }
            out[j] = __float2bfloat16_rn(code);
        }
        *reinterpret_cast<uint4*>(p.xp + ((size_t)pixel * p.Cp + chunk * 8)) = *reinterpret_cast<const uint4*>(out);
    }
    if (p.xmax_out) {
        vmax = nn_warp_max(vmax);
        if ((threadIdx.x & 31) == 0 && vmax > 0.f) nn_atomic_max_float(p.xmax_out, vmax);
    }
}

// Hot-path variant of k_bn_act_pack (training: k-bit quantisation, stochastic rounding from Philox, no injected draws,
// no fp32 copy): same thread mapping and arithmetic, but the run-time option checks are compiled out and the index
// arithmetic is 32-bit.  Registers are capped for 6 blocks/SM: the kernel is latency-bound, occupancy matters more
// than instruction count (variants that kept parameters in registers were slower).
template <bool DROP>
__global__ void __launch_bounds__(256, DROP ? 5 : 6)      // the keep bits need a few registers more than 6 blocks leave
k_bn_act_pack_lean(const BnActP p) {
    const NnRng rs = nn_rng_load(p.rng);
    NnRng ds{};
    if (DROP) ds = nn_rng_load(p.drop_rng);
    const unsigned chunks = (unsigned)(p.Cp >> 3), HW = (unsigned)p.HW, C = (unsigned)p.C;
    const unsigned npix = (unsigned)p.B * HW, total = npix * chunks;
    const float act_hi = p.act_max > 0.f ? p.act_max : __int_as_float(0x7f800000);
    const float two_s = __fmul_rn(2.0f, p.stoch), q_scale = p.q_scale, q_max = p.q_max, stoch = p.stoch;
    float vmax = 0.f;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const unsigned pixel = i / chunks, chunk = i - pixel * chunks;
        const unsigned b = pixel / HW, r = pixel - b * HW;
        const unsigned c0 = chunk * 8;
        const float* src = p.x + (b * C + c0) * HW + r;           // element index < 2^31 (host check)
        const unsigned kbits = DROP ? stage_keep_bits(ds, i, p.drop_p) : 0u;     // before the rounding words are live
        const uint4 r0 = nn_philox(rs, (uint64_t)i * 2), r1 = nn_philox(rs, (uint64_t)i * 2 + 1);
        const uint32_t rr[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
        __align__(16) __nv_bfloat16 out[8];
#pragma unroll
        for (unsigned j = 0; j < 8; ++j) {
            float code = 0.f;
            const unsigned c = c0 + j;
            if (c < C) {
                float v = (__ldg(src + j * HW) - __ldg(p.mean + c)) * __ldg(p.invstd + c) * __ldg(p.gamma + c) + __ldg(p.beta + c);
                v = fminf(fmaxf(v, 0.f), act_hi);                                   // ReLU, clamp(max=act_max)
                if (DROP) {
                    const bool keep = (kbits >> j) & 1u;
                    p.keep[(b * C + c0) * HW + r + j * HW] = (uint8_t)keep;
                    v = stage_drop(v, keep, p.drop_k);
                }
                const float u = __fadd_rn(__fmul_rn(nn_u01(rr[j]), two_s), -stoch);    // == nn_usym(rr[j], stoch)
                code = quant_code(v, q_scale, q_max, u);
                vmax = fmaxf(vmax, __fmul_rn(code, q_scale));
            }
            out[j] = __float2bfloat16_rn(code);
        }
        *reinterpret_cast<uint4*>(p.xp + ((size_t)pixel * p.Cp + c0)) = *reinterpret_cast<const uint4*>(out);
    }
    if (p.xmax_out) {
        vmax = nn_warp_max(vmax);
        if ((threadIdx.x & 31) == 0 && vmax > 0.f) nn_atomic_max_float(p.xmax_out, vmax);
    }
}

// Tiled variant of the hot path for HW >= 32 (the conv stages): same arithmetic and the same Philox counter per (pixel,
// chunk) as k_bn_act_pack_lean, but the thread mapping follows the memory instead of the output.  A block owns 32
// consecutive pixels: lane = pixel, so every channel read is one 128-byte line of the NCHW input (the chunk-fastest
// mapping touched 32 different lines per load instruction); the codes are staged in shared memory as the tile's NHWC
// image and leave as one contiguous 32 x Cp x 2 byte run.  Measured at batch 512, 65 channels 14x14: 43.5 -> see DESIGN.
template <bool DROP>
__global__ void __launch_bounds__(256)
k_bn_act_pack_tiled(const BnActP p) {
    extern __shared__ uint4 s_tile[];                       // [32 pixels][pitch] 16-byte chunks
    const NnRng rs = nn_rng_load(p.rng);
    NnRng ds{};
    if (DROP) ds = nn_rng_load(p.drop_rng);
    const unsigned chunks = (unsigned)(p.Cp >> 3), HW = (unsigned)p.HW, C = (unsigned)p.C;
    const unsigned pitch = chunks | 1u;                      // odd pitch: conflict-free 16-byte column writes
    const unsigned npix = (unsigned)p.B * HW;
    const float act_hi = p.act_max > 0.f ? p.act_max : __int_as_float(0x7f800000);
    const float two_s = __fmul_rn(2.0f, p.stoch), q_scale = p.q_scale, q_max = p.q_max, stoch = p.stoch;
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    float vmax = 0.f;
    for (unsigned tile = blockIdx.x; tile * 32u < npix; tile += gridDim.x) {
        const unsigned pixel = tile * 32u + lane;
        const bool pix_ok = pixel < npix;
        const unsigned b = pixel / HW, r = pixel - b * HW;
        for (unsigned chunk = warp; chunk < chunks; chunk += 8u) {
            const unsigned c0 = chunk * 8u;
            __align__(16) __nv_bfloat16 out[8];
            if (pix_ok) {
                const unsigned i = pixel * chunks + chunk;
                const float* src = p.x + (b * C + c0) * HW + r;           // element index < 2^31 (host check)
                const unsigned kbits = DROP ? stage_keep_bits(ds, i, p.drop_p) : 0u;
                const uint4 r0 = nn_philox(rs, (uint64_t)i * 2), r1 = nn_philox(rs, (uint64_t)i * 2 + 1);
                const uint32_t rr[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
                for (unsigned j = 0; j < 8; ++j) {
                    float code = 0.f;
                    const unsigned c = c0 + j;
                    if (c < C) {
                        float v = (__ldg(src + j * HW) - __ldg(p.mean + c)) * __ldg(p.invstd + c) * __ldg(p.gamma + c) + __ldg(p.beta + c);
                        v = fminf(fmaxf(v, 0.f), act_hi);                                   // ReLU, clamp(max=act_max)
                        if (DROP) {
                            const bool keep = (kbits >> j) & 1u;
                            p.keep[(b * C + c0) * HW + r + j * HW] = (uint8_t)keep;      // lane = pixel: 32 consecutive bytes
                            v = stage_drop(v, keep, p.drop_k);
                        }
                        const float u = __fadd_rn(__fmul_rn(nn_u01(rr[j]), two_s), -stoch);    // == nn_usym(rr[j], stoch)
                        code = quant_code(v, q_scale, q_max, u);
                        vmax = fmaxf(vmax, __fmul_rn(code, q_scale));
                    }
                    out[j] = __float2bfloat16_rn(code);
                }
                s_tile[lane * pitch + chunk] = *reinterpret_cast<const uint4*>(out);
            }
        }
        __syncthreads();
        const unsigned valid = min(32u, npix - tile * 32u) * chunks;        // 16-byte chunks of this tile's NHWC image
        uint4* dst = reinterpret_cast<uint4*>(p.xp + (size_t)tile * 32u * p.Cp);
        for (unsigned k = threadIdx.x; k < valid; k += 256u) {
            const unsigned px = k / chunks, ch = k - px * chunks;
            dst[k] = s_tile[px * pitch + ch];
        }
        __syncthreads();
    }
    if (p.xmax_out) {
        vmax = nn_warp_max(vmax);
        if ((threadIdx.x & 31) == 0 && vmax > 0.f) nn_atomic_max_float(p.xmax_out, vmax);
    }
}

// ------------------------------------------------------------------ B1: masks + per-channel sums of dv, dv*xhat
struct BnBwdP {
    const float *g, *x, *mean, *invstd, *gamma, *beta;
    double* scratch;              // channel records: partial sums + arrival counter (self-resetting)
    float *dbeta, *dgamma;        // written by the last slice's block of each channel
    int B, C, HW;
    float act_max, q_hi;
    const uint8_t* keep;          // dropout mask of the forward (DROP instantiations only), BN-input layout
    float drop_k;                 // 1 / (1 - p)
};

template <bool DROP>
__device__ __forceinline__ float stage_dv(float g, float x, float mean, float invstd, float gamma, float beta,
                                          float act_max, float q_hi, float& xhat, bool keep = true, float k = 1.f) {
    xhat = (x - mean) * invstd;
    const float v = xhat * gamma + beta;
    // ReLU: v > 0; clamp(max): v <= act_max; quantizer STE (hardware_model.py:176-183): 0 <= clamped <= q_hi
    bool pass = v > 0.f;
    if (act_max > 0.f) pass = pass && (v <= act_max);
    if (DROP) {
        // dropout: the quantizer saw fl(clamped * k) and the gradient is fl(g * k) on kept elements, 0 on dropped ones
        pass = pass && keep;
        if (q_hi > 0.f) pass = pass && (__fmul_rn(fminf(v, act_max > 0.f ? act_max : v), k) <= q_hi);
        return pass ? __fmul_rn(g, k) : 0.f;
    }
    if (q_hi > 0.f) pass = pass && (fminf(v, act_max > 0.f ? act_max : v) <= q_hi);
    return pass ? g : 0.f;
}

template <bool DROP>
__global__ void __launch_bounds__(256)
k_bn_bwd_stats(const BnBwdP p) {
    const int c = blockIdx.x, sp = blockIdx.y;
    const int b0 = (int)((int64_t)p.B * sp / (int)gridDim.y), b1 = (int)((int64_t)p.B * (sp + 1) / (int)gridDim.y);
    const int n = (b1 - b0) * p.HW;
    const float mean = p.mean[c], invstd = p.invstd[c], gamma = p.gamma[c], beta = p.beta[c];
    double s1 = 0.0, s2 = 0.0;
    const unsigned step_b = blockDim.x / (unsigned)p.HW, step_r = blockDim.x - step_b * (unsigned)p.HW;
    unsigned bi = threadIdx.x / (unsigned)p.HW, r = threadIdx.x - bi * (unsigned)p.HW;
    unsigned i = threadIdx.x;
    for (; i + 3 * blockDim.x < (unsigned)n; i += 4 * blockDim.x) {         // eight loads in flight, sums in element order
        float gv[4], xv[4];
        bool kv[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int64_t o = ((int64_t)(b0 + (int)bi) * p.C + c) * p.HW + r;
            gv[k] = __ldg(p.g + o); xv[k] = __ldg(p.x + o);
            kv[k] = DROP ? __ldg(p.keep + o) != 0 : true;
            bi += step_b; r += step_r;
            if (r >= (unsigned)p.HW) { r -= (unsigned)p.HW; ++bi; }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float xhat;
            const float dv = stage_dv<DROP>(gv[k], xv[k], mean, invstd, gamma, beta, p.act_max, p.q_hi, xhat, kv[k], p.drop_k);
            s1 += dv; s2 += (double)dv * xhat;
        }
    }
    for (; i < (unsigned)n; i += blockDim.x) {
        const int b = b0 + (int)bi;
        const int64_t o = ((int64_t)b * p.C + c) * p.HW + r;
        float xhat;
        const float dv = stage_dv<DROP>(__ldg(p.g + o), __ldg(p.x + o), mean, invstd, gamma, beta, p.act_max, p.q_hi, xhat,
                                        DROP ? __ldg(p.keep + o) != 0 : true, p.drop_k);
        s1 += dv; s2 += (double)dv * xhat;
        bi += step_b; r += step_r;
        if (r >= (unsigned)p.HW) { r -= (unsigned)p.HW; ++bi; }
    }
    __shared__ double sh[2][8];
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s1; sh[1][threadIdx.x >> 5] = s2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, b = 0;
        for (int w = 0; w < 8; ++w) { a += sh[0][w]; b += sh[1][w]; }
        double* rec = stage_rec(p.scratch, c);
        rec[sp * 2 + 0] = a;
        rec[sp * 2 + 1] = b;
        if (stage_last_slice(rec, (int)gridDim.y)) {
            const int splits = (int)gridDim.y;
            double s1 = 0, s2 = 0;
            for (int s = 0; s < splits; ++s) { s1 += __ldcg(rec + s * 2); s2 += __ldcg(rec + s * 2 + 1); }
            p.dbeta[c] = (float)s1;        // grads are OVERWRITTEN (the step zeroes them anyway)
            p.dgamma[c] = (float)s2;
        }
    }
}

// ------------------------------------------------------------------ B2: BN backward + max-pool routing -> NHWC bf16
// one thread = (output pixel (b, oh, ow), 8-channel chunk) of gyp [B,OH,OW,Cp]; pool = 0 -> no pooling (HW = OH*OW)
struct BnBwdApplyP {
    const float *g, *x, *mean, *invstd, *gamma, *beta, *dbeta, *dgamma;
    const uint8_t* amax;
    __nv_bfloat16* gyp;
    float* gy_f32;                // optional NCHW fp32 copy of the same gradient [B,C,OH,OW]
    int B, C, OH, OW, Cp, pool;
    float act_max, q_hi, inv_count;
    int planes, vH, vW;           // planes = 1: output in the planes layout [chunk][plane_stride][8] on a vH x vW grid
    long long plane_stride;
    const uint8_t* keep;          // dropout mask (DROP instantiations only), read at the index of g and x
    float drop_k;
};

template <bool DROP>
__global__ void __launch_bounds__(256)
k_bn_bwd_apply(const BnBwdApplyP p) {
    // one thread = (pooled pixel, 8-channel chunk): the BN-backward value of each channel is computed ONCE and
    // written to its arg-max window position (zeros to the other three) -- 4x fewer loads than a thread per
    // output pixel.  32-bit index arithmetic (sizes are < 2^31 by the API checks).
    const int chunks = p.Cp >> 3;
    const int PH = p.pool ? p.OH >> 1 : p.OH, PW = p.pool ? p.OW >> 1 : p.OW, PHW = PH * PW;
    const unsigned npp = (unsigned)p.B * PHW, total = npp * chunks;
    const int npos = p.pool ? 4 : 1;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        // NHWC output: chunk fastest (a warp writes whole pixels); planes output: pixel fastest (a warp writes one plane)
        const bool chunk_fast = ST_CHUNK_FAST && !p.planes;
        const unsigned pp = chunk_fast ? i / chunks : i % npp;
        const int chunk = (int)(chunk_fast ? i % chunks : i / npp);
        const int b = (int)(pp / PHW), r = (int)(pp - (unsigned)b * PHW);
        const int ph = r / PW, pw = r - ph * PW;
        float d[8];
        int pos[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = chunk * 8 + j;
            d[j] = 0.f; pos[j] = -1;
            if (c < p.C) {
                const size_t o = ((size_t)b * p.C + c) * PHW + r;
                float xhat;
                const float invstd = __ldg(p.invstd + c), gamma = __ldg(p.gamma + c);
                const float dv = stage_dv<DROP>(__ldg(p.g + o), __ldg(p.x + o), __ldg(p.mean + c), invstd, gamma,
                                                __ldg(p.beta + c), p.act_max, p.q_hi, xhat, DROP ? __ldg(p.keep + o) != 0 : true, p.drop_k);
                d[j] = gamma * invstd * (dv - __ldg(p.dbeta + c) * p.inv_count - xhat * __ldg(p.dgamma + c) * p.inv_count);
                pos[j] = p.pool ? (int)__ldg(p.amax + o) : 0;
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (q >= npos) break;
            const int oh = p.pool ? 2 * ph + (q >> 1) : ph, ow = p.pool ? 2 * pw + (q & 1) : pw;
            __align__(16) __nv_bfloat16 out[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float v = (pos[j] == q) ? d[j] : 0.f;
                out[j] = __float2bfloat16_rn(v);
                if (p.gy_f32 && pos[j] >= 0)
                    p.gy_f32[(((size_t)b * p.C + chunk * 8 + j) * p.OH + oh) * p.OW + ow] = v;
            }
            const size_t off = p.planes ? ((size_t)chunk * p.plane_stride + ((size_t)b * p.vH + oh) * p.vW + ow) * 8
                                        : (((size_t)b * p.OH + oh) * p.OW + ow) * p.Cp + chunk * 8;
            *reinterpret_cast<uint4*>(p.gyp + off) = *reinterpret_cast<const uint4*>(out);
        }
    }
}

// Hot-path variant of k_bn_bwd_apply: same thread mapping and arithmetic; pooling and the output layout are
// compile-time, no fp32 copy, 32-bit indices, registers capped for occupancy (see k_bn_act_pack_lean).
template <bool POOL, bool PLANES, bool DROP>
__global__ void __launch_bounds__(256, 5)
k_bn_bwd_apply_lean(const BnBwdApplyP p) {
    const unsigned chunks = (unsigned)(p.Cp >> 3), C = (unsigned)p.C;
    const unsigned PH = POOL ? p.OH >> 1 : p.OH, PW = POOL ? p.OW >> 1 : p.OW, PHW = PH * PW;
    const unsigned npp = (unsigned)p.B * PHW, total = npp * chunks;
    const float inv_count = p.inv_count;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const bool chunk_fast = ST_CHUNK_FAST && !PLANES;
        const unsigned pp = chunk_fast ? i / chunks : i % npp;
        const unsigned chunk = chunk_fast ? i - pp * chunks : i / npp;
        const unsigned b = pp / PHW, r = pp - b * PHW;
        const unsigned ph = r / PW, pw = r - ph * PW;
        const unsigned c0 = chunk * 8;
        const unsigned o0 = (b * C + c0) * PHW + r;                    // element index < 2^31 (host check)
        float d[8];
        int pos[8];
#pragma unroll
        for (unsigned j = 0; j < 8; ++j) {
            const unsigned c = c0 + j;
            d[j] = 0.f; pos[j] = -1;
            if (c < C) {
                const unsigned o = o0 + j * PHW;
                float xhat;
                const float invstd = __ldg(p.invstd + c), gamma = __ldg(p.gamma + c);
                const float dv = stage_dv<DROP>(__ldg(p.g + o), __ldg(p.x + o), __ldg(p.mean + c), invstd, gamma,
                                                __ldg(p.beta + c), p.act_max, p.q_hi, xhat, DROP ? __ldg(p.keep + o) != 0 : true, p.drop_k);
                d[j] = gamma * invstd * (dv - __ldg(p.dbeta + c) * inv_count - xhat * __ldg(p.dgamma + c) * inv_count);
                pos[j] = POOL ? (int)__ldg(p.amax + o) : 0;
            }
        }
#pragma unroll
        for (int q = 0; q < (POOL ? 4 : 1); ++q) {
            const unsigned oh = POOL ? 2 * ph + (q >> 1) : ph, ow = POOL ? 2 * pw + (q & 1) : pw;
            __align__(16) __nv_bfloat16 out[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) out[j] = __float2bfloat16_rn(pos[j] == q ? d[j] : 0.f);
            const size_t off = PLANES ? ((size_t)chunk * p.plane_stride + ((size_t)b * p.vH + oh) * p.vW + ow) * 8
                                      : (((size_t)b * p.OH + oh) * p.OW + ow) * p.Cp + c0;
            *reinterpret_cast<uint4*>(p.gyp + off) = *reinterpret_cast<const uint4*>(out);
        }
    }
}

// Per-image variant for pooled stages with NHWC output (stage 2: 120 x 5x5 -> 10x10): one block = one sample.  Its g / x /
// argmax slices are CONTIGUOUS (C * PH * PW elements): thread t reads element t, t + 256, ... (the chunk-fastest mapping of
// k_bn_bwd_apply_lean touched 32 cache lines per load instruction); the sample's NHWC bf16 gradient image (zeros included)
// is assembled in shared memory and leaves as one contiguous run.  Same arithmetic as k_bn_bwd_apply.
template <bool DROP>
__global__ void __launch_bounds__(256)
k_bn_bwd_apply_img(const BnBwdApplyP p) {
    extern __shared__ uint4 s_img4[];
    __nv_bfloat16* s_img = reinterpret_cast<__nv_bfloat16*>(s_img4);
    const unsigned C = (unsigned)p.C, PH = p.OH >> 1, PW = p.OW >> 1, PHW = PH * PW, n = C * PHW;
    const unsigned img16 = (unsigned)(p.OH * p.OW * p.Cp) >> 3;          // 16-byte chunks of the sample's output image
    const float inv_count = p.inv_count;
    for (unsigned b = blockIdx.x; b < (unsigned)p.B; b += gridDim.x) {
        for (unsigned k = threadIdx.x; k < img16; k += 256u) s_img4[k] = make_uint4(0u, 0u, 0u, 0u);
        __syncthreads();
        const unsigned o0 = b * n;                                       // element index < 2^31 (host check)
        for (unsigned e = threadIdx.x; e < n; e += 256u) {
            const unsigned c = e / PHW, r = e - c * PHW, ph = r / PW, pw = r - ph * PW;
            float xhat;
            const float invstd = __ldg(p.invstd + c), gamma = __ldg(p.gamma + c);
            const float dv = stage_dv<DROP>(__ldg(p.g + o0 + e), __ldg(p.x + o0 + e), __ldg(p.mean + c), invstd, gamma, __ldg(p.beta + c),
                                            p.act_max, p.q_hi, xhat, DROP ? __ldg(p.keep + o0 + e) != 0 : true, p.drop_k);
            const float d = gamma * invstd * (dv - __ldg(p.dbeta + c) * inv_count - xhat * __ldg(p.dgamma + c) * inv_count);
            const unsigned pos = __ldg(p.amax + o0 + e);
            const unsigned oh = 2 * ph + (pos >> 1), ow = 2 * pw + (pos & 1);
            s_img[(oh * p.OW + ow) * p.Cp + c] = __float2bfloat16_rn(d);
        }
        __syncthreads();
        uint4* dst = reinterpret_cast<uint4*>(p.gyp + (size_t)b * p.OH * p.OW * p.Cp);
        for (unsigned k = threadIdx.x; k < img16; k += 256u) dst[k] = s_img4[k];
        __syncthreads();
    }
}

// ------------------------------------------------------------------ input quantize + pack (noisynet.py:390-393)
__global__ void __launch_bounds__(256)
k_quant_pack_input(const float* __restrict__ x, __nv_bfloat16* __restrict__ xp, float* __restrict__ act, int B, int C, int HW,
                   int Cp, int quant, float q_scale, float q_max, float stoch, const float* __restrict__ u_inject, nn_rng rng) {
    const NnRng rs = nn_rng_load(rng);
    const int chunks = Cp >> 3;
    const unsigned npix = (unsigned)B * HW, total = npix * chunks;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const unsigned pixel = i % npix;
        const int chunk = (int)(i / npix);
        const int b = (int)(pixel / HW), r = (int)(pixel - (unsigned)b * HW);
        uint4 rnd[2];
        if (quant && stoch > 0.f && !u_inject) {
            rnd[0] = nn_philox(rs, (uint64_t)i * 2);
            if (chunk * 8 + 4 < C) rnd[1] = nn_philox(rs, (uint64_t)i * 2 + 1);       // words for channels 4..7 of the chunk
        }
        const uint32_t* rr = reinterpret_cast<const uint32_t*>(rnd);
        __align__(16) __nv_bfloat16 out[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = chunk * 8 + j;
            float code = 0.f;
            if (c < C) {
                const int64_t o = ((int64_t)b * C + c) * HW + r;
                const float v = __ldg(x + o);
                if (quant) {
                    code = quant_code(v, q_scale, q_max, stoch > 0.f ? (u_inject ? __ldg(u_inject + o) : nn_usym(rr[j], stoch)) : 0.f);
                    if (act) act[o] = __fmul_rn(code, q_scale);
                } else {
                    code = v;
                    if (act) act[o] = v;
                }
            }
            out[j] = __float2bfloat16_rn(code);
        }
        *reinterpret_cast<uint4*>(xp + ((size_t)pixel * Cp + chunk * 8)) = *reinterpret_cast<const uint4*>(out);
    }
}

// ------------------------------------------------------------------ head: BatchNorm1d(C<=16) + cross entropy + backward
// single block, thread = row (rows strided by blockDim when B > blockDim).  Per-channel sums: registers ->
// warp shuffle tree -> fixed-order sum over warps in shared memory (deterministic).
constexpr int HEAD_MAXC = 16;

__device__ __forceinline__ void head_block_sum(double (&v)[HEAD_MAXC], int C, double (*sh)[HEAD_MAXC], double* out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c) {
        if (c < C) {
            double x = v[c];
            for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
            if (lane == 0) sh[warp][c] = x;
        }
    }
    __syncthreads();
    if (threadIdx.x < C) {
        double t = 0;
        for (int w = 0; w < nwarp; ++w) t += sh[w][threadIdx.x];
        out[threadIdx.x] = t;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(1024)
k_head(const float* __restrict__ z, const int64_t* __restrict__ label, int B, int C, const float* __restrict__ gamma,
       const float* __restrict__ beta, float* __restrict__ running_mean, float* __restrict__ running_var, float momentum,
       float eps, float* __restrict__ loss_out, float* __restrict__ out, float* __restrict__ g, __nv_bfloat16* __restrict__ gp,
       int Cp, float* __restrict__ dgamma, float* __restrict__ dbeta) {
    __shared__ double sh[32][HEAD_MAXC];
    __shared__ double tot1[HEAD_MAXC], tot2[HEAD_MAXC];
    __shared__ float s_mean[HEAD_MAXC], s_invstd[HEAD_MAXC], s_g[HEAD_MAXC], s_b[HEAD_MAXC];
    const int tid = threadIdx.x, nthr = blockDim.x;
    double a1[HEAD_MAXC], a2[HEAD_MAXC];
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c) { a1[c] = 0; a2[c] = 0; }
    for (int b = tid; b < B; b += nthr) {
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c)
            if (c < C) { const double v = z[(size_t)b * C + c]; a1[c] += v; a2[c] += v * v; }
    }
    head_block_sum(a1, C, sh, tot1);
    head_block_sum(a2, C, sh, tot2);
    if (tid < C) {
        const double m = tot1[tid] / B;
        double var = tot2[tid] / B - m * m;
        if (var < 0) var = 0;
        s_mean[tid] = (float)m;
        s_invstd[tid] = (float)(1.0 / sqrt(var + (double)eps));
        s_g[tid] = gamma[tid]; s_b[tid] = beta[tid];
        if (running_mean) {
            const double unb = B > 1 ? var * B / (B - 1) : var;
            running_mean[tid] = (float)((1.0 - momentum) * running_mean[tid] + momentum * m);
            running_var[tid] = (float)((1.0 - momentum) * running_var[tid] + momentum * unb);
        }
    }
    __syncthreads();
    // softmax / CE per row; dv = (softmax - onehot) / B kept in g; per-channel sums of dv and dv * xhat
    double lsum[HEAD_MAXC];
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c) { a1[c] = 0; a2[c] = 0; lsum[c] = 0; }
    for (int b = tid; b < B; b += nthr) {
        float v[HEAD_MAXC], xh[HEAD_MAXC];
        float mx = -3.4e38f;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) {
            if (c < C) {
                xh[c] = (z[(size_t)b * C + c] - s_mean[c]) * s_invstd[c];
                v[c] = xh[c] * s_g[c] + s_b[c];
                if (out) out[(size_t)b * C + c] = v[c];
                mx = fmaxf(mx, v[c]);
            }
        }
        float se = 0.f;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) if (c < C) se += expf(v[c] - mx);
        const int lab = (int)label[b];
        float vl = 0.f;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) if (c == lab) vl = v[c];
        lsum[0] += (double)(logf(se) + mx - vl);
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) {
            if (c < C) {
                const float dv = (expf(v[c] - mx) / se - (c == lab ? 1.f : 0.f)) / (float)B;
                g[(size_t)b * C + c] = dv;
                a1[c] += dv; a2[c] += (double)dv * xh[c];
            }
        }
    }
    head_block_sum(lsum, 1, sh, tot1);
    if (tid == 0) *loss_out = (float)(tot1[0] / B);
    __syncthreads();
    head_block_sum(a1, C, sh, tot1);
    head_block_sum(a2, C, sh, tot2);
    if (tid < C) { dbeta[tid] = (float)tot1[tid]; dgamma[tid] = (float)tot2[tid]; }
    const float invB = 1.f / (float)B;
    for (int b = tid; b < B; b += nthr) {
        for (int c = 0; c < Cp; ++c) {
            float d = 0.f;
            if (c < C) {
                const float xhat = (z[(size_t)b * C + c] - s_mean[c]) * s_invstd[c];
                d = s_g[c] * s_invstd[c] * (g[(size_t)b * C + c] - (float)tot1[c] * invB - xhat * (float)tot2[c] * invB);
                g[(size_t)b * C + c] = d;
            }
            if (gp) gp[(size_t)b * Cp + c] = __float2bfloat16_rn(d);
        }
    }
}

// Faster formulation for B <= blockDim (one thread per row, the training batch): the per-channel reductions run
// one WARP PER CHANNEL over shared-memory columns (lane-strided fp64 partials, then one shuffle tree) instead of 16
// fp64 shuffle trees per warp -- fp64 issue is the scarce resource here.  Same arithmetic and summation order
// independent of the launch; results differ from k_head only in the (fixed) order of the fp64 sums.
__device__ __forceinline__ double head_col_sum(const float* col, int B) {
    const int lane = threadIdx.x & 31;
    double s = 0;
    for (int b = lane; b < B; b += 32) s += (double)col[b];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

__global__ void __launch_bounds__(1024)
k_head_rows(const float* __restrict__ z, const int64_t* __restrict__ label, int B, int C, const float* __restrict__ gamma,
            const float* __restrict__ beta, float* __restrict__ running_mean, float* __restrict__ running_var, float momentum,
            float eps, float* __restrict__ loss_out, float* __restrict__ out, float* __restrict__ g, __nv_bfloat16* __restrict__ gp,
            int Cp, float* __restrict__ dgamma, float* __restrict__ dbeta) {
    extern __shared__ float hsm[];
    float* colA = hsm;                       // [C][B]: z, then dv
    float* colB = hsm + (size_t)C * B;       // [C][B]: z^2, then dv * xhat
    float* lrow = colB + (size_t)C * B;      // [B] loss terms
    __shared__ float s_mean[HEAD_MAXC], s_invstd[HEAD_MAXC], s_g[HEAD_MAXC], s_b[HEAD_MAXC], s_db[HEAD_MAXC], s_dg[HEAD_MAXC];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarp = blockDim.x >> 5;
    const bool row = tid < B;
    float zr[HEAD_MAXC];
#pragma unroll
    for (int c = 0; c < HEAD_MAXC; ++c) {
        zr[c] = 0.f;
        if (c < C && row) {
            zr[c] = z[(size_t)tid * C + c];
            colA[(size_t)c * B + tid] = zr[c];
            colB[(size_t)c * B + tid] = zr[c] * zr[c];
        }
    }
    __syncthreads();
    for (int c = warp; c < C; c += nwarp) {
        const double t1 = head_col_sum(colA + (size_t)c * B, B), t2 = head_col_sum(colB + (size_t)c * B, B);
        if (lane == 0) {
            const double m = t1 / B;
            double var = t2 / B - m * m;
            if (var < 0) var = 0;
            s_mean[c] = (float)m;
            s_invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
            s_g[c] = gamma[c]; s_b[c] = beta[c];
            if (running_mean) {
                const double unb = B > 1 ? var * B / (B - 1) : var;
                running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * m);
                running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unb);
            }
        }
    }
    __syncthreads();
    float xh[HEAD_MAXC], dvr[HEAD_MAXC];
    if (row) {
        float vv[HEAD_MAXC];
        float mx = -3.4e38f;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) {
            if (c < C) {
                xh[c] = (zr[c] - s_mean[c]) * s_invstd[c];
                vv[c] = xh[c] * s_g[c] + s_b[c];
                if (out) out[(size_t)tid * C + c] = vv[c];
                mx = fmaxf(mx, vv[c]);
            }
        }
        float se = 0.f;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) if (c < C) se += expf(vv[c] - mx);
        const int lab = (int)label[tid];
        float vl = 0.f;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) if (c == lab) vl = vv[c];
        lrow[tid] = logf(se) + mx - vl;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) {
            if (c < C) {
                dvr[c] = (expf(vv[c] - mx) / se - (c == lab ? 1.f : 0.f)) / (float)B;
                colA[(size_t)c * B + tid] = dvr[c];
                colB[(size_t)c * B + tid] = dvr[c] * xh[c];
            }
        }
    }
    __syncthreads();
    for (int c = warp; c <= C; c += nwarp) {
        if (c == C) {
            const double t = head_col_sum(lrow, B);
            if (lane == 0) *loss_out = (float)(t / B);
        } else {
            const double t1 = head_col_sum(colA + (size_t)c * B, B), t2 = head_col_sum(colB + (size_t)c * B, B);
            if (lane == 0) { s_db[c] = (float)t1; s_dg[c] = (float)t2; dbeta[c] = (float)t1; dgamma[c] = (float)t2; }
        }
    }
    __syncthreads();
    if (row) {
        const float invB = 1.f / (float)B;
        for (int c = 0; c < Cp; ++c) {
            float d = 0.f;
            if (c < C) {
                d = s_g[c] * s_invstd[c] * (dvr[c] - s_db[c] * invB - xh[c] * s_dg[c] * invB);
                g[(size_t)tid * C + c] = d;
            }
            if (gp) gp[(size_t)tid * Cp + c] = __float2bfloat16_rn(d);
        }
    }
}

// ------------------------------------------------------------------ classifier tail, fused (noisynet.py:589-594, :1278)
// fc2 forward with its current noise -> BatchNorm1d (batch statistics) -> mean cross entropy -> gradient back
// through both -> fc2 dgrad, for a layer with <= 16 output units: three launches of a few microseconds of work each
// sat back to back on the critical path of the step (tensor-core forward, head, tensor-core dgrad).
// ONE thread-block cluster of 8 CTAs: each CTA owns B/8 samples, keeps its activation rows (bf16 codes) and the
// whole weight matrix (codes + g(|w|)) in shared memory, and the two batch-wide reductions (BN statistics; dbeta /
// dgamma / loss) go through distributed shared memory with a cluster barrier -- fixed summation order, identical in
// every CTA.  Arithmetic mirrors the separate kernels: integer-code main contraction (exact), sigma^2 from
// bf16-rounded g(|w|) with fp32 accumulation, Philox group = m * ceil(C/4) + n/4, bf16-rounded gradient as the dgrad
// operand, dgrad scaled by the weight code scale.
constexpr int TAIL_CTAS = 8;
constexpr int TAIL_THREADS = 256;

struct TailP {
    const __nv_bfloat16* xp; int B, K, Kp, C, R;       // R = rows per CTA
    const int8_t* w_codes; const float* w_raw;
    float y_scale, s_scale, w_code_scale;
    int noise_mode; float current; const float* scale_dev; const float* z_inject; nn_rng rng;
    const int64_t* labels; const float *gamma, *beta; float *running_mean, *running_var; float momentum, eps;
    float *loss_out, *logits_out, *g; __nv_bfloat16* gp; int Cp_g;
    float* gx; float *dgamma, *dbeta;
    int xs_stride;                                      // bf16 elements per shared activation row (odd word count)
};

__device__ __forceinline__ void tail_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t tail_pack_bf16(float lo, float hi) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&v);
}

__device__ __forceinline__ double tail_cluster_sum(cg::cluster_group& cluster, double* slot, int idx) {
    // slot[idx] of every CTA, summed in rank order (every CTA computes the same value); all remote loads are issued
    // before the first add (a distributed-shared-memory read is a ~1 us round trip)
    double v[TAIL_CTAS];
#pragma unroll
    for (int r = 0; r < TAIL_CTAS; ++r) v[r] = cluster.map_shared_rank(slot, r)[idx];
    double t = 0;
#pragma unroll
    for (int r = 0; r < TAIL_CTAS; ++r) t += v[r];
    return t;
}

__global__ void __launch_bounds__(TAIL_THREADS, 1)
k_classifier_tail(const TailP p) {
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) uint8_t tsm[];
    const int R = p.R, C = p.C, K = p.K;
    // shared memory: operands as bf16 for mma.sync (integer codes and bf16-rounded g(|w|) are exact in bf16)
    const int K16 = (K + 15) & ~15, KS = p.xs_stride, R16 = (R + 15) & ~15;
    __nv_bfloat16* wq = reinterpret_cast<__nv_bfloat16*>(tsm);                      // [16][KS] weight codes (rows >= C zero)
    __nv_bfloat16* wg = wq + 16 * KS;                                               // [16][KS] g(|w_raw|)
    __nv_bfloat16* wqT = wg + 16 * KS;                                              // [K16][16] codes, transposed (dgrad)
    __nv_bfloat16* xs = wqT + (size_t)K16 * 16;                                     // [R16][KS] activation codes
    float* ysm = reinterpret_cast<float*>(xs + (size_t)R16 * KS);                   // [R16][16] logits -> dv
    float* ssm = ysm + R16 * 16;                                                    // [R16][16] S -> xhat
    float* gsm = ssm + R16 * 16;                                                    // [R16][16] bf16-rounded final gradient
    __shared__ double part[2][HEAD_MAXC + 1];          // this CTA's partial sums (exchanged through DSMEM)
    __shared__ float s_mean[HEAD_MAXC], s_invstd[HEAD_MAXC], s_g[HEAD_MAXC], s_b[HEAD_MAXC], s_db[HEAD_MAXC], s_dg[HEAD_MAXC];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int row0 = (int)cluster.block_rank() * R;
    const int nrows = max(0, min(R, p.B - row0));

    // ---- stage operands (vector loads, several in flight; everything not loaded is zero)
    {
        uint4* z = reinterpret_cast<uint4*>(tsm);
        const int n16 = (int)(((size_t)(2 * 16 * KS + K16 * 16 + (size_t)R16 * KS) * 2 + (size_t)3 * R16 * 16 * 4) / 16);
        for (int i = tid; i < n16; i += TAIL_THREADS) z[i] = make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    {
        const int total = C * K, groups = (total + 3) >> 2;                 // 4 consecutive parameters per thread
        const bool vec = ((reinterpret_cast<uintptr_t>(p.w_codes) & 3) == 0) &&
                         (p.noise_mode == NN_NOISE_NONE || (reinterpret_cast<uintptr_t>(p.w_raw) & 15) == 0);
#pragma unroll 4
        for (int gi = tid; gi < groups; gi += TAIL_THREADS) {
            const int i0 = gi * 4;
            int8_t cq[4] = {0, 0, 0, 0};
            float wr[4] = {0.f, 0.f, 0.f, 0.f};
            if (vec && i0 + 4 <= total) {
                const uint32_t w4 = __ldg(reinterpret_cast<const uint32_t*>(p.w_codes) + gi);
                cq[0] = (int8_t)(w4 & 0xff); cq[1] = (int8_t)((w4 >> 8) & 0xff); cq[2] = (int8_t)((w4 >> 16) & 0xff); cq[3] = (int8_t)(w4 >> 24);
                if (p.noise_mode != NN_NOISE_NONE) {
                    const float4 f = __ldg(reinterpret_cast<const float4*>(p.w_raw) + gi);
                    wr[0] = f.x; wr[1] = f.y; wr[2] = f.z; wr[3] = f.w;
                }
            } else {
                for (int e = 0; e < 4; ++e)
                    if (i0 + e < total) { cq[e] = p.w_codes[i0 + e]; if (p.noise_mode != NN_NOISE_NONE) wr[e] = __ldg(p.w_raw + i0 + e); }
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int i = i0 + e;
                if (i < total) {
                    const int n = i / K, k = i - n * K;
                    const __nv_bfloat16 cb = __float2bfloat16_rn((float)cq[e]);
                    wq[n * KS + k] = cb;
                    wqT[k * 16 + n] = cb;
                    if (p.noise_mode != NN_NOISE_NONE) {
                        const float a = fabsf(wr[e]);
                        wg[n * KS + k] = __float2bfloat16_rn((p.noise_mode == NN_NOISE_MERGED) ? a : __fadd_rn(__fmul_rn(a, a), a));
                    }
                }
            }
        }
    }
    {
        const bool vec = (p.Kp % 8 == 0) && ((reinterpret_cast<uintptr_t>(p.xp) & 15) == 0);
        const int vpr = vec ? p.Kp / 8 : 0;                                // 16-byte vectors per global row
#pragma unroll 4
        for (int i = tid; i < nrows * vpr; i += TAIL_THREADS) {
            const int r = i / vpr, q4 = i - r * vpr;
            const uint4 x4 = __ldg(reinterpret_cast<const uint4*>(p.xp + (size_t)(row0 + r) * p.Kp) + q4);
            uint32_t* dst = reinterpret_cast<uint32_t*>(xs + (size_t)r * KS) + q4 * 4;
            const uint32_t w[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) if ((q4 * 4 + e) * 2 < K16) dst[e] = w[e];
        }
        if (!vec)
            for (int i = tid; i < nrows * (p.Kp / 2); i += TAIL_THREADS) {
                const int r = i / (p.Kp / 2), kk = (i - r * (p.Kp / 2)) * 2;
                if (kk < K16) *reinterpret_cast<uint32_t*>(xs + (size_t)r * KS + kk) =
                    *reinterpret_cast<const uint32_t*>(p.xp + (size_t)(row0 + r) * p.Kp + kk);
            }
    }
    __syncthreads();

    // ---- forward contraction on the tensor cores (mma.sync m16n8k16, bf16 x bf16 -> fp32): a warp owns 16 rows and
    // both 8-unit column tiles; main accumulators are exact integer sums, sigma^2 accumulators fp32
    {
        const int gq = lane >> 2, tig = lane & 3;
        for (int rb = warp; rb < R16 / 16; rb += TAIL_THREADS / 32) {
            float cm[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}}, cs[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
            const __nv_bfloat16* xa = xs + (size_t)(rb * 16 + gq) * KS + 2 * tig;
            for (int k0 = 0; k0 < K16; k0 += 16) {
                uint32_t af[4];
                af[0] = *reinterpret_cast<const uint32_t*>(xa + k0);
                af[1] = *reinterpret_cast<const uint32_t*>(xa + 8 * KS + k0);
                af[2] = *reinterpret_cast<const uint32_t*>(xa + k0 + 8);
                af[3] = *reinterpret_cast<const uint32_t*>(xa + 8 * KS + k0 + 8);
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) {
                    const int wo = (nt * 8 + gq) * KS + k0 + 2 * tig;
                    tail_mma(cm[nt], af, *reinterpret_cast<const uint32_t*>(wq + wo), *reinterpret_cast<const uint32_t*>(wq + wo + 8));
                    if (p.noise_mode != NN_NOISE_NONE)
                        tail_mma(cs[nt], af, *reinterpret_cast<const uint32_t*>(wg + wo), *reinterpret_cast<const uint32_t*>(wg + wo + 8));
                }
            }
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
                const int c0 = nt * 8 + 2 * tig, r0 = rb * 16 + gq;
                ysm[r0 * 16 + c0] = cm[nt][0] * p.y_scale;       ysm[r0 * 16 + c0 + 1] = cm[nt][1] * p.y_scale;
                ysm[(r0 + 8) * 16 + c0] = cm[nt][2] * p.y_scale; ysm[(r0 + 8) * 16 + c0 + 1] = cm[nt][3] * p.y_scale;
                ssm[r0 * 16 + c0] = cs[nt][0] * p.s_scale;       ssm[r0 * 16 + c0 + 1] = cs[nt][1] * p.s_scale;
                ssm[(r0 + 8) * 16 + c0] = cs[nt][2] * p.s_scale; ssm[(r0 + 8) * 16 + c0 + 1] = cs[nt][3] * p.s_scale;
            }
        }
    }
    __syncthreads();
    // ---- current noise: thread = (row, group of 4 units), the Philox mapping of every other path
    if (p.noise_mode != NN_NOISE_NONE) {
        const int ngrp = (C + 3) >> 2;
        const float coef = nn_noise_coef(*p.scale_dev, p.current);
        const NnRng rs = nn_rng_load(p.rng);
        for (int i = tid; i < nrows * ngrp; i += TAIL_THREADS) {
            const int r = i / ngrp, gq = i - r * ngrp, m = row0 + r;
            float z[4];
            if (!p.z_inject) nn_normal4(rs, (uint64_t)m * ngrp + (uint64_t)gq, z);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int n = gq * 4 + j;
                if (n < C) {
                    const float zz = p.z_inject ? __ldg(p.z_inject + (size_t)m * C + n) : z[j];
                    ysm[r * 16 + n] = __fadd_rn(ysm[r * 16 + n], __fmul_rn(zz, nn_sigma(coef, ssm[r * 16 + n])));
                }
            }
        }
        __syncthreads();
    }
    if (p.logits_out)
        for (int i = tid; i < nrows * C; i += TAIL_THREADS) p.logits_out[(size_t)(row0 + i / C) * C + i % C] = ysm[(i / C) * 16 + i % C];

    // ---- BatchNorm statistics over the whole batch
    for (int c = warp; c < C; c += TAIL_THREADS / 32) {
        double s1 = 0, s2 = 0;
        for (int r = lane; r < nrows; r += 32) { const double v = ysm[r * 16 + c]; s1 += v; s2 += v * v; }
        for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
        if (lane == 0) { part[0][c] = s1; part[1][c] = s2; }
    }
    cluster.sync();
    if (tid < C) {
        const double t1 = tail_cluster_sum(cluster, &part[0][0], tid), t2 = tail_cluster_sum(cluster, &part[1][0], tid);
        const double mean = t1 / p.B;
        double var = t2 / p.B - mean * mean;
        if (var < 0) var = 0;
        s_mean[tid] = (float)mean;
        s_invstd[tid] = (float)(1.0 / sqrt(var + (double)p.eps));
        s_g[tid] = p.gamma[tid]; s_b[tid] = p.beta[tid];
        if (p.running_mean && cluster.block_rank() == 0) {
            const double unb = p.B > 1 ? var * p.B / (p.B - 1) : var;
            p.running_mean[tid] = (float)((1.0 - p.momentum) * p.running_mean[tid] + p.momentum * mean);
            p.running_var[tid] = (float)((1.0 - p.momentum) * p.running_var[tid] + p.momentum * unb);
        }
    }
    cluster.sync();                      // everyone has read the first round of partials before they are overwritten
    // ---- softmax / cross entropy per row; dv = (softmax - onehot) / B
    float lrow = 0.f;
    if (tid < nrows) {
        const int r = tid;
        float vv[HEAD_MAXC], xh[HEAD_MAXC];
        float mx = -3.4e38f;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c)
            if (c < C) { xh[c] = (ysm[r * 16 + c] - s_mean[c]) * s_invstd[c]; vv[c] = xh[c] * s_g[c] + s_b[c]; mx = fmaxf(mx, vv[c]); }
        float se = 0.f;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) if (c < C) se += expf(vv[c] - mx);
        const int lab = (int)p.labels[row0 + r];
        float vl = 0.f;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c) if (c == lab) vl = vv[c];
        lrow = logf(se) + mx - vl;
#pragma unroll
        for (int c = 0; c < HEAD_MAXC; ++c)
            if (c < C) {
                ysm[r * 16 + c] = (expf(vv[c] - mx) / se - (c == lab ? 1.f : 0.f)) / (float)p.B;     // dv
                ssm[r * 16 + c] = xh[c];
            }
    }
    __syncthreads();
    for (int c = warp; c <= C; c += TAIL_THREADS / 32) {
        double s1 = 0, s2 = 0;
        if (c < C) {
            for (int r = lane; r < nrows; r += 32) { const double dv = ysm[r * 16 + c]; s1 += dv; s2 += dv * (double)ssm[r * 16 + c]; }
        }
        for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
        if (lane == 0 && c < C) { part[0][c] = s1; part[1][c] = s2; }
    }
    {   // loss: sum of the per-row terms of this CTA (warp 0 gathers through shared memory)
        __shared__ float lsh[TAIL_THREADS / 32];
        float l = lrow;
        for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
        if (lane == 0) lsh[warp] = l;
        __syncthreads();
        if (tid == 0) { double t = 0; for (int w = 0; w < TAIL_THREADS / 32; ++w) t += lsh[w]; part[0][HEAD_MAXC] = t; }
    }
    cluster.sync();
    if (tid < C) {
        const double t1 = tail_cluster_sum(cluster, &part[0][0], tid), t2 = tail_cluster_sum(cluster, &part[1][0], tid);
        s_db[tid] = (float)t1; s_dg[tid] = (float)t2;
        if (cluster.block_rank() == 0) { p.dbeta[tid] = (float)t1; p.dgamma[tid] = (float)t2; }
    }
    if (tid == 0 && cluster.block_rank() == 0) *p.loss_out = (float)(tail_cluster_sum(cluster, &part[0][0], HEAD_MAXC) / p.B);
    __syncthreads();
    // ---- gradient w.r.t. the fc2 output
    const float invB = 1.f / (float)p.B;
    for (int i = tid; i < nrows * 16; i += TAIL_THREADS) {
        const int r = i >> 4, c = i & 15;
        float d = 0.f;
        if (c < C) {
            d = s_g[c] * s_invstd[c] * (ysm[r * 16 + c] - s_db[c] * invB - ssm[r * 16 + c] * s_dg[c] * invB);
            p.g[(size_t)(row0 + r) * C + c] = d;
        }
        const __nv_bfloat16 db = __float2bfloat16_rn(d);
        gsm[i] = __bfloat162float(db);
        if (p.gp && c < p.Cp_g) p.gp[(size_t)(row0 + r) * p.Cp_g + c] = db;
    }
    __syncthreads();
    // ---- dgrad on the tensor cores: gx[m][k] = w_code_scale * sum_n g_bf16[m][n] * code[n][k]
    {
        const int gq = lane >> 2, tig = lane & 3;
        for (int rb = warp; rb < R16 / 16; rb += TAIL_THREADS / 32) {
            const int r0 = rb * 16 + gq;
            uint32_t af[4];
            af[0] = tail_pack_bf16(gsm[r0 * 16 + 2 * tig], gsm[r0 * 16 + 2 * tig + 1]);
            af[1] = tail_pack_bf16(gsm[(r0 + 8) * 16 + 2 * tig], gsm[(r0 + 8) * 16 + 2 * tig + 1]);
            af[2] = tail_pack_bf16(gsm[r0 * 16 + 8 + 2 * tig], gsm[r0 * 16 + 8 + 2 * tig + 1]);
            af[3] = tail_pack_bf16(gsm[(r0 + 8) * 16 + 8 + 2 * tig], gsm[(r0 + 8) * 16 + 8 + 2 * tig + 1]);
            for (int nt = 0; nt < K16 / 8; ++nt) {
                float d[4] = {0.f, 0.f, 0.f, 0.f};
                const __nv_bfloat16* wb = wqT + (size_t)(nt * 8 + gq) * 16 + 2 * tig;
                tail_mma(d, af, *reinterpret_cast<const uint32_t*>(wb), *reinterpret_cast<const uint32_t*>(wb + 8));
                const int c0 = nt * 8 + 2 * tig;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = r0 + 8 * h;
                    if (r < nrows) {
                        float* o = p.gx + (size_t)(row0 + r) * K + c0;
                        if (c0 < K) o[0] = d[2 * h] * p.w_code_scale;
                        if (c0 + 1 < K) o[1] = d[2 * h + 1] * p.w_code_scale;
                    }
                }
            }
        }
    }
    cluster.sync();                      // distributed shared memory stays valid until every CTA is done reading
}

static inline int grid_cap(int64_t items, int device, int waves = 8) {
    int64_t blocks = (items + 255) / 256, cap = (int64_t)nn_num_sms(device) * waves;
    if (blocks > cap) blocks = cap;
    return (int)(blocks < 1 ? 1 : blocks);
}

}  // namespace

// C channel records (stage_rec): monotone in C, so one scratch sized for the widest stage serves every stage
extern "C" int64_t nn_stage_scratch_bytes(int C) { return (int64_t)C * ST_REC * sizeof(double); }

extern "C" int nn_stage_fwd(const nn_stage_args* a, int device, void* stream) {
    if (!a || !a->in || !a->xp || !a->scratch || !a->mean || !a->invstd)
        return nn_fail("nn_stage_fwd: null argument%s", "");
    if (a->pool && ((a->H | a->W) & 1)) return nn_fail("nn_stage_fwd: pooling needs even H, W%s", "");
    if (a->Cp % 8 || a->Cp < a->C) return nn_fail("nn_stage_fwd: bad Cp%s", "");
    if (a->eval_mode && (!a->running_mean || !a->running_var)) return nn_fail("nn_stage_fwd: eval_mode needs the running statistics%s", "");
    if (!(a->drop_p >= 0.0 && a->drop_p < 1.0)) return nn_fail("nn_stage_fwd: drop_p must lie in [0, 1)%s", "");
    const bool drop = a->drop_p > 0.0;
    if (drop && !a->keep) return nn_fail("nn_stage_fwd: drop_p > 0 needs the keep mask buffer%s", "");
    if (drop && a->eval_mode) return nn_fail("nn_stage_fwd: dropout is the identity in eval mode (pass drop_p = 0)%s", "");
    NN_SET_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const float* bn_in = a->in;
    int HW = a->H * a->W;
    double* scratch = (double*)a->scratch;
    int splits = ST_SPLITS;
    BnFinP fin;
    fin.eps = a->eps; fin.momentum = a->momentum; fin.mean = a->mean; fin.invstd = a->invstd; fin.running_mean = a->running_mean;
    fin.running_var = a->running_var; fin.xmax_out = a->xmax_out; fin.eval_mode = a->eval_mode;
    if (a->stats_ready) {
        // mean / invstd / running statistics / *xmax_out = 0 come from the conv launch that produced `in` (fused pool + stats)
        if (a->pool) return nn_fail("nn_stage_fwd: stats_ready goes with pool = 0 (the conv launch pooled already)%s", "");
    } else if (a->pool) {
        if (!a->pooled || !a->argmax) return nn_fail("nn_stage_fwd: pooled/argmax buffers missing%s", "");
        HW = (a->H / 2) * (a->W / 2);
        splits = stage_splits((int64_t)a->B * HW);
        dim3 grid(a->C, splits);
        fin.count = (double)a->B * HW;
        k_pool_stats<<<grid, 256, 0, st>>>(a->in, a->pooled, a->argmax, scratch, fin, a->B, a->C, a->H, a->W);
        NN_LAUNCH_OK();
        bn_in = a->pooled;
    } else {
        splits = stage_splits((int64_t)a->B * HW);
        dim3 grid(a->C, splits);
        fin.count = (double)a->B * HW;
        k_chan_stats<<<grid, 256, 0, st>>>(a->in, scratch, fin, a->B, a->C, HW);
        NN_LAUNCH_OK();
    }
    BnActP p;
    p.x = bn_in; p.mean = a->mean; p.invstd = a->invstd; p.gamma = a->gamma; p.beta = a->beta; p.u_inject = a->u_inject;
    p.xp = (__nv_bfloat16*)a->xp; p.act = a->act; p.xmax_out = a->xmax_out;
    p.B = a->B; p.C = a->C; p.HW = HW; p.Cp = a->Cp; p.act_max = a->act_max;
    p.quant = a->q_bits > 0;
    double qmax = a->q_bits > 0 ? (double)((1u << a->q_bits) - 1u) : 0.0;
    double scale = a->q_bits > 0 ? a->q_hi / qmax : 1.0;
    if (scale < 1e-6) scale = 1e-6;
    p.q_scale = (float)scale; p.q_max = (float)qmax; p.stoch = a->stochastic; p.rng = a->rng;
    // dropout: k = fl(1 / fl(1 - p)) as torch forms bernoulli_(1 - p).div_(1 - p) on fp32 (noisynet.py:375-376)
    p.keep = drop ? a->keep : nullptr; p.keep_inject = drop ? a->keep_inject : nullptr;
    p.drop_p = (float)a->drop_p; p.drop_k = drop ? 1.0f / (float)(1.0 - a->drop_p) : 1.0f; p.drop_rng = a->drop_rng;
    const int64_t items = (int64_t)a->B * HW * (a->Cp / 8);
    const bool lean = ST_CHUNK_FAST && p.quant && p.stoch > 0.f && !p.u_inject && !p.keep_inject && !p.act &&
                      (int64_t)a->B * a->C * HW < ((int64_t)1 << 31) && items < ((int64_t)1 << 31);
    const size_t tile_smem = (size_t)32 * ((a->Cp / 8) | 1) * 16;
    if (lean && HW >= 32 && tile_smem <= 48 * 1024) {
        const int64_t tiles = ((int64_t)a->B * HW + 31) / 32;
        const int64_t cap = (int64_t)nn_num_sms(device) * 16;
        if (drop) k_bn_act_pack_tiled<true><<<(int)(tiles < cap ? tiles : cap), 256, tile_smem, st>>>(p);
        else k_bn_act_pack_tiled<false><<<(int)(tiles < cap ? tiles : cap), 256, tile_smem, st>>>(p);
    } else if (lean) {
        if (drop) k_bn_act_pack_lean<true><<<grid_cap(items, device), 256, 0, st>>>(p);
        else k_bn_act_pack_lean<false><<<grid_cap(items, device), 256, 0, st>>>(p);
    } else if (drop) k_bn_act_pack<true><<<grid_cap(items, device), 256, 0, st>>>(p);
    else k_bn_act_pack<false><<<grid_cap(items, device), 256, 0, st>>>(p);
    NN_LAUNCH_OK();
    return 0;
}

extern "C" int nn_stage_bwd(const nn_stage_bwd_args* a, int device, void* stream) {
    if (!a || !a->g || !a->x || !a->gyp || !a->scratch) return nn_fail("nn_stage_bwd: null argument%s", "");
    if (!(a->drop_p >= 0.0 && a->drop_p < 1.0)) return nn_fail("nn_stage_bwd: drop_p must lie in [0, 1)%s", "");
    const bool drop = a->drop_p > 0.0;
    if (drop && !a->keep) return nn_fail("nn_stage_bwd: drop_p > 0 needs the forward's keep mask%s", "");
    NN_SET_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const int PH = a->pool ? a->H / 2 : a->H, PW = a->pool ? a->W / 2 : a->W;
    BnBwdP q;
    q.g = a->g; q.x = a->x; q.mean = a->mean; q.invstd = a->invstd; q.gamma = a->gamma; q.beta = a->beta;
    q.scratch = (double*)a->scratch;
    q.dbeta = a->dbeta; q.dgamma = a->dgamma; q.B = a->B; q.C = a->C; q.HW = PH * PW; q.act_max = a->act_max;
    q.q_hi = a->q_bits > 0 ? (float)a->q_hi : 0.f;
    q.keep = drop ? a->keep : nullptr; q.drop_k = drop ? 1.0f / (float)(1.0 - a->drop_p) : 1.0f;
    const int splits = stage_splits((int64_t)a->B * PH * PW);
    dim3 grid(a->C, splits);
    if (drop) k_bn_bwd_stats<true><<<grid, 256, 0, st>>>(q);
    else k_bn_bwd_stats<false><<<grid, 256, 0, st>>>(q);
    NN_LAUNCH_OK();
    BnBwdApplyP p;
    p.g = a->g; p.x = a->x; p.mean = a->mean; p.invstd = a->invstd; p.gamma = a->gamma; p.beta = a->beta;
    p.dbeta = a->dbeta; p.dgamma = a->dgamma; p.amax = a->argmax; p.gyp = (__nv_bfloat16*)a->gyp; p.gy_f32 = a->gy_f32;
    p.B = a->B; p.C = a->C; p.OH = a->H; p.OW = a->W; p.Cp = a->Cp; p.pool = a->pool;
    p.act_max = a->act_max; p.q_hi = q.q_hi; p.inv_count = 1.f / ((float)a->B * PH * PW);
    p.keep = q.keep; p.drop_k = q.drop_k;
    if (a->pool && !a->argmax) return nn_fail("nn_stage_bwd: argmax missing%s", "");
    p.planes = a->gy_layout == NN_PACK_SHIFT ? 1 : 0;
    p.vH = p.vW = 0; p.plane_stride = 0;
    if (p.planes) {
        if (a->virt_H < a->H || a->virt_W < a->W) return nn_fail("nn_stage_bwd: virtual grid smaller than the stage input%s", "");
        p.vH = a->virt_H; p.vW = a->virt_W;
        const long long total = (long long)a->B * a->virt_H * a->virt_W;
        p.plane_stride = (total + 127) / 128 * 128;
    }
    const int64_t items = (int64_t)a->B * PH * PW * (a->Cp / 8);
    const int agrid = grid_cap(items, device);
    const bool lean = !p.gy_f32 && (int64_t)a->B * a->C * PH * PW < ((int64_t)1 << 31) && items < ((int64_t)1 << 31);
    const size_t img_bytes = (size_t)a->H * a->W * a->Cp * 2;
    if (lean && a->pool && !p.planes && img_bytes <= 48 * 1024 && PH * PW >= 16) {
        const int cap = nn_num_sms(device) * 8;
        if (drop) k_bn_bwd_apply_img<true><<<a->B < cap ? a->B : cap, 256, img_bytes, st>>>(p);
        else k_bn_bwd_apply_img<false><<<a->B < cap ? a->B : cap, 256, img_bytes, st>>>(p);
    } else if (!lean) {
        if (drop) k_bn_bwd_apply<true><<<agrid, 256, 0, st>>>(p);
        else k_bn_bwd_apply<false><<<agrid, 256, 0, st>>>(p);
    } else if (drop) {
        if (a->pool && p.planes) k_bn_bwd_apply_lean<true, true, true><<<agrid, 256, 0, st>>>(p);
        else if (a->pool) k_bn_bwd_apply_lean<true, false, true><<<agrid, 256, 0, st>>>(p);
        else if (p.planes) k_bn_bwd_apply_lean<false, true, true><<<agrid, 256, 0, st>>>(p);
        else k_bn_bwd_apply_lean<false, false, true><<<agrid, 256, 0, st>>>(p);
    } else if (a->pool && p.planes) k_bn_bwd_apply_lean<true, true, false><<<agrid, 256, 0, st>>>(p);
    else if (a->pool) k_bn_bwd_apply_lean<true, false, false><<<agrid, 256, 0, st>>>(p);
    else if (p.planes) k_bn_bwd_apply_lean<false, true, false><<<agrid, 256, 0, st>>>(p);
    else k_bn_bwd_apply_lean<false, false, false><<<agrid, 256, 0, st>>>(p);
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ data path (section 8f.4): batch assembly on the device
// noisynet.py:1232-1269 permutes the whole resident dataset every epoch (a 600 MB gather), slices a batch, crops it at a
// random offset of the zero-padded images and flips it; here the batch is gathered BY INDEX from the padded dataset with
// the crop offset / flip folded into the read, and handed to quantize1 + the NHWC pack in the same pass.
struct GatherP {
    const float* data; const int64_t* idx; const int32_t* aug_dev; int B, C, Hp, Wp, H, W, off_y, off_x, flip, Cp, quant;
    __nv_bfloat16* xp; float* act; float q_scale, q_max, stoch; const float* u_inject; nn_rng rng;
};
__global__ void __launch_bounds__(256)
k_gather_quant_pack(const GatherP p) {
    const NnRng rs = nn_rng_load(p.rng);
    const int chunks = p.Cp >> 3, HW = p.H * p.W;
    const unsigned npix = (unsigned)p.B * HW, total = npix * chunks;
    int off_y = p.off_y, off_x = p.off_x, flip = p.flip;
    if (p.aug_dev) {        // crop offset / flip of this step in device memory: a captured CUDA graph replays with new values
        off_y = min(max(p.aug_dev[0], 0), p.Hp - p.H); off_x = min(max(p.aug_dev[1], 0), p.Wp - p.W); flip = p.aug_dev[2] != 0;
    }
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const unsigned pixel = i % npix;
        const int chunk = (int)(i / npix);
        const int b = (int)(pixel / HW), r = (int)(pixel - (unsigned)b * HW);
        const int y = r / p.W, x = r - y * p.W;
        const int sx = off_x + (flip ? p.W - 1 - x : x), sy = off_y + y;
        const int64_t img = p.idx ? p.idx[b] : (int64_t)b;
        uint4 rnd[2];
        if (p.quant && p.stoch > 0.f && !p.u_inject) {
            rnd[0] = nn_philox(rs, (uint64_t)i * 2);
            if (chunk * 8 + 4 < p.C) rnd[1] = nn_philox(rs, (uint64_t)i * 2 + 1);
        }
        const uint32_t* rr = reinterpret_cast<const uint32_t*>(rnd);
        __align__(16) __nv_bfloat16 out[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = chunk * 8 + j;
            float code = 0.f;
            if (c < p.C) {
                const float v = __ldg(p.data + ((img * p.C + c) * p.Hp + sy) * p.Wp + sx);
                const int64_t o = ((int64_t)b * p.C + c) * HW + r;
                if (p.quant) {
                    code = quant_code(v, p.q_scale, p.q_max, p.stoch > 0.f ? (p.u_inject ? __ldg(p.u_inject + o) : nn_usym(rr[j], p.stoch)) : 0.f);
                    if (p.act) p.act[o] = __fmul_rn(code, p.q_scale);
                } else {
                    code = v;
                    if (p.act) p.act[o] = v;
                }
            }
            out[j] = __float2bfloat16_rn(code);
        }
        *reinterpret_cast<uint4*>(p.xp + ((size_t)pixel * p.Cp + chunk * 8)) = *reinterpret_cast<const uint4*>(out);
    }
}

extern "C" int nn_input_gather_quant_pack(const float* data, const int64_t* idx, int B, int C, int Hp, int Wp, int H, int W, int off_y,
                                          int off_x, int flip, const int32_t* aug_dev, void* xp, float* act, int Cp, int q_bits,
                                          double q_hi, float stochastic, const float* u_inject, nn_rng rng, int device, void* stream) {
    if (!data || !xp || Cp % 8 || Cp < C || off_y < 0 || off_x < 0 || off_y + H > Hp || off_x + W > Wp)
        return nn_fail("nn_input_gather_quant_pack: bad argument%s", "");
    NN_SET_DEVICE(device);
    double qmax = q_bits > 0 ? (double)((1u << q_bits) - 1u) : 0.0;
    double scale = q_bits > 0 ? q_hi / qmax : 1.0;
    if (scale < 1e-6) scale = 1e-6;
    GatherP p;
    p.data = data; p.idx = idx; p.aug_dev = aug_dev; p.B = B; p.C = C; p.Hp = Hp; p.Wp = Wp; p.H = H; p.W = W; p.off_y = off_y; p.off_x = off_x; p.flip = flip;
    p.Cp = Cp; p.quant = q_bits > 0; p.xp = (__nv_bfloat16*)xp; p.act = act; p.q_scale = (float)scale; p.q_max = (float)qmax;
    p.stoch = stochastic; p.u_inject = u_inject; p.rng = rng;
    k_gather_quant_pack<<<grid_cap((int64_t)B * H * W * (Cp / 8), device), 256, 0, (cudaStream_t)stream>>>(p);
    NN_LAUNCH_OK();
    return 0;
}

// Hot path of the first layer's input (C <= 4 channels in ONE 8-channel chunk, k-bit codes, Philox stochastic rounding, no
// fp32 copy): a thread owns FOUR consecutive pixels -- one float4 load per channel, four 16-byte code stores = 64 contiguous
// bytes -- so every thread has all its loads in flight at once (the one-item-per-trip kernel above ran two latency-bound
// rounds).  Same Philox counter per pixel and the same arithmetic: bit-identical codes.
__global__ void __launch_bounds__(256)
k_quant_pack_input4(const float* __restrict__ x, __nv_bfloat16* __restrict__ xp, int B, int C, int HW, float q_scale, float q_max,
                    float stoch, nn_rng rng) {
    const NnRng rs = nn_rng_load(rng);
    const unsigned quads = ((unsigned)B * HW) >> 2;
    for (unsigned t = blockIdx.x * blockDim.x + threadIdx.x; t < quads; t += gridDim.x * blockDim.x) {
        const unsigned pixel = t * 4u, b = pixel / (unsigned)HW, r = pixel - b * (unsigned)HW;       // HW % 4 == 0: one sample
        float4 v[4];
#pragma unroll
        for (int c = 0; c < 4; ++c)
            v[c] = c < C ? __ldg(reinterpret_cast<const float4*>(x + ((size_t)b * C + c) * HW + r)) : make_float4(0.f, 0.f, 0.f, 0.f);
        uint4 rnd[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) rnd[k] = nn_philox(rs, (uint64_t)(pixel + k) * 2);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t rr[4] = {rnd[k].x, rnd[k].y, rnd[k].z, rnd[k].w};
            __align__(16) __nv_bfloat16 out[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float code = 0.f;
                if (c < 4 && c < C) {
                    const float xv = k == 0 ? v[c].x : (k == 1 ? v[c].y : (k == 2 ? v[c].z : v[c].w));
                    code = quant_code(xv, q_scale, q_max, nn_usym(rr[c], stoch));
                }
                out[c] = __float2bfloat16_rn(code);
            }
            *reinterpret_cast<uint4*>(xp + (size_t)(pixel + k) * 8) = *reinterpret_cast<const uint4*>(out);
        }
    }
}

extern "C" int nn_input_quant_pack(const float* x, void* xp, float* act, int B, int C, int HW, int Cp, int q_bits,
                                   double q_hi, float stochastic, const float* u_inject, nn_rng rng, int device,
                                   void* stream) {
    if (!x || !xp || Cp % 8 || Cp < C) return nn_fail("nn_input_quant_pack: bad argument%s", "");
    NN_SET_DEVICE(device);
    double qmax = q_bits > 0 ? (double)((1u << q_bits) - 1u) : 0.0;
    double scale = q_bits > 0 ? q_hi / qmax : 1.0;
    if (scale < 1e-6) scale = 1e-6;
    if (q_bits > 0 && stochastic > 0.f && !u_inject && !act && Cp == 8 && C <= 4 && HW % 4 == 0 && ((uintptr_t)x % 16) == 0 &&
        (int64_t)B * HW < ((int64_t)1 << 31)) {
        k_quant_pack_input4<<<grid_cap((int64_t)B * HW / 4, device), 256, 0, (cudaStream_t)stream>>>(
            x, (__nv_bfloat16*)xp, B, C, HW, (float)scale, (float)qmax, stochastic, rng);
        NN_LAUNCH_OK();
        return 0;
    }
    k_quant_pack_input<<<grid_cap((int64_t)B * HW * (Cp / 8), device), 256, 0, (cudaStream_t)stream>>>(
        x, (__nv_bfloat16*)xp, act, B, C, HW, Cp, q_bits > 0, (float)scale, (float)qmax, stochastic, u_inject, rng);
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ input pack for the shift kernel's row-plane image
// The first layer's input as the row-plane image of k_conv_shift (nn_conv_shift_planes_bytes): P planes [plane][B][H][W][8],
// element j of plane q at pixel (b, h, w) = the code of x[b, c, h, w + kw] for kw C + c = 8 q + j, zero past the right
// edge and past KW C; optionally the NHWC code image [B,H,W,8] from the same pass.  The codes are nn_input_quant_pack's:
// same arithmetic, same Philox counter per pixel (pixel * 2, + 1 for channels 4..7), bit-identical.
struct RowsP {
    const float* x; __nv_bfloat16* xp; __nv_bfloat16* planes; const float* u_inject;
    int B, C, H, W, KW, P, quant; float q_scale, q_max, stoch; nn_rng rng;
};

// Hot path (32-wide rows, C <= 4 channels: one draw per pixel; draws from the Philox stream or none): a warp owns one image
// row, lane = column, so every load and store of the warp is one contiguous run (128 B per channel, 512 B per image), and
// the codes of the KW - 1 pixels to the right of a lane come from its neighbours by shuffle.
template <int C, int KW>
__global__ void __launch_bounds__(256)
k_quant_pack_rows32(const RowsP p) {
    constexpr int P = 2 * ((KW * C + 15) / 16);
    const NnRng rs = nn_rng_load(p.rng);
    const int lane = threadIdx.x & 31;
    const unsigned rows = (unsigned)p.B * p.H, HW = (unsigned)p.H * 32u, npix = rows * 32u;
    const unsigned warps = (gridDim.x * blockDim.x) >> 5;
    for (unsigned row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {     // warp-uniform
        const unsigned pixel = row * 32u + lane, b = row / (unsigned)p.H, r = pixel - b * HW;
        float v[C];
#pragma unroll
        for (int c = 0; c < C; ++c) v[c] = __ldg(p.x + ((size_t)b * C + c) * HW + r);
        uint32_t rr[4] = {0u, 0u, 0u, 0u};
        if (p.stoch > 0.f) {
            const uint4 rnd = nn_philox(rs, (uint64_t)pixel * 2);
            rr[0] = rnd.x; rr[1] = rnd.y; rr[2] = rnd.z; rr[3] = rnd.w;
        }
        float cd[C];
#pragma unroll
        for (int c = 0; c < C; ++c) cd[c] = quant_code(v[c], p.q_scale, p.q_max, p.stoch > 0.f ? nn_usym(rr[c], p.stoch) : 0.f);
        if (p.xp) {
            __align__(16) __nv_bfloat16 out[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) out[c] = __float2bfloat16_rn(c < C ? cd[c] : 0.f);
            *reinterpret_cast<uint4*>(p.xp + (size_t)pixel * 8) = *reinterpret_cast<const uint4*>(out);
        }
#pragma unroll
        for (int q = 0; q < P; ++q) {
            __align__(16) __nv_bfloat16 out[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int e = 8 * q + j, kw = e / C, c = e - kw * C;
                float f = 0.f;
                if (kw < KW) {
                    f = __shfl_down_sync(0xffffffffu, cd[c], kw);
                    if (lane + kw >= 32) f = 0.f;                      // past the right edge of the row
                }
                out[j] = __float2bfloat16_rn(f);
            }
            *reinterpret_cast<uint4*>(p.planes + ((size_t)q * npix + pixel) * 8) = *reinterpret_cast<const uint4*>(out);
        }
    }
}

// the code of channel c at pixel (b, r) of the input: quantized from x as k_quant_pack_input, or read from the NHWC code
// image when x is NULL
__device__ __forceinline__ float rows_code(const RowsP& p, const NnRng& rs, unsigned pixel, int b, int r, int c) {
    if (!p.x) return __bfloat162float(p.xp[(size_t)pixel * 8 + c]);
    const int64_t o = ((int64_t)b * p.C + c) * (p.H * p.W) + r;
    const float v = __ldg(p.x + o);
    if (!p.quant) return v;
    float u = 0.f;
    if (p.stoch > 0.f) {
        if (p.u_inject) u = __ldg(p.u_inject + o);
        else {
            const uint4 rnd = nn_philox(rs, (uint64_t)pixel * 2 + (c >> 2));
            const uint32_t rr[4] = {rnd.x, rnd.y, rnd.z, rnd.w};
            u = nn_usym(rr[c & 3], p.stoch);
        }
    }
    return quant_code(v, p.q_scale, p.q_max, u);
}

// every other case: a thread per pixel, each code made where it is needed
__global__ void __launch_bounds__(256)
k_quant_pack_rows(const RowsP p) {
    const NnRng rs = nn_rng_load(p.rng);
    const int HW = p.H * p.W;
    const unsigned npix = (unsigned)p.B * HW;
    for (unsigned pixel = blockIdx.x * blockDim.x + threadIdx.x; pixel < npix; pixel += gridDim.x * blockDim.x) {
        const int b = (int)(pixel / (unsigned)HW), r = (int)(pixel - (unsigned)b * HW), w = r % p.W;
        __align__(16) __nv_bfloat16 out[8];
        if (p.x && p.xp) {
            for (int c = 0; c < 8; ++c) out[c] = __float2bfloat16_rn(c < p.C ? rows_code(p, rs, pixel, b, r, c) : 0.f);
            *reinterpret_cast<uint4*>(p.xp + (size_t)pixel * 8) = *reinterpret_cast<const uint4*>(out);
        }
        for (int q = 0; q < p.P; ++q) {
            for (int j = 0; j < 8; ++j) {
                const int e = 8 * q + j, kw = e / p.C, c = e - kw * p.C;
                out[j] = __float2bfloat16_rn(kw < p.KW && w + kw < p.W ? rows_code(p, rs, pixel + kw, b, r + kw, c) : 0.f);
            }
            *reinterpret_cast<uint4*>(p.planes + ((size_t)q * npix + pixel) * 8) = *reinterpret_cast<const uint4*>(out);
        }
    }
}

extern "C" int nn_input_quant_pack_rows(const float* x, void* xp, void* planes, int B, int C, int H, int W, int KW, int q_bits,
                                        double q_hi, float stochastic, const float* u_inject, nn_rng rng, int device, void* stream) {
    if (!planes || (!x && !xp) || C < 1 || C > 8 || KW < 1 || KW > W || B < 1 || H < 1 || (int64_t)B * H * W >= ((int64_t)1 << 31))
        return nn_fail("nn_input_quant_pack_rows: bad argument%s", "");
    NN_SET_DEVICE(device);
    double qmax = q_bits > 0 ? (double)((1u << q_bits) - 1u) : 0.0;
    double scale = q_bits > 0 ? q_hi / qmax : 1.0;
    if (scale < 1e-6) scale = 1e-6;
    RowsP p;
    p.x = x; p.xp = (__nv_bfloat16*)xp; p.planes = (__nv_bfloat16*)planes; p.u_inject = u_inject;
    p.B = B; p.C = C; p.H = H; p.W = W; p.KW = KW; p.P = 2 * ((KW * C + 15) / 16); p.quant = q_bits > 0;
    p.q_scale = (float)scale; p.q_max = (float)qmax; p.stoch = stochastic; p.rng = rng;
    const int64_t npix = (int64_t)B * H * W;
    const bool hot = x && q_bits > 0 && !u_inject && W == 32;
    cudaStream_t st = (cudaStream_t)stream;
#define NN_ROWS32(CC, KK)                                                                         \
    if (hot && C == CC && KW == KK) {                                                            \
        k_quant_pack_rows32<CC, KK><<<grid_cap(npix, device), 256, 0, st>>>(p);                  \
        NN_LAUNCH_OK();                                                                          \
        return 0;                                                                                \
    }
    NN_ROWS32(3, 5) NN_ROWS32(4, 5) NN_ROWS32(1, 5) NN_ROWS32(3, 3)
#undef NN_ROWS32
    k_quant_pack_rows<<<grid_cap(npix, device), 256, 0, st>>>(p);
    NN_LAUNCH_OK();
    return 0;
}

extern "C" int nn_head_fwd_bwd(const float* logits, const int64_t* labels, int B, int C, const float* gamma,
                               const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                               float* loss_out, float* out, float* g, void* g_packed, int Cp, float* dgamma,
                               float* dbeta, int device, void* stream) {
    if (C > HEAD_MAXC || C < 1) return nn_fail("nn_head_fwd_bwd: C must be <= 16%s", "");
    if (!logits || !labels || !loss_out || !g || !dgamma || !dbeta) return nn_fail("nn_head_fwd_bwd: null argument%s", "");
    NN_SET_DEVICE(device);
    int threads = B >= 1024 ? 1024 : ((B + 31) / 32) * 32;
    if (threads < 32) threads = 32;
    const size_t hsm = ((size_t)2 * C * B + B) * sizeof(float);
    if (B <= 1024 && hsm <= 160 * 1024) {        // one thread per row, warp-per-channel reductions
        NN_ONCE_PER_DEVICE({
            NN_CUDA_OK(cudaFuncSetAttribute(k_head_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
        });
        if (threads < 32 * (C + 1) && 32 * (C + 1) <= 1024) threads = 32 * (C + 1);      // a warp per channel + the loss
        k_head_rows<<<1, threads, hsm, (cudaStream_t)stream>>>(logits, labels, B, C, gamma, beta, running_mean, running_var,
                                                              momentum, eps, loss_out, out, g, (__nv_bfloat16*)g_packed, Cp,
                                                              dgamma, dbeta);
    } else
    k_head<<<1, threads, 0, (cudaStream_t)stream>>>(logits, labels, B, C, gamma, beta, running_mean, running_var, momentum,
                                                    eps, loss_out, out, g, (__nv_bfloat16*)g_packed, Cp, dgamma, dbeta);
    NN_LAUNCH_OK();
    return 0;
}

// BatchNorm1d in eval mode on the last layer's output (noisynet.py:594 under model.eval()): the logits
__global__ void k_head_eval(const float* __restrict__ x, int B, int C, const float* __restrict__ gamma, const float* __restrict__ beta,
                            const float* __restrict__ rm, const float* __restrict__ rv, float eps, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * C) return;
    const int c = i % C;
    const float inv = (float)(1.0 / sqrt((double)rv[c] + (double)eps));
    out[i] = (x[i] - rm[c]) * inv * gamma[c] + beta[c];
}

extern "C" int nn_head_eval(const float* x, int B, int C, const float* gamma, const float* beta, const float* running_mean,
                            const float* running_var, float eps, float* out, int device, void* stream) {
    if (!x || !gamma || !beta || !running_mean || !running_var || !out || B < 1 || C < 1) return nn_fail("nn_head_eval: bad argument%s", "");
    NN_SET_DEVICE(device);
    k_head_eval<<<(B * C + 255) / 256, 256, 0, (cudaStream_t)stream>>>(x, B, C, gamma, beta, running_mean, running_var, eps, out);
    NN_LAUNCH_OK();
    return 0;
}

extern "C" int nn_classifier_tail(const nn_tail_args* a, int device, void* stream) {
    if (!a || !a->xp || !a->w_codes || !a->labels || !a->gamma || !a->beta || !a->loss_out || !a->g || !a->gx || !a->dgamma || !a->dbeta)
        return nn_fail("nn_classifier_tail: null argument%s", "");
    if (a->C < 1 || a->C > HEAD_MAXC || a->B < 1 || a->B > TAIL_CTAS * TAIL_THREADS || a->K < 1 || a->Kp < a->K || (a->Kp & 1))
        return nn_fail("nn_classifier_tail: served for C <= 16, B <= 2048, even Kp >= K%s", "");
    if (a->noise_mode < 0 || a->noise_mode > 2) return nn_fail("nn_classifier_tail: bad noise_mode%s", "");
    if (a->noise_mode != NN_NOISE_NONE && (!a->w_raw || !a->scale_dev || !(a->current > 0.f)))
        return nn_fail("nn_classifier_tail: noise needs w_raw, scale_dev and current > 0%s", "");
    NN_SET_DEVICE(device);
    TailP p;
    memset(&p, 0, sizeof(p));
    p.xp = (const __nv_bfloat16*)a->xp; p.B = a->B; p.K = a->K; p.Kp = a->Kp; p.C = a->C;
    p.R = (a->B + TAIL_CTAS - 1) / TAIL_CTAS;
    p.w_codes = a->w_codes; p.w_raw = a->w_raw;
    const float as = a->a_code_scale > 0.f ? a->a_code_scale : 1.f, ws = a->w_code_scale > 0.f ? a->w_code_scale : 1.f;
    p.y_scale = as * ws; p.s_scale = as; p.w_code_scale = ws;
    p.noise_mode = a->noise_mode; p.current = a->current; p.scale_dev = a->scale_dev; p.z_inject = a->z_inject; p.rng = a->rng;
    p.labels = a->labels; p.gamma = a->gamma; p.beta = a->beta; p.running_mean = a->running_mean; p.running_var = a->running_var;
    p.momentum = a->momentum; p.eps = a->eps; p.loss_out = a->loss_out; p.logits_out = a->logits_out; p.g = a->g;
    p.gp = (__nv_bfloat16*)a->g_packed; p.Cp_g = a->Cp_g; p.gx = a->gx; p.dgamma = a->dgamma; p.dbeta = a->dbeta;
    const int K16 = (a->K + 15) & ~15, R16 = (p.R + 15) & ~15;
    p.xs_stride = K16 + 2;                                       // bf16 per shared row: K16/2 + 1 words, odd -> conflict-free fragments
    const size_t smem = ((size_t)2 * 16 * p.xs_stride + (size_t)K16 * 16 + (size_t)R16 * p.xs_stride) * 2 +
                        (size_t)3 * R16 * 16 * sizeof(float) + 64;
    if (smem > 200 * 1024) return nn_fail("nn_classifier_tail: layer too large for one cluster%s", "");
    NN_ONCE_PER_DEVICE({
        NN_CUDA_OK(cudaFuncSetAttribute(k_classifier_tail, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    });
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(TAIL_CTAS); cfg.blockDim = dim3(TAIL_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = TAIL_CTAS; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    NN_CUDA_OK(cudaLaunchKernelEx(&cfg, k_classifier_tail, p));
    NN_LAUNCH_OK();
    return 0;
}
