// Warpgroup-MMA (wgmma, sm_90a) implicit-GEMM kernels for the fused noisy conv / linear.
//
//   D[m, n] = sum_k A[m, k] * B[n, k]        m = output pixel (b, oh, ow), k = (tap, c), n = output channel
//
// * A (im2col of the activations) is never materialised: the layer input is first packed to
//   NHWC bf16 with the channel count padded to a multiple of 8 (pack_act: this is where activations are
//   re-coded to their 4-bit integer codes in registers), and 128 producer threads gather 16-byte
//   channel chunks with cp.async (zero-fill for padding taps) straight into the 128B-swizzled K-major
//   shared-memory tile the tensor core reads.
// * B (weights) is packed once per call into the exact swizzled shared-memory image, one contiguous
//   block per (n-tile, k-block), so a single cp.async.bulk (TMA engine, mbarrier complete_tx) stages it.
//   Rows of a tile:  [ main weights n_t | g(|w_raw|) n_t | colsum(|w_raw|) 1 | zero pad ]  -> ONE
//   MMA per 16-wide k step feeds the Y, sigma^2 and power-statistic accumulators from one A tile.
// * Two consumer warpgroups (64 rows of the 128-row tile each) accumulate in registers; after the last k-block they
//   write the accumulators to a shared-memory tile (over the then idle operand ring) and run the epilogue from it: scale /
//   bias, Philox normals, sigma*z, NCHW fp32 stores.
// * Warp roles: warps 0-3 cp.async producers (warp 0 also issues the weight bulk copy), warps 4-11 the two MMA
//   warpgroups, which then run the epilogue.
// * Every mbarrier wait is bounded (clock64 watchdog): a protocol bug sets an error flag instead of
//   hanging the GPU.
#include <cuda_bf16.h>
#include <stdio.h>
#include <stdlib.h>

#include "nn_common.cuh"
#include "nn_wgmma.cuh"
#include "nn_conv_tma.h"

namespace {

constexpr int UM_BLOCK_M = 128;
constexpr int UM_BLOCK_K = 64;                       // bf16 per k-block = 128 bytes = one SWIZZLE_128B row
constexpr int UM_THREADS = 384;                     // 4 producer warps + 2 MMA / epilogue warpgroups
constexpr int UM_ACC_CH = 4;                         // 64-column accumulator chunks per warpgroup (up to 256 columns)
constexpr int UM_A_STAGE = UM_BLOCK_M * 128;         // 16 KB
constexpr int UM_MAX_NT = 120;                       // output channels per n-tile when sigma rows are present

// ------------------------------------------------------------------ kernel parameters
struct UmmaP {
    int B, H, W, Cp;               // packed input  [B, H, W, Cp] bf16
    int KH, KW, stride, pad, OH, OW;
    int M, Cout, n_t, n_mma, num_kb, stages, acc_cols;
    int main_col, sig_col, wsum_col;   // accumulator column offsets inside an n-tile, -1 = absent
    int ring_bytes;                    // max(operand ring, accumulator tile): the barriers follow
    const __nv_bfloat16* xp;
    const __nv_bfloat16* wp;       // [n_tiles][num_kb][n_mma * 64] bf16, pre-swizzled smem image
    float y_scale, s_scale;
    const float* bias;
    float* y;                      // written iff main_col >= 0 && y != nullptr
    const float* y_in;             // noise-only mode (main_col < 0): the clean output
    float* y_noisy;
    int noise_mode;
    float current;
    const float *scale_dev, *z_inject;
    float *z_export, *sigma_export, *stats;
    nn_rng rng;
    const float* mask_x;           // optional STE mask source, same NCHW shape as the output
    float mask_lo, mask_hi;
    int* err_flag;
    long long* dbg;                // optional per-CTA phase timestamps (clock64): [cta][8]
    int rows_tile;                 // valid rows per m-tile (128)
    float* partial;                // split-K (gridDim.z > 1): raw accumulators [z][n_tile][column][m_pad] instead of the epilogue
    int m_pad;
    int inc_taps;                  // producers track (tap, channel) incrementally instead of dividing per k-block
    long long* kdbg;               // optional per-k-block stamps [cta][num_kb][4]: producer woke / arrived, MMA woke / committed
    int a_tma;                     // linear layers (the im2col row of sample m is row m of a row-major matrix): A by ONE tensor-map copy
    // optional (split-K linear layers): BatchNorm batch statistics of the output from the split-K epilogue (nn_conv_fwd_args.bn_mean)
    BnFinP bn_fin;                 // bn_fin.mean != nullptr selects it
    void* bn_scratch;              // nn_stage_scratch_bytes(Cout) bytes: [Cout][16][2] double partial sums, then [Cout] arrival counters
    float* zero_out;
};
struct UmmaAMap { alignas(64) unsigned char bytes[128]; };      // CUtensorMap of the activation matrix (a_tma)

// EPI selects the epilogue at compile time: 0 = generic (every option), 1 = lean noisy (main + sigma, Philox z,
// y_noisy [+ y], no bias / mask / inject / export / stats) -- the training hot path, 2 = lean plain (y only).
// The epilogue is issue-bound (Philox + Box-Muller per output), so the hot variants carry no per-element
// option checks.
template <int EPI>
__global__ void __launch_bounds__(UM_THREADS, 1)
k_conv_umma(const UmmaP p, const __grid_constant__ UmmaAMap amap) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int S = p.stages;
    const uint32_t b_stage = (uint32_t)p.n_mma * 128u;
    const uint32_t a_base = base;
    const uint32_t b_base = base + (uint32_t)S * UM_A_STAGE;
    const uint32_t bar_base = base + (uint32_t)p.ring_bytes;        // 8-byte barriers: full[S], empty[S]
    const uint32_t full_bar = bar_base, empty_bar = bar_base + 8u * S;
    const uint32_t abort_slot = bar_base + 16u * S;
    uint8_t* gen0 = smem_raw + (base - smem_u32(smem_raw));
    volatile uint32_t* abort_g = reinterpret_cast<volatile uint32_t*>(gen0 + (abort_slot - base));
    // the accumulator tile overlays the operand ring once every MMA has retired
    const AccTile acc_tile = {reinterpret_cast<float*>(gen0), p.acc_cols + 4};

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);       // warp-uniform for the compiler (see elect_one_sync)
    const int m0 = blockIdx.x * p.rows_tile;
    const int tile_n = blockIdx.y;
    // split-K: this CTA's share of the k-blocks (gridDim.z == 1: all of them)
    const int kb_per = (p.num_kb + (int)gridDim.z - 1) / (int)gridDim.z;
    const int kb0 = (int)blockIdx.z * kb_per, kb1 = min(p.num_kb, kb0 + kb_per);
    long long* dbg = p.dbg ? p.dbg + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 8 : nullptr;
    if (dbg && tid == 0) dbg[0] = clock64();

    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full_bar + 8 * s, p.a_tma ? 2 : 128 + 1);   // 128 producer arrivals (or 1 expect_tx of the A copy) + 1 expect_tx of the weights
            mbar_init(empty_bar + 8 * s, 2);                       // both MMA warpgroups have read the stage
        }
        *abort_g = 0;
        fence_mbar_init();
    }
    __syncthreads();
    if (dbg && tid == 0) dbg[1] = clock64();

    // ================================================================ main loop roles
    const __nv_bfloat16* wt = p.wp + (size_t)tile_n * p.num_kb * p.n_mma * 64;     // this n-tile's weight blocks
    if (warp < 4 && p.a_tma) {
        // ---------------- A by the copy engine (linear layers): the 128 x 64 tile of the row-major activation matrix is one
        // cp.async.bulk.tensor.2d into the SWIZZLE_128B stage; rows >= M and columns >= K read as zeros
        if (warp == 0) {
            int s = 0;
            uint32_t ph = 1u;
            for (int kb = kb0; kb < kb1; ++kb) {
                if (!mbar_wait(empty_bar + 8 * s, ph)) { *abort_g = 1; break; }
                if (*abort_g) break;
                if (elect_one_sync()) {
                    mbar_arrive_expect_tx(full_bar + 8 * s, UM_A_STAGE);
                    tma_tile_2d(a_base + (uint32_t)s * UM_A_STAGE, &amap, full_bar + 8 * s, kb * UM_BLOCK_K, m0);
                    mbar_arrive_expect_tx(full_bar + 8 * s, b_stage);
                    bulk_g2s(b_base + (uint32_t)s * b_stage, wt + (size_t)kb * p.n_mma * 64, b_stage, full_bar + 8 * s);
                }
                __syncwarp();
                if (++s == S) { s = 0; ph ^= 1u; }
            }
        }
    } else if (warp < 4) {
        // ---------------- A producers.  Lane mapping: 8 consecutive lanes fetch the 8 consecutive 16-byte
        // chunks of ONE tile row (contiguous channels of one tap, 128 B), so a warp instruction touches 4 rows
        // = 4-8 cache lines instead of 32 (the gather is L1-wavefront-bound otherwise).  Thread t owns chunk
        // j = t % 8 of rows (t / 8) + 16 i, i = 0..7.
        const int j = tid & 7;
        int rbase[8], rih[8], riw[8];                 // per row: pixel base index (may be negative), ih0, iw0
        {
            const int ohw = p.OH * p.OW;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int m = m0 + (tid >> 3) + 16 * i;
                if (m < p.M && (tid >> 3) + 16 * i < p.rows_tile) {
                    const int b = m / ohw; const int r = m - b * ohw; const int oh = r / p.OW; const int ow = r - oh * p.OW;
                    rih[i] = oh * p.stride - p.pad; riw[i] = ow * p.stride - p.pad;
                    rbase[i] = (b * p.H + rih[i]) * p.W + riw[i];
                } else {
                    rih[i] = -100000; riw[i] = -100000; rbase[i] = 0;      // fails every bounds check -> zero fill
                }
            }
        }
        // (tap, channel offset) of this thread's chunk: divisions once, then incremental (+64 channels per k-block)
        int c0, kh, kw;
        {
            const int k = kb0 * UM_BLOCK_K + j * 8;
            const int tap = k / p.Cp;
            c0 = k - tap * p.Cp; kh = tap / p.KW; kw = tap - kh * p.KW;
        }
        int s = 0, ph = 1;                            // ring stage and the parity to wait for (no % / per k-block)
#ifdef NN_KDEBUG      // per-k-block clock stamps (tools/kblock_timeline.py): build with NN_EXTRA_NVCC=-DNN_KDEBUG
        long long* const kd0 = (p.kdbg && tid == 0) ? p.kdbg + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * p.num_kb * 4 : nullptr;
#else
        long long* const kd0 = nullptr;
#endif
        for (int kb = kb0; kb < kb1; ++kb) {
            if (!mbar_wait(empty_bar + 8 * s, ph)) { *abort_g = 1; break; }
            if (*abort_g) break;
            long long* const kd = kd0 ? kd0 + kb * 4 : nullptr;
            if (kd) kd[0] = clock64();
            const bool tap_ok = kh < p.KH;
            const int koff = kh * p.W + kw;
            const uint32_t dst0 = a_base + (uint32_t)s * UM_A_STAGE;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int row = (tid >> 3) + 16 * i;
                const int ih = rih[i] + kh, iw = riw[i] + kw;
                const bool ok = tap_ok && (unsigned)ih < (unsigned)p.H && (unsigned)iw < (unsigned)p.W;
                const uint32_t dst = dst0 + (uint32_t)row * 128u + ((((uint32_t)j) ^ (uint32_t)(row & 7)) << 4);
                const __nv_bfloat16* src = ok ? p.xp + (size_t)(rbase[i] + koff) * p.Cp + c0 : p.xp;
                cp_async_16(dst, src, ok ? 16u : 0u);
            }
            cp_async_mbar_arrive_noinc(full_bar + 8 * s);
            if (warp == 0) {                          // B: one bulk copy (TMA engine) per k-block
                if (elect_one_sync()) {
                    mbar_arrive_expect_tx(full_bar + 8 * s, b_stage);
                    bulk_g2s(b_base + (uint32_t)s * b_stage, wt + (size_t)kb * p.n_mma * 64, b_stage, full_bar + 8 * s);
                }
                __syncwarp();
            }
            if (kd) kd[1] = clock64();
            if (++s == S) { s = 0; ph ^= 1; }
            if (p.inc_taps) {
                c0 += UM_BLOCK_K;
                while (c0 >= p.Cp) { c0 -= p.Cp; if (++kw == p.KW) { kw = 0; ++kh; } }
            } else {
                const int k = (kb + 1) * UM_BLOCK_K + j * 8;
                const int tap = k / p.Cp;
                c0 = k - tap * p.Cp; kh = tap / p.KW; kw = tap - kh * p.KW;
            }
        }
        if (dbg && tid == 0) dbg[6] = clock64();
    } else {
        // ---------------- MMA warpgroups: warpgroup g owns rows 64 g .. 64 g + 63 of the tile (A descriptor + 8 KB)
        const int wg = (warp - 4) >> 2;
        const uint64_t d0 = gmma_desc_sw128(0u);
        float acc[UM_ACC_CH][32];
        int s = 0, fail = 0;
        uint32_t ph = 0u;
#ifdef NN_KDEBUG
        long long* const kd0 = p.kdbg ? p.kdbg + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * p.num_kb * 4 : nullptr;
#else
        long long* const kd0 = nullptr;
#endif
        for (int kb = kb0; kb < kb1; ++kb) {
            if (!mbar_wait(full_bar + 8 * s, ph)) { fail = 2; break; }
            long long* const kd = (kd0 && warp == 4 && lane == 0) ? kd0 + kb * 4 : nullptr;
            if (kd) kd[2] = clock64();
            fence_proxy_async();            // cp.async (generic proxy) writes -> tensor-core (async proxy) reads
            const uint32_t a_s = (a_base + (uint32_t)s * UM_A_STAGE + (uint32_t)wg * 8192u) >> 4, b_s = (b_base + (uint32_t)s * b_stage) >> 4;
            const uint64_t ad = d0 | (uint64_t)(a_s & 0x3FFFu), bd = d0 | (uint64_t)(b_s & 0x3FFFu);
            wg_fence();
#pragma unroll
            for (int k = 0; k < UM_BLOCK_K / 16; ++k)       // 64 B rows of the next 64-row chunk of B: + 8 KB = 512 units
                wg_mma<UM_ACC_CH, 0, 0>(acc, ad + 2 * k, bd + 2 * k, 512u, p.n_mma, (kb != kb0 || k != 0) ? 1 : 0);
            wg_commit();
            wg_wait_all();
            wg_fence_acc(acc);
            __syncwarp();
            if ((warp & 3) == 0 && elect_one_sync()) mbar_arrive(empty_bar + 8 * s);      // the stage may be refilled
            __syncwarp();
            if (kd) kd[3] = clock64();
            if (++s == S) { s = 0; ph ^= 1u; }
        }
        if (fail) *abort_g = (uint32_t)fail;
        named_bar_sync(1, 256);              // both warpgroups are done with the operand ring: it becomes the accumulator tile
        if (!*abort_g && kb1 > kb0) wg_acc_store(acc, acc_tile, 64 * wg, 0, p.n_mma);
        named_bar_sync(1, 256);
        if (dbg && tid == 128) dbg[2] = clock64();
    }
    // ================================================================ epilogue (the 8 MMA warps)
    if (warp < 4) {
    } else if (*abort_g) {
        if (tid == 128) nn_pipeline_abort(p.err_flag, 100 + (int)*abort_g);
    } else if (p.partial) {
        // split-K: raw fp32 accumulators, column-major per n-tile (lanes = consecutive rows: coalesced); the noise
        // epilogue runs in k_splitk_epilogue once all shares are summed.  A share without k-blocks contributes zeros.
        const int q = warp & 3, half = (warp - 4) >> 2, row = q * 32 + lane, m = m0 + row;
        const uint32_t t_lane = (uint32_t)(q * 32) << 16;
        float* dst = p.partial + (((size_t)blockIdx.z * gridDim.y + tile_n) * p.n_mma) * p.m_pad + m;
        for (int ci = half; ci * 16 < p.n_mma; ci += 2) {
            float v[16];
            acc_ld16(acc_tile, t_lane + (uint32_t)(ci * 16), v);
            if (m < p.m_pad) {
#pragma unroll
                for (int e = 0; e < 16; ++e) dst[(size_t)(ci * 16 + e) * p.m_pad] = kb1 > kb0 ? v[e] : 0.f;
            }
        }
    } else {
        const int q = warp & 3, half = (warp - 4) >> 2;
        const int row = q * 32 + lane;
        const int m = m0 + row;
        const bool row_ok = m < p.M && row < p.rows_tile;
        const int ohw = p.OH * p.OW;
        int b = 0, pix = 0;
        if (row_ok) { b = m / ohw; pix = m - b * ohw; }
        const size_t out_row = (size_t)b * p.Cout * ohw + pix;
        const uint32_t t_lane = (uint32_t)(q * 32) << 16;
        const bool noise = p.noise_mode != NN_NOISE_NONE;
        float coef = 0.f;
        NnRng rs = {0, 0, 0, 0};
        if (noise) { coef = nn_noise_coef(*p.scale_dev, p.current); rs = nn_rng_load(p.rng); }
        const int ngrp = (p.Cout + 3) >> 2;
        const int n_base = tile_n * p.n_t;
        float s_plain = 0.f, s_abs = 0.f, s_max = __int_as_float(0xff800000);
        const bool want_stats = p.stats != nullptr;
        const int nchunks = (p.n_t + 15) >> 4;
        if (EPI == 1 || EPI == 2) {
            const float y_scale = p.y_scale, s_scale = p.s_scale;
            const uint64_t grp_row = (uint64_t)m * ngrp;
            float* const out_main = (EPI == 1 ? p.y_noisy : p.y) + out_row;
            float* const out_y = (EPI == 1 && p.y) ? p.y + out_row : nullptr;
            // linear layers (one output pixel per sample): a thread's channels are contiguous in memory -> vector stores
            const bool vec4 = (ohw == 1) && ((p.Cout & 3) == 0) && (out_y == nullptr);
            for (int ci = half; ci < nchunks; ci += 2) {
                const int cc = ci * 16;
                float am[16], as[16];
                acc_ld16(acc_tile, t_lane + (uint32_t)(p.main_col + cc), am);
                if (EPI == 1) acc_ld16(acc_tile, t_lane + (uint32_t)(p.sig_col + cc), as);
                if (!row_ok) continue;
                const int nb = n_base + cc;
                const int nvalid = min(16, min(p.n_t - cc, p.Cout - nb));
                float* o = out_main + (size_t)nb * ohw;
                float* oy = out_y ? out_y + (size_t)nb * ohw : nullptr;
#pragma unroll
                for (int g4 = 0; g4 < 4; ++g4) {
                    if (g4 * 4 < nvalid) {
                        float z[4];
                        if (EPI == 1) nn_normal4(rs, grp_row + (uint64_t)((nb + g4 * 4) >> 2), z);
                        if (!vec4 && oy == nullptr && g4 * 4 + 4 <= nvalid) {
                            // hot path of the conv layers: full group, no clean-output copy -- straight-line code with
                            // one running pointer (the per-element predicates and 64-bit index maths below cost more
                            // than the noise arithmetic; same restructuring as in k_conv_shift)
                            float* o_run = o + (size_t)(g4 * 4) * ohw;
                            asm volatile("" : "+l"(o_run));
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const int e = g4 * 4 + j;
                                const float yv = am[e] * y_scale;
                                st_global_f32(o_run, (EPI == 1) ? __fadd_rn(yv, __fmul_rn(z[j], nn_sigma(coef, as[e] * s_scale))) : yv);
                                o_run += ohw;
                            }
                            continue;
                        }
                        if (vec4 && g4 * 4 + 4 <= nvalid) {
                            float r4[4];
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const int e = g4 * 4 + j;
                                const float yv = am[e] * y_scale;
                                r4[j] = (EPI == 1) ? __fadd_rn(yv, __fmul_rn(z[j], nn_sigma(coef, as[e] * s_scale))) : yv;
                            }
                            *reinterpret_cast<float4*>(o + g4 * 4) = make_float4(r4[0], r4[1], r4[2], r4[3]);
                            continue;
                        }
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int e = g4 * 4 + j;
                            if (e < nvalid) {
                                const float yv = am[e] * y_scale;
                                if (EPI == 1) {
                                    const float sg = nn_sigma(coef, as[e] * s_scale);
                                    o[(size_t)e * ohw] = __fadd_rn(yv, __fmul_rn(z[j], sg));
                                    if (oy) oy[(size_t)e * ohw] = yv;
                                } else {
                                    o[(size_t)e * ohw] = yv;
                                }
                            }
                        }
                    }
                }
            }
        } else
        for (int ci = half; ci < nchunks; ci += 2) {
            const int cc = ci * 16;
            float am[16], as[16];
            if (p.main_col >= 0) acc_ld16(acc_tile, t_lane + (uint32_t)(p.main_col + cc), am);
            if (noise) acc_ld16(acc_tile, t_lane + (uint32_t)(p.sig_col + cc), as);
            if (!row_ok) continue;
#pragma unroll
            for (int g4 = 0; g4 < 4; ++g4) {
                const int n0 = n_base + cc + g4 * 4;
                if (n0 >= p.Cout || cc + g4 * 4 >= p.n_t) continue;
                float z[4] = {0.f, 0.f, 0.f, 0.f};
                if (noise && !p.z_inject) nn_normal4(rs, (uint64_t)m * ngrp + (uint64_t)(n0 >> 2), z);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int n = n0 + j;
                    if (n >= p.Cout) continue;
                    const size_t o = out_row + (size_t)n * ohw;
                    float yv;
                    if (p.main_col >= 0) {
                        yv = am[g4 * 4 + j] * p.y_scale;
                        if (p.bias) yv = __fadd_rn(yv, __ldg(p.bias + n));
                        if (p.mask_x) { const float xv = __ldg(p.mask_x + o); if (xv > p.mask_hi || xv < p.mask_lo) yv = 0.f; }
                        if (p.y) p.y[o] = yv;
                    } else {
                        yv = __ldg(p.y_in + o);
                    }
                    if (noise) {
                        const float Sv = as[g4 * 4 + j] * p.s_scale;
                        const float sg = nn_sigma(coef, Sv);
                        const float zz = p.z_inject ? __ldg(p.z_inject + o) : z[j];
                        const float nz = __fmul_rn(zz, sg);
                        p.y_noisy[o] = __fadd_rn(yv, nz);
                        if (p.z_export) p.z_export[o] = zz;
                        if (p.sigma_export) p.sigma_export[o] = sg;
                        if (want_stats) {
                            if (p.noise_mode == NN_NOISE_MERGED) s_plain += Sv;
                            s_abs += fabsf(nz);
                            s_max = fmaxf(s_max, yv);
                        }
                    }
                }
            }
        }
        if (EPI == 0 && noise && p.stats) {
            if (p.wsum_col >= 0 && half == 0) {      // external DAC: row sum of x (*) |w| from the colsum row
                float ws[16];
                acc_ld16(acc_tile, t_lane + (uint32_t)p.wsum_col, ws);
                if (row_ok) s_plain += ws[0] * p.s_scale;
            }
            s_plain = nn_warp_sum(s_plain); s_abs = nn_warp_sum(s_abs); s_max = nn_warp_max(s_max);
            if (lane == 0) {
                atomicAdd(p.stats + 0, s_plain);
                atomicAdd(p.stats + 1, s_abs);
                nn_atomic_max_float(p.stats + 2, s_max);
            }
        }
    }
    if (dbg && tid == 128) { dbg[4] = clock64(); unsigned smid; asm volatile("mov.u32 %0, %%smid;" : "=r"(smid)); dbg[7] = smid; }
}


// Split-K second pass for linear layers (one output pixel per sample): sum the shares, then the lean noisy / plain
// epilogue of k_conv_umma with the same Philox group mapping (m * ceil(N/4) + n/4): one thread = one row m and one
// group of 4 output units.
struct SplitEpiP {
    const float* partial; int splits, n_tiles, n_mma, n_t, main_col, sig_col, m_pad, M, Cout;
    float y_scale, s_scale, current; const float* scale_dev; nn_rng rng; float *y, *y_noisy; int noisy;
    // optional: per-channel sums of the outputs (the BatchNorm1d that follows a fully connected layer, noisynet.py:540-546).
    // Needs M % 256 == 0 and one block per 256 rows of one 4-channel group: the block is slice blockIdx.x % (M / 256) of its
    // four channels; the last slice of a channel finalizes it (fixed order: deterministic).
    double* stat_partial; unsigned* stat_counters; BnFinP fin; float* zero_out;
};
__global__ void __launch_bounds__(256)
k_splitk_epilogue(const SplitEpiP p) {
    const int ngrp = (p.Cout + 3) >> 2;
    const int total = p.M * ngrp;
    float coef = 0.f;
    NnRng rs = {0, 0, 0, 0};
    if (p.noisy) { coef = nn_noise_coef(*p.scale_dev, p.current); rs = nn_rng_load(p.rng); }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int m = i % p.M, g = i / p.M;                 // m fastest: coalesced partial reads
        const int n0 = g * 4;
        const int tile = n0 / p.n_t, c0 = n0 - tile * p.n_t;   // n_t % 4 == 0 (multiple of 8): a group never straddles tiles
        float am[4] = {0.f, 0.f, 0.f, 0.f}, as[4] = {0.f, 0.f, 0.f, 0.f};
        for (int z = 0; z < p.splits; ++z) {
            const float* src = p.partial + (((size_t)z * p.n_tiles + tile) * p.n_mma) * p.m_pad + m;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                am[j] += src[(size_t)(p.main_col + c0 + j) * p.m_pad];
                if (p.noisy) as[j] += src[(size_t)(p.sig_col + c0 + j) * p.m_pad];
            }
        }
        float zz[4] = {0.f, 0.f, 0.f, 0.f};
        if (p.noisy) nn_normal4(rs, (uint64_t)m * ngrp + (uint64_t)g, zz);
        float* o = (p.noisy ? p.y_noisy : p.y) + (size_t)m * p.Cout + n0;
        float ov[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (n0 + j < p.Cout) {
                const float yv = am[j] * p.y_scale;
                ov[j] = p.noisy ? __fadd_rn(yv, __fmul_rn(zz[j], nn_sigma(coef, as[j] * p.s_scale))) : yv;
                o[j] = ov[j];
                if (p.noisy && p.y) p.y[(size_t)m * p.Cout + n0 + j] = yv;
            }
        }
        if (p.stat_partial) {
            // (the host launched exactly one trip per thread: this block = 256 consecutive rows of group g)
            __shared__ double sh[8][8];
            const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                double s1 = (double)ov[j], s2 = (double)ov[j] * (double)ov[j];
#pragma unroll
                for (int o2 = 16; o2 > 0; o2 >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o2); s2 += __shfl_xor_sync(0xffffffffu, s2, o2); }
                if (lane == 0) { sh[wi][2 * j] = s1; sh[wi][2 * j + 1] = s2; }
            }
            __syncthreads();
            if (threadIdx.x < 4 && n0 + (int)threadIdx.x < p.Cout) {
                const int j = threadIdx.x, c = n0 + j, slices = p.M >> 8, slice = (m >> 8);
                double a1 = 0.0, a2 = 0.0;
#pragma unroll
                for (int w = 0; w < 8; ++w) { a1 += sh[w][2 * j]; a2 += sh[w][2 * j + 1]; }
                double* part = p.stat_partial + (size_t)c * slices * 2;
                part[slice * 2] = a1; part[slice * 2 + 1] = a2;
                __threadfence();
                if (atomicAdd(p.stat_counters + c, 1u) == (unsigned)slices - 1u) {
                    p.stat_counters[c] = 0u;
                    __threadfence();
                    bn_finalize_channel(part, slices, 2, c, p.fin);
                    if (c == 0 && p.zero_out) *p.zero_out = 0.f;
                }
            }
        }
    }
}

// ================================================================== shift-GEMM forward (narrow-input layers)
// For a stride-1, unpadded conv whose input has <= 8 channels (the first layer: 3), the K dimension of kernel row kh is its
// KW horizontal taps x Cin channels, k = kw * Cin + c (conv1: 15 of 16).  The input arrives as a ROW-PLANE image
// (nn_conv_shift_planes_bytes): P = 2 ceil(KW Cin / 16) planes [plane][B][H][W][8], element j of plane q at pixel (b, h, w)
// being x[b, c, h, w + kw] for kw * Cin + c = 8 q + j (zero past the right edge and past KW Cin).  With the SWIZZLE_NONE
// ("interleave") K-major descriptor a core matrix is 8 rows x 16 B = 8 CONSECUTIVE PIXELS of a plane, so the im2col rows
// of kernel row kh are the plane pixels themselves, shifted by kh*W: one K = 16 wgmma per (kernel row, plane pair), its
// two 8-wide K chunks one plane apart (LBO) -- nothing is gathered.  An m-tile is 128 consecutive positions of the INPUT
// pixel grid ("virtual" outputs: positions with ow >= OW or oh >= OH are computed and dropped, 12.5 % for 32 -> 28),
// staged by P cp.async.bulk copies of (128 + (KH-1) W) pixels each.  The whole weight image ([kh][plane][row][8],
// 23 KB for conv1) stays resident in shared memory, so the CTA is persistent:
//   warps 0 .. SH_EPI_WARPS - 1 : epilogue (scale, Philox/Box-Muller noise -> NCHW stores) from a shared-memory
//              accumulator tile; warps with (warp & 3) < 2 read its rows 0-63 (half 0), the others rows 64-127 (half 1)
//   next 8 warps : two MMA warpgroups, one per 64-row half of the tile.  Each issues KH P / 2 wgmmas (conv1: 5) per column
//              pass over the accumulator width, and stores its half into the tile as soon as that half's epilogue warps
//              have released it -- so it runs up to one tile ahead of them.  The first warp of warpgroup 0 also issues
//              the bulk copies (weights once, then the A ring, which runs ahead of the tiles).
// 24 warps are 6 per SM sub-partition: a cap of 80 registers per thread, which both roles fit without spilling.
constexpr int SH_MAX_STEPS = 64;                    // K = 16 steps of a chain (kernel rows x plane pairs)
constexpr int SH_STAGES = 2;
constexpr int SH_MAX_N = 256;                       // accumulator columns
constexpr int SH_MAX_N1 = 80;                       // widest chain of one column pass (40 accumulators) under the 80-register cap
constexpr int SH_POOL_IT = 5;                       // pooled launches: 4-channel groups per epilogue warp (<= 80 channels at 16 warps)

struct ShiftP {
    int H, W, OH, OW, KH, KW, Cout;
    int n_mma, main_col, sig_col, n_steps, n_planes;
    int a_pixels, a_plane, a_stage, b_bytes, n_tiles;   // pixels / bytes per plane of an A stage, bytes per A stage, weight image bytes, m-tiles
    int acc_bufs;                                       // accumulator tiles (1 or 2): live tile i of a CTA uses tile i % acc_bufs
    long long total_pixels;
    const __nv_bfloat16 *xp, *wp;   // xp: the row-plane image, planes total_pixels apart
    float y_scale, s_scale;
    float *y, *y_noisy;
    float* pooled;            // optional: fused MaxPool2d(2,2) of the (noisy) output [B,Cout,OH/2,OW/2]; then y / y_noisy are not written
    uint8_t* pool_arg;        // window position 0..3 of the maximum (first maximum in row-major order, as nn.MaxPool2d)
    // pooled launches use BLOCK tiles: 16 image rows x 8 columns (blk = 1; the 8-pixel row groups of the A operand are one
    // image row apart, SBO = W), so that every 2x2 window lies inside one warp of the epilogue
    int blk, tiles_x, tiles_per_img, sbo_units;
    double* stat_partial;     // optional [gridDim.x][Cout][2]: per-CTA sums of the pooled values (BatchNorm statistics)
    unsigned* stat_ticket;
    BnFinP fin;               // the last CTA to finish turns the partials into mean / invstd / running statistics
    float* zero_out;
    const float* z_inject;
    float current;
    const float* scale_dev;
    nn_rng rng;
    int* err_flag;
    long long* dbg;          // optional [cta][32 tiles][SH_DBG] clock64 stamps (shift_dbg)
};

// debug stamps per tile (NN_KDEBUG builds, tools/shift_timeline.py): MMA warpgroup 0 A ready / half 0 stored, MMA warpgroup
// 1 half 1 stored, epilogue warp 0 (half 0) accumulators seen / done, epilogue warp 2 (half 1) accumulators seen / done
constexpr int SH_DBG = 8;
__device__ __forceinline__ void shift_dbg(const ShiftP& p, int i, int k) {
    if (p.dbg && i < 32) p.dbg[((size_t)blockIdx.x * 32 + i) * SH_DBG + k] = clock64();
}

// first pixel of tile t (block tiles: image b, rows 16 rb .., columns 8 cb ..)
__device__ __forceinline__ long long shift_tile_v0(const ShiftP& p, int t, int& b, int& r0, int& c0) {
    if (!p.blk) { b = 0; r0 = 0; c0 = 0; return (long long)t * UM_BLOCK_M; }
    b = t / p.tiles_per_img;
    const int rem = t - b * p.tiles_per_img, rb = rem / p.tiles_x;
    r0 = rb * 16; c0 = (rem - rb * p.tiles_x) * 8;
    return ((long long)b * p.H + r0) * p.W + c0;
}
// a tile is skipped when none of its 128 positions can be a real output (whole rows oh >= OH of one image).
// 32-bit arithmetic: the host rejects inputs with 2^31 pixels or more.
__device__ __forceinline__ bool shift_tile_live(const ShiftP& p, int t) {
    if (p.blk) {
        const int rem = t % p.tiles_per_img, rb = rem / p.tiles_x;
        return rb * 16 < p.OH && (rem - rb * p.tiles_x) * 8 < p.OW;
    }
    const unsigned v0 = (unsigned)t * UM_BLOCK_M, total = (unsigned)p.total_pixels;
    unsigned v1 = v0 + UM_BLOCK_M - 1;
    if (v1 >= total) v1 = total - 1;
    const unsigned hw = (unsigned)(p.H * p.W);
    const unsigned b0 = v0 / hw, b1 = v1 / hw;
    if (b0 != b1) return true;
    return (int)((v0 - b0 * hw) / (unsigned)p.W) < p.OH;
}

// K = 16 steps j0 .. j0 + L - 1 of a half's chain: one m64nNk16 wgmma each, committed as one group.  A: the stage's half
// at 16-byte unit a16, shifted per step (tap_tab: shift | lbo << 16); B: the step's weight rows, b_step units apart.
template <int N, int L>
__device__ __forceinline__ void shift_chain(float* acc, const uint32_t* tap_tab, uint64_t ad_t, uint32_t a16, uint64_t bd, uint32_t b_step,
                                            int j0) {
    wg_fence();
#pragma unroll
    for (int k = 0; k < L; ++k) {
        const uint32_t e = tap_tab[j0 + k];
        const uint64_t ad = ad_t | (uint64_t)((a16 + (e & 0xFFFFu)) & 0x3FFFu) | ((uint64_t)((e >> 16) & 0x3FFFu) << 16);
        wgmma_c<N, 0, 0>(acc, ad, bd + (uint64_t)(j0 + k) * b_step, j0 + k != 0);
    }
    wg_commit();
}
// the whole chain of a half (n_steps K = 16 steps, in blocks of up to 5: a 5 x 5 kernel on 2 planes is one block), drained
template <int N>
__device__ __forceinline__ void shift_half_mma(float* acc, const uint32_t* tap_tab, uint64_t ad_t, uint32_t a16, uint64_t bd, uint32_t b_step,
                                               int n_steps) {
    for (int j0 = 0; j0 < n_steps; j0 += 5) {
        switch (min(5, n_steps - j0)) {
            case 5: shift_chain<N, 5>(acc, tap_tab, ad_t, a16, bd, b_step, j0); break;
            case 4: shift_chain<N, 4>(acc, tap_tab, ad_t, a16, bd, b_step, j0); break;
            case 3: shift_chain<N, 3>(acc, tap_tab, ad_t, a16, bd, b_step, j0); break;
            case 2: shift_chain<N, 2>(acc, tap_tab, ad_t, a16, bd, b_step, j0); break;
            default: shift_chain<N, 1>(acc, tap_tab, ad_t, a16, bd, b_step, j0); break;
        }
    }
    wg_wait_all();
    wg_fence_regs<N / 2>(acc);
}
// fragments of D[64 x N] into rows row0 .. row0 + 63, columns col0 .. col0 + N - 1 of the accumulator tile
template <int N>
__device__ __forceinline__ void shift_acc_store(const float* acc, const AccTile& t, int row0, int col0) {
    const int wt = threadIdx.x & 127, l = wt & 31;
    float* r0 = t.p + (size_t)(row0 + 16 * (wt >> 5) + (l >> 2)) * t.stride + col0 + 2 * (l & 3);
    float* r1 = r0 + 8 * t.stride;
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
        *reinterpret_cast<float2*>(r0 + 8 * i) = make_float2(acc[4 * i], acc[4 * i + 1]);
        *reinterpret_cast<float2*>(r1 + 8 * i) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    }
}

// column passes of k_conv_shift's MMA warpgroup for an accumulator width of nc (a multiple of 16): the fewest equal passes of
// at most SH_MAX_N1 columns, each a multiple of 8
__host__ __device__ constexpr int shift_passes(int nc) {
    int np = 1;
    while (nc / np > SH_MAX_N1 || nc % (8 * np) != 0) ++np;
    return np;
}

// the MMA warpgroup's bulk copies of the next live tile from t_ld on into A stage s, one per plane onto the stage's full
// barrier (the ring is filled in the order it is consumed); the first warp of the warpgroup (loader) issues them
__device__ __forceinline__ void shift_load_next(const ShiftP& p, uint32_t a_base, uint32_t a_full, int s, bool loader, int& t_ld) {
    while (t_ld < p.n_tiles && !shift_tile_live(p, t_ld)) t_ld += gridDim.x;
    if (t_ld >= p.n_tiles) return;
    if (loader) {
        int tb, tr0, tc0;
        const long long v0 = shift_tile_v0(p, t_ld, tb, tr0, tc0);
        long long px = p.total_pixels - v0;
        if (px > p.a_pixels) px = p.a_pixels;
        const uint32_t bytes = (uint32_t)px * 16u;
        if (elect_one_sync()) {
            mbar_arrive_expect_tx(a_full + 8 * s, bytes * (uint32_t)p.n_planes);
            for (int q = 0; q < p.n_planes; ++q)
                bulk_g2s(a_base + (uint32_t)s * p.a_stage + (uint32_t)q * p.a_plane, p.xp + ((long long)q * p.total_pixels + v0) * 8, bytes,
                         a_full + 8 * s);
        }
        __syncwarp();
    }
    t_ld += gridDim.x;
}

// MMA warpgroup h (0 / 1) of k_conv_shift for an accumulator width of NC columns (n_mma), in column passes of at most
// SH_MAX_N1: per live tile i, the chain over rows 64 h .. 64 h + 63 of the resident operands, then -- once the half's
// epilogue warps have released it (acc_empty[buf][h], buf = i % acc_bufs) -- the fragments into those rows of
// accumulator tile buf and an arrival on acc_full[buf][h].  The two warpgroups run side by side, each up to acc_bufs
// tiles ahead of its half's epilogue warps: with two accumulator tiles the stores of tile i + 1, and the second column
// pass between them, are no longer on the epilogue's path.  The first warp
// of warpgroup 0 also issues the bulk copies: the weights once, then the A ring, refilling a stage once both chains that
// read it have completed (its own, and warpgroup 1's arrival on a_empty).  Returns a nonzero abort code when a barrier
// wait times out.
template <int NC>
__device__ __forceinline__ uint32_t shift_mma_role(const ShiftP& p, int h, uint32_t a_base, uint32_t b_base, uint32_t a_full,
                                                   uint32_t a_empty, uint32_t b_full, uint32_t acc_full, uint32_t acc_empty,
                                                   const uint32_t* tap_tab, const AccTile& acc_tile, volatile uint32_t* abort_g) {
    static_assert(SH_STAGES == 2, "k_conv_shift: stage and phase are derived from the tile count");
    constexpr int NP = shift_passes(NC), N = NC / NP;                 // NP passes of N columns
    const bool first_warp = (threadIdx.x & 127) < 32, loader = h == 0 && first_warp;
    if (loader) {
        if (elect_one_sync()) {
            mbar_arrive_expect_tx(b_full, (uint32_t)p.b_bytes);
            bulk_g2s(b_base, p.wp, (uint32_t)p.b_bytes, b_full);
        }
        __syncwarp();
    }
    // live tile i of the CTA uses stage i % 2 in phase (i / 2) % 2: nothing else about the ring is kept in registers, which the
    // chain needs; t_ld is the next live tile to load
    int t_ld = blockIdx.x;
    if (loader) {
        shift_load_next(p, a_base, a_full, 0, true, t_ld);
        shift_load_next(p, a_base, a_full, 1, true, t_ld);
    }
    if (!mbar_wait(b_full, 0)) return 2;
    const uint64_t bd0 = gmma_desc_none(b_base, (uint32_t)NC, 8u);
    const uint64_t ad_t = gmma_desc_none(0u, 0u, (uint32_t)p.sbo_units);     // A template: start address and LBO come from tap_tab
    const uint32_t b_step = 2u * NC;
    int i = 0;
    for (int t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
        if (!shift_tile_live(p, t)) continue;
        const int s = i & 1, buf = p.acc_bufs > 1 ? (i & 1) : 0;
        const uint32_t ph = ((uint32_t)i >> 1) & 1u;
        if (!mbar_wait(a_full + 8 * s, ph)) return 4;
        if (*abort_g) return 0;
        if (loader && (threadIdx.x & 31) == 0) shift_dbg(p, i, 0);
        const uint32_t a16h = ((a_base + (uint32_t)s * p.a_stage) >> 4) + (uint32_t)h * 8u * (uint32_t)p.sbo_units;   // + 8 row groups
#pragma unroll
        for (int c = 0; c < NP; ++c) {
            float acc[N / 2];
            shift_half_mma<N>(acc, tap_tab, ad_t, a16h, bd0 + (uint64_t)(c * N), b_step, p.n_steps);
            if (c == NP - 1) {          // this warpgroup's chains over stage s have completed
                if (h == 1) {
                    if (first_warp && elect_one_sync()) mbar_arrive(a_empty + 8 * s);
                    __syncwarp();
                } else if (loader) {    // refill stage s once warpgroup 1 is done with it too
                    if (!mbar_wait(a_empty + 8 * s, ph)) return 8;
                    shift_load_next(p, a_base, a_full, s, true, t_ld);
                }
            }
            if (c == 0 && !mbar_wait(acc_empty + 8 * (2 * buf + h), ((uint32_t)(i / p.acc_bufs) & 1u) ^ 1u)) return 6;
            shift_acc_store<N>(acc, acc_tile, 128 * buf + 64 * h, c * N);
        }
        __syncwarp();
        if (elect_one_sync()) mbar_arrive(acc_full + 8 * (2 * buf + h));
        __syncwarp();
        if (first_warp && (threadIdx.x & 31) == 0) shift_dbg(p, i, 1 + h);
        ++i;
    }
    return 0;
}

// MODE: 0 plain, 1 noisy (Philox z), 2 noisy with injected z (parity hook); SH_EPI_WARPS: epilogue warps, a
// multiple of 4 and at least 8 (one quarter of the tile rows per warp % 4)
template <int MODE, int SH_EPI_WARPS, bool POOL>
__global__ void __launch_bounds__((SH_EPI_WARPS + 8) * 32, 1)
k_conv_shift(const ShiftP p) {
    constexpr bool NOISY = MODE != 0;
    constexpr int SH_THREADS = (SH_EPI_WARPS + 8) * 32;      // epilogue warps, then the two MMA warpgroups
    static_assert(SH_EPI_WARPS >= 8 && SH_EPI_WARPS % 4 == 0, "the MMA warpgroups start on a warpgroup boundary");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    const uint32_t b_base = base;
    const uint32_t a_base = b_base + (uint32_t)p.b_bytes;
    const uint32_t bar_base = a_base + (uint32_t)SH_STAGES * (uint32_t)p.a_stage;
    const uint32_t a_full = bar_base, a_empty = bar_base + 8u * SH_STAGES;
    const uint32_t b_full = bar_base + 16u * SH_STAGES;
    const uint32_t acc_full = b_full + 8u, acc_empty = acc_full + 32u;          // [accumulator tile][half]
    const uint32_t abort_slot = acc_empty + 32u, tab_slot = abort_slot + 4u;
    const uint32_t pool_slot = (tab_slot + 4u * SH_MAX_STEPS + 15u) & ~15u;      // pooling exchange: [warp pair][2][8][16] floats
    const uint32_t acc_slot = pool_slot + 12u * 1024u;                            // accumulator tiles: acc_bufs x 128 rows x (n_mma + 4) floats
    uint8_t* gen0 = smem_raw + (base - smem_u32(smem_raw));
    const AccTile acc_tile = {reinterpret_cast<float*>(gen0 + (acc_slot - base)), p.n_mma + 4};
    volatile uint32_t* abort_g = reinterpret_cast<volatile uint32_t*>(gen0 + (abort_slot - base));
    uint32_t* tap_tab = reinterpret_cast<uint32_t*>(gen0 + (tab_slot - base));   // per K = 16 step: shift | lbo << 16

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);       // warp-uniform for the compiler (see elect_one_sync)
    if (tid < p.n_steps) {       // descriptor of every K = 16 step (kernel row kh, planes 2 u and 2 u + 1), in 16-byte units
        const int half = p.n_planes >> 1, kh = tid / half, u = tid - kh * half, plane = p.a_plane >> 4;
        tap_tab[tid] = (uint32_t)(2 * u * plane + kh * p.W) | ((uint32_t)plane << 16);
    }
    if (tid == 0) {
        for (int s = 0; s < SH_STAGES; ++s) { mbar_init(a_full + 8 * s, 1); mbar_init(a_empty + 8 * s, 1); }
        mbar_init(b_full, 1);
        for (int h = 0; h < 4; ++h) {
            mbar_init(acc_full + 8 * h, 4);                         // the MMA warps
            mbar_init(acc_empty + 8 * h, SH_EPI_WARPS / 2);         // the epilogue warps that read the half
        }
        *abort_g = 0;
        fence_mbar_init();
    }
    {   // the A ring starts as zeros: positions past the end of the image are never loaded, yet feed (dropped) virtual
        // outputs -- they have to be finite
        uint4* az = reinterpret_cast<uint4*>(gen0 + (a_base - base));
        const int n16 = SH_STAGES * p.a_stage / 16;
        for (int i = tid; i < n16; i += SH_THREADS) az[i] = make_uint4(0, 0, 0, 0);
        fence_proxy_async();
    }
    __syncthreads();
    const int hw = p.H * p.W;

    // role loops run on whole warps with warp-uniform control flow; one elected lane issues the single-thread instructions
    // (nn_wgmma.cuh: elect_one_sync)
    if (warp >= SH_EPI_WARPS) {
        // ---- MMA warpgroups (one per accumulator half): the chain width is fixed once per launch (every n_mma the shift plan
        // can produce)
        const int h = (warp - SH_EPI_WARPS) >> 2;
        uint32_t fail = 0;
#define NN_SHIFT_MMA(NC)                                                                                                         \
    case NC:                                                                                                                     \
        fail = shift_mma_role<NC>(p, h, a_base, b_base, a_full, a_empty, b_full, acc_full, acc_empty, tap_tab, acc_tile, abort_g); \
        break
        switch (p.n_mma) {
            NN_SHIFT_MMA(16); NN_SHIFT_MMA(32); NN_SHIFT_MMA(48); NN_SHIFT_MMA(64); NN_SHIFT_MMA(80); NN_SHIFT_MMA(96);
            NN_SHIFT_MMA(112); NN_SHIFT_MMA(128); NN_SHIFT_MMA(144); NN_SHIFT_MMA(160); NN_SHIFT_MMA(176); NN_SHIFT_MMA(192);
            NN_SHIFT_MMA(208); NN_SHIFT_MMA(224); NN_SHIFT_MMA(240); NN_SHIFT_MMA(256);
            default: fail = 7; break;
        }
#undef NN_SHIFT_MMA
        if (fail) *abort_g = fail;
    } else {
        // ---- epilogue warps: a warp reads the rows of one accumulator half
        const int q = warp & 3, jq = warp >> 2, h = q >> 1;
        constexpr int per_q = SH_EPI_WARPS / 4;
        const int ohw = p.OH * p.OW;
        const int ngrp = (p.Cout + 3) >> 2;
        float coef = 0.f;
        NnRng rs = {0, 0, 0, 0};
        if (NOISY) coef = nn_noise_coef(*p.scale_dev, p.current);
        if (MODE == 1) rs = nn_rng_load(p.rng);
        const float y_scale = p.y_scale, s_scale = p.s_scale;
        float st1[SH_POOL_IT], st2[SH_POOL_IT];          // pooled launches: per-thread sums of the pooled values it finalized
#pragma unroll
        for (int it = 0; it < SH_POOL_IT; ++it) { st1[it] = 0.f; st2[it] = 0.f; }
        const bool stamp = lane == 0 && (warp == 0 || warp == 2);      // one warp per half (shift_dbg)
        int i = 0;
        for (int t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
            if (!shift_tile_live(p, t)) continue;
            const int buf = p.acc_bufs > 1 ? (i & 1) : 0;
            if (!mbar_wait(acc_full + 8 * (2 * buf + h), (uint32_t)(i / p.acc_bufs) & 1u)) { *abort_g = 5; break; }     // this half's accumulators are in the tile
            if (*abort_g) break;
            if (stamp) shift_dbg(p, i, 3 + 2 * h);
            int b, ih, iw;
            bool row_ok;
            if (p.blk) {        // block tile: tile row = 8 * (image row in tile) + column, so a warp holds 4 rows x 8 columns
                int r0, c0;
                shift_tile_v0(p, t, b, r0, c0);
                ih = r0 + q * 4 + (lane >> 3); iw = c0 + (lane & 7);
                row_ok = ih < p.OH && iw < p.OW;
            } else {
                const unsigned v = (unsigned)t * UM_BLOCK_M + q * 32 + lane;
                b = (int)(v / (unsigned)hw);
                const int rem = (int)(v - (unsigned)b * (unsigned)hw);
                ih = (int)((unsigned)rem / (unsigned)p.W); iw = rem - ih * p.W;
                row_ok = v < (unsigned)p.total_pixels && ih < p.OH && iw < p.OW;
            }
            const int pix = ih * p.OW + iw;
            const uint64_t grp_row = (uint64_t)((long long)b * ohw + pix) * ngrp;
            const size_t out_row = (size_t)b * p.Cout * ohw + pix;
            float* const out_main = (NOISY ? p.y_noisy : p.y) + out_row;
            float* const out_y = (NOISY && p.y) ? p.y + out_row : nullptr;
            const uint32_t t_lane = (uint32_t)(128 * buf + q * 32) << 16;
            if (POOL) {
                // Fused MaxPool2d(2,2) on block tiles: the window of lane l is {l, l^1, l^8, l^9} (columns iw, iw+1 of rows
                // ih, ih+1).  The four lanes of a window SHARE the work: the lane at window position w finalizes channel w of
                // the 4-channel group -- it collects that channel from its three partners (each lane offers the channel its
                // partner wants: 3 shuffles per group instead of 12), takes the first maximum in row-major order (as
                // nn.MaxPool2d), stores ONE pooled value + window index (all 32 lanes store) and keeps ONE pair of sums for the
                // BatchNorm statistics of the stage that follows.  No shared memory, no barrier.  The first 4 * (ngrp / 4)
                // groups of a lane quarter are dealt FIXED (g4 = jq + it * per_q: their sums live in registers for the whole
                // kernel), a remaining odd group rotates over the warps with the tile index (its sums are added over all warps).
                const int PW = p.OW >> 1, PHW = (p.OH >> 1) * PW;
                const int w = (lane & 1) | ((lane >> 2) & 2);
                const bool w1 = (w & 1) != 0, w2 = (w & 2) != 0;
                const size_t pbase = (size_t)b * p.Cout * PHW + (size_t)(ih >> 1) * PW + (iw >> 1);      // same for the 4 lanes of a window
                const bool warp_live = __any_sync(0xffffffffu, row_ok);
                const int n_fix = ngrp / per_q, g_extra = n_fix * per_q;
                // window exchange + first maximum + store + statistics of one group's four values (channel w of this lane)
                auto pool_group = [&](const float (&v)[4], int nb, float& s1, float& s2) {
                    // v[w ^ k] for k = 0..3 (w is a per-thread constant: two predicates)
                    const float s01 = w1 ? v[1] : v[0], s10 = w1 ? v[0] : v[1], s23 = w1 ? v[3] : v[2], s32 = w1 ? v[2] : v[3];
                    const float own = w2 ? s23 : s01;           // v[w]
                    const float c1 = w2 ? s32 : s10;            // v[w ^ 1]: what the horizontal partner finalizes
                    const float c2 = w2 ? s01 : s23;            // v[w ^ 2]: the vertical partner
                    const float c3 = w2 ? s10 : s32;            // v[w ^ 3]: the diagonal partner
                    const float a1 = __shfl_xor_sync(0xffffffffu, c1, 1), a2 = __shfl_xor_sync(0xffffffffu, c2, 8),
                                a3 = __shfl_xor_sync(0xffffffffu, c3, 9);
                    // candidates of channel w at window positions w (own), w^1, w^2, w^3: maximum, ties to the lowest position
                    float m = own; int a = w;
                    if (a1 > m || (a1 == m && (w ^ 1) < a)) { m = a1; a = w ^ 1; }
                    if (a2 > m || (a2 == m && (w ^ 2) < a)) { m = a2; a = w ^ 2; }
                    if (a3 > m || (a3 == m && (w ^ 3) < a)) { m = a3; a = w ^ 3; }
                    if (row_ok && nb + w < p.Cout) {            // OH, OW even: a window is valid as a whole
                        const size_t o = pbase + (size_t)(nb + w) * PHW;
                        p.pooled[o] = m;
                        p.pool_arg[o] = (uint8_t)a;
                        s1 += m; s2 = fmaf(m, m, s2);
                    }
                };
                auto noisy_values = [&](const float (&am)[4], const float (&as)[4], const float (&z)[4], int nb, float (&v)[4]) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        v[j] = am[j] * y_scale;
                        if (NOISY) {
                            const float zz = MODE == 2 ? ((row_ok && nb + j < p.Cout) ? __ldg(p.z_inject + out_row + (size_t)(nb + j) * ohw) : 0.f) : z[j];
                            v[j] = __fadd_rn(v[j], __fmul_rn(zz, nn_sigma(coef, as[j] * s_scale)));
                        }
                    }
                };
#pragma unroll
                for (int it = 0; it < SH_POOL_IT; ++it) {
                    if (MODE == 1 && (it & 1) == 0 && it + 1 < SH_POOL_IT - 1) {
                        // two fixed groups per trip where there are two: one accumulator read, two independent Philox chains
                        if (it + 1 < n_fix) {
                            if (!warp_live) continue;
                            const int ga = jq + it * per_q, gb = ga + per_q;
                            float am[4], as[4], bm[4], bs[4], za[4], zb[4], va[4], vb[4];
                            acc_ld4x4(acc_tile, t_lane + (uint32_t)(p.main_col + ga * 4), t_lane + (uint32_t)(p.sig_col + ga * 4),
                                       t_lane + (uint32_t)(p.main_col + gb * 4), t_lane + (uint32_t)(p.sig_col + gb * 4), am, as, bm, bs);
                            nn_normal4(rs, grp_row + (uint64_t)ga, za);
                            nn_normal4(rs, grp_row + (uint64_t)gb, zb);
                            noisy_values(am, as, za, ga * 4, va);
                            noisy_values(bm, bs, zb, gb * 4, vb);
                            pool_group(va, ga * 4, st1[it], st2[it]);
                            pool_group(vb, gb * 4, st1[it + 1], st2[it + 1]);
                            continue;
                        }
                    } else if (MODE == 1 && (it & 1) == 1 && it < SH_POOL_IT - 1) {
                        if (it < n_fix) continue;               // done with its even neighbour
                    }
                    int g4;
                    if (it < SH_POOL_IT - 1) { g4 = jq + it * per_q; if (it >= n_fix) continue; }
                    else { g4 = g_extra; if (g4 >= ngrp || (i % per_q) != jq) continue; }
                    if (!warp_live) continue;
                    float am[4], as[4];
                    if (NOISY) acc_ld4x2(acc_tile, t_lane + (uint32_t)(p.main_col + g4 * 4), t_lane + (uint32_t)(p.sig_col + g4 * 4), am, as);
                    else acc_ld4(acc_tile, t_lane + (uint32_t)(p.main_col + g4 * 4), am);
                    const int nb = g4 * 4;
                    float z[4] = {0.f, 0.f, 0.f, 0.f};
                    if (MODE == 1) nn_normal4(rs, grp_row + (uint64_t)g4, z);
                    float v[4];
                    noisy_values(am, as, z, nb, v);
                    pool_group(v, nb, st1[it], st2[it]);
                }
            } else
            // 4-channel groups (one Philox call each), dealt round-robin to the warps of this lane quarter; the deal
            // rotates with the tile so that an uneven group count (17 for 65 channels) averages out across tiles
            {
            auto one_group = [&](int g4) {
                float am[4], as[4];
                if (NOISY) acc_ld4x2(acc_tile, t_lane + (uint32_t)(p.main_col + g4 * 4), t_lane + (uint32_t)(p.sig_col + g4 * 4), am, as);
                else acc_ld4(acc_tile, t_lane + (uint32_t)(p.main_col + g4 * 4), am);
                if (!row_ok) return;
                const int nb = g4 * 4;
                float z[4];
                if (MODE == 1) nn_normal4(rs, grp_row + (uint64_t)g4, z);
                float* o = out_main + (size_t)nb * ohw;
                if (nb + 4 <= p.Cout && (!NOISY || out_y == nullptr) && MODE != 2) {
                    float* o_run = o;
                    asm volatile("" : "+l"(o_run));      // one live 64-bit pointer per group, bumped per store
                    // hot path: full group, no clean-output copy -- straight-line code, no per-element predicates
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float yv = am[j] * y_scale;
                        st_global_f32(o_run, NOISY ? __fadd_rn(yv, __fmul_rn(z[j], nn_sigma(coef, as[j] * s_scale))) : yv);
                        o_run += ohw;
                    }
                    return;
                }
                const int nvalid = min(4, p.Cout - nb);
                float* oy = out_y ? out_y + (size_t)nb * ohw : nullptr;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (j < nvalid) {
                        const float yv = am[j] * y_scale;
                        if (NOISY) {
                            const float sg = nn_sigma(coef, as[j] * s_scale);
                            const float zz = MODE == 2 ? __ldg(p.z_inject + out_row + (size_t)(nb + j) * ohw) : z[j];
                            o[(size_t)j * ohw] = __fadd_rn(yv, __fmul_rn(zz, sg));
                            if (oy) oy[(size_t)j * ohw] = yv;
                        } else {
                            o[(size_t)j * ohw] = yv;
                        }
                    }
                }
            };
            const bool hot = MODE == 1 && out_y == nullptr;
            for (int g4 = (jq + i) % per_q; g4 < ngrp; g4 += 2 * per_q) {
                const int g4b = g4 + per_q;
                if (hot && g4b * 4 + 4 <= p.Cout) {
                    // two groups per trip: one accumulator read for both, and two independent Philox / Box-Muller chains for the
                    // scheduler to interleave (the epilogue is latency-bound: one chain per warp left it at ~0.3 IPC)
                    float am[4], as[4], bm[4], bs[4];
                    acc_ld4x4(acc_tile, t_lane + (uint32_t)(p.main_col + g4 * 4), t_lane + (uint32_t)(p.sig_col + g4 * 4),
                               t_lane + (uint32_t)(p.main_col + g4b * 4), t_lane + (uint32_t)(p.sig_col + g4b * 4), am, as, bm, bs);
                    if (!row_ok) continue;
                    float za[4], zb[4];
                    nn_normal4(rs, grp_row + (uint64_t)g4, za);
                    nn_normal4(rs, grp_row + (uint64_t)g4b, zb);
                    float* oa = out_main + (size_t)(g4 * 4) * ohw;
                    float* ob = out_main + (size_t)(g4b * 4) * ohw;
                    asm volatile("" : "+l"(oa), "+l"(ob));
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        st_global_f32(oa, __fadd_rn(am[j] * y_scale, __fmul_rn(za[j], nn_sigma(coef, as[j] * s_scale))));
                        st_global_f32(ob, __fadd_rn(bm[j] * y_scale, __fmul_rn(zb[j], nn_sigma(coef, bs[j] * s_scale))));
                        oa += ohw; ob += ohw;
                    }
                    continue;
                }
                one_group(g4);
                if (g4b < ngrp) one_group(g4b);
            }
            }
            __syncwarp();
            // this warp's rows of the half may be overwritten (t_lane holds the tile: rows 128 buf + 32 q)
            if (elect_one_sync()) mbar_arrive(acc_empty + 8 * (2 * (t_lane >> 23) + h));
            __syncwarp();
            if (stamp) shift_dbg(p, i, 4 + 2 * h);
            ++i;
        }
        if (POOL && p.stat_partial) {
            // ---- BatchNorm statistics of the pooled output: lanes -> warp -> CTA partial (fixed order), once per kernel
            float* ssum = reinterpret_cast<float*>(gen0 + (pool_slot - base));      // [epilogue warp][SH_POOL_IT][4 channels][2]
            const int w = (lane & 1) | ((lane >> 2) & 2);
#pragma unroll
            for (int it = 0; it < SH_POOL_IT; ++it) {
                float a1 = st1[it], a2 = st2[it];
#pragma unroll
                for (int o = 2; o <= 16; o <<= 1) {             // lanes of equal window position: bits 1, 2, 4 (not 3)
                    if (o == 8) continue;
                    a1 += __shfl_xor_sync(0xffffffffu, a1, o); a2 += __shfl_xor_sync(0xffffffffu, a2, o);
                }
                if ((lane & ~9) == 0) { ssum[((warp * SH_POOL_IT + it) * 4 + w) * 2] = a1; ssum[((warp * SH_POOL_IT + it) * 4 + w) * 2 + 1] = a2; }
            }
            asm volatile("bar.sync 1, %0;" ::"r"(SH_EPI_WARPS * 32) : "memory");
            const int et = tid;                                                    // epilogue thread index
            if (et < p.Cout) {
                const int g4 = et >> 2, j = et & 3, n_fix = ngrp / per_q;
                double d1 = 0.0, d2 = 0.0;
                if (g4 < n_fix * per_q) {           // fixed deal: the four lane quarters of group column wj (warps 4 wj .. 4 wj + 3)
                    const int it = g4 / per_q, wj = g4 - it * per_q;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        d1 += (double)ssum[(((wj * 4 + k) * SH_POOL_IT + it) * 4 + j) * 2];
                        d2 += (double)ssum[(((wj * 4 + k) * SH_POOL_IT + it) * 4 + j) * 2 + 1];
                    }
                } else {                            // the rotating odd group: every warp may hold a share
                    for (int k = 0; k < SH_EPI_WARPS; ++k) {
                        d1 += (double)ssum[((k * SH_POOL_IT + SH_POOL_IT - 1) * 4 + j) * 2];
                        d2 += (double)ssum[((k * SH_POOL_IT + SH_POOL_IT - 1) * 4 + j) * 2 + 1];
                    }
                }
                p.stat_partial[((size_t)blockIdx.x * p.Cout + et) * 2] = d1;
                p.stat_partial[((size_t)blockIdx.x * p.Cout + et) * 2 + 1] = d2;
                __threadfence();
            }
            asm volatile("bar.sync 1, %0;" ::"r"(SH_EPI_WARPS * 32) : "memory");
            volatile int* last_g = reinterpret_cast<volatile int*>(ssum);
            if (et == 0) *last_g = (atomicAdd(p.stat_ticket, 1u) == gridDim.x - 1) ? 1 : 0;
            asm volatile("bar.sync 1, %0;" ::"r"(SH_EPI_WARPS * 32) : "memory");
            if (*last_g) {          // the last CTA: sums over the CTAs in index order (deterministic), then the statistics
                __threadfence();
                if (et < p.Cout) bn_finalize_channel(p.stat_partial + (size_t)et * 2, (int)gridDim.x, (int64_t)p.Cout * 2, et, p.fin);
                if (et == 0) { *p.stat_ticket = 0u; if (p.zero_out) *p.zero_out = 0.f; }
            }
        } else if (p.zero_out && blockIdx.x == 0 && tid == 0) {
            *p.zero_out = 0.f;
        }
    }
    __syncthreads();
    if (*abort_g && tid == 0) nn_pipeline_abort(p.err_flag, 200 + (int)*abort_g);
}

// ------------------------------------------------------------------ operand packing
// NCHW fp32 -> NHWC bf16 with Cp (multiple of 8) channels.  inv_scale > 0: integer-code mode, the value
// written is rne(x * ... ) -- the activation's quantisation code recovered in registers (exact in bf16).
__global__ void __launch_bounds__(256)
k_pack_act(const float* __restrict__ x, __nv_bfloat16* __restrict__ xp, int B, int C, int HW, int Cp, float code_scale) {
    const int chunks = Cp >> 3;
    const int64_t total = (int64_t)B * HW * chunks;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pixel = i % ((int64_t)B * HW);          // pixel index fastest -> coalesced reads
        const int chunk = (int)(i / ((int64_t)B * HW));
        const int b = (int)(pixel / HW), p = (int)(pixel - (int64_t)b * HW);
        __align__(16) __nv_bfloat16 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = chunk * 8 + j;
            float f = 0.f;
            if (c < C) {
                f = __ldg(x + ((int64_t)b * C + c) * HW + p);
                if (code_scale > 0.f) f = rintf(__fdiv_rn(f, code_scale));
            }
            v[j] = __float2bfloat16_rn(f);
        }
        *reinterpret_cast<uint4*>(xp + (pixel * Cp + chunk * 8)) = *reinterpret_cast<const uint4*>(v);
    }
}

// Activations -> the row-plane image of the shift kernel ([plane][B][H][W][8]: element j of plane q at pixel (b, h, w) is
// x[b, c, h, w + kw] for kw Cin + c = 8 q + j; zero past the right edge and past KW Cin), codes as k_pack_act
__global__ void __launch_bounds__(256)
k_pack_act_rows(const float* __restrict__ x, __nv_bfloat16* __restrict__ xp, int B, int C, int H, int W, int KW, int planes,
                float code_scale) {
    const int64_t npix = (int64_t)B * H * W, total = npix * planes;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pixel = i % npix;
        const int q = (int)(i / npix);
        const int b = (int)(pixel / ((int64_t)H * W)), r = (int)(pixel - (int64_t)b * H * W), w = r % W;
        __align__(16) __nv_bfloat16 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = q * 8 + j, kw = k / C, c = k - kw * C;
            float f = 0.f;
            if (kw < KW && w + kw < W) {
                f = __ldg(x + ((int64_t)b * C + c) * H * W + r + kw);
                if (code_scale > 0.f) f = rintf(__fdiv_rn(f, code_scale));
            }
            v[j] = __float2bfloat16_rn(f);
        }
        *reinterpret_cast<uint4*>(xp + i * 8) = *reinterpret_cast<const uint4*>(v);
    }
}

// Weights -> pre-swizzled smem image.  mode 0 (forward): rows [main | sigma | wsum], k = tap*Cp + c reads
// w[n][c][tap].  mode 1 (dgrad): "output channel" r = input channel c_in, k = tap'*Cp + n with the taps
// flipped: reads w[n][r][KHW-1-tap'] (Cp = padded Cout).
struct PackWP {
    const float *w_eff, *w_raw;
    __nv_bfloat16* wp;
    int Cout, Cin, KHW, Cp, n_t, n_mma, num_kb, n_tiles;
    int main_col, sig_col, wsum_col, noise_mode, mode;
    int layout;                    // 0: swizzled [tile][k-block] images, 1: shift-GEMM [kh][plane][row][8] (num_kb = KH x planes)
    int sh_kw, sh_planes;          // layout 1: kernel width and planes (K chunk q of kernel row kh holds k = kw Cin + c in 8 q .. 8 q + 7)
    float w_code_scale;
    // optional in-register weight quantizer (hardware_model.py:323, :343; range [-q_hi, q_hi] symmetric): the
    // main rows are then produced from w_raw directly -- k = rne(clamp((w + q_hi)/s + u, 0, qmax)), stored as the
    // odd-integer code 2k - qmax (exact in bf16; epilogue scale s/2).  u: Philox word (idx/4, idx%4), i.e. the
    // same draw nn_quantize_fwd would make for element idx with the same rng, or u_inject[idx].
    int q_bits;
    float q_hi, q_scale, q_max, q_stoch;
    const float* u_inject;
    nn_rng rng;
    const int8_t* codes;           // optional: the quantizer's codes 2k - qmax, computed once per parameter (k_quant_codes)
    // layout 2 (NN_PACK_TMA, nn_conv_tma.cu): [n-tile][tap][group][cta rank][chunk a rows | chunk b rows], chunks of 64
    // channels (128-byte swizzled rows) plus a tail chunk of t_tail channels (32 / 64 / 128-byte rows)
    int t_nc64, t_tail, t_nc, t_wt, t_nhalf, t_tapbytes;
};

__device__ __forceinline__ float pack_main_value(const PackWP& p, const NnRng& rs, int64_t idx) {
    if (p.codes) return (float)p.codes[idx];
    if (p.q_bits > 0) {
        const float w = __ldg(p.w_raw + idx);
        float u = 0.f;
        if (p.q_stoch > 0.f) {
            if (p.u_inject) u = __ldg(p.u_inject + idx);
            else {
                const uint4 r = nn_philox(rs, (uint64_t)(idx >> 2));
                const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
                u = nn_usym(rr[idx & 3], p.q_stoch);
            }
        }
        float t = __fadd_rn(__fdiv_rn(__fadd_rn(w, p.q_hi), p.q_scale), u);
        t = rintf(fminf(fmaxf(t, 0.f), p.q_max));
        return 2.f * t - p.q_max;
    }
    float f = __ldg(p.w_eff + idx);
    if (p.w_code_scale > 0.f) f = rintf(__fdiv_rn(f, p.w_code_scale));
    return f;
}

__device__ __forceinline__ void pack_w_job(const PackWP& p, int64_t start, int64_t stride) {
    const NnRng rs = nn_rng_load(p.rng);
    const bool shift = p.layout == 1, tma = p.layout == 2;
    const int64_t total = shift ? (int64_t)p.num_kb * p.n_mma
                          : tma ? (int64_t)p.n_tiles * p.n_mma * p.KHW * (p.t_wt >> 3)
                                : (int64_t)p.n_tiles * p.num_kb * p.n_mma * 8;     // one thread per 16-byte chunk
    for (int64_t i = start; i < total; i += stride) {
        int j, r, kb, tile, kbase;
        int tap_t = 0, c_first_t = 0;
        int64_t off_t = 0;
        if (tma) {
            // consecutive lanes take consecutive TAPS of one (row, 8-channel chunk): contiguous parameter reads
            const int cpt = p.t_wt >> 3;
            tap_t = (int)(i % p.KHW);
            const int qc = (int)((i / p.KHW) % cpt);
            const int R = (int)(i / ((int64_t)p.KHW * cpt));
            tile = R / p.n_mma; r = R - tile * p.n_mma;
            c_first_t = qc * 8;
            int ci = c_first_t >> 6;
            if (ci > p.t_nc64) ci = p.t_nc64;
            const int w = ci < p.t_nc64 ? 64 : p.t_tail;
            j = (c_first_t - 64 * ci) >> 3;
            const int gi = ci >> 1, slot = ci & 1;
            const int wa = (2 * gi < p.t_nc64) ? 64 : p.t_tail;
            const int wb = (2 * gi + 1 < p.t_nc) ? ((2 * gi + 1 < p.t_nc64) ? 64 : p.t_tail) : 0;
            const int rank = r / p.t_nhalf, rr = r - rank * p.t_nhalf;
            const int swz = w == 64 ? (rr & 7) : (w == 32 ? ((rr >> 1) & 3) : ((rr >> 2) & 1));
            off_t = ((int64_t)tile * p.KHW + tap_t) * p.t_tapbytes + (int64_t)gi * (p.t_nhalf * 512) +
                    (int64_t)rank * (p.t_nhalf * 2 * (wa + wb)) + (slot ? p.t_nhalf * 2 * wa : 0) + (int64_t)rr * (2 * w) + ((j ^ swz) << 4);
            kb = 0; kbase = 0;
        } else if (shift) {
            r = (int)(i % p.n_mma); kb = (int)(i / p.n_mma); j = 0; tile = 0; kbase = 0;
        } else {
            // Thread -> 16-byte chunk, enumerated so that a warp READS contiguous parameters (the kernel was bound by
            // 4-byte loads 100 B apart: one sector per lane): the parameter tensor is [n][c][tap] with tap fastest, so
            // for KHW > 1 consecutive lanes take consecutive TAPS of one (row, 8-channel chunk) -- for each of the 8
            // channels a warp then reads KHW contiguous floats; for a transposed 1x1 (linear dgrad) consecutive lanes
            // take consecutive ROWS (= contiguous input features of one output unit).
            const int cpr = p.num_kb * 8, rows_total = p.n_tiles * p.n_mma;      // chunks per row (incl. zero padding)
            int R, qk;
            if (p.KHW > 1) {
                const int ch = p.Cp >> 3, real = p.KHW * ch;
                const int q = (int)(i % cpr);
                R = (int)(i / cpr);
                qk = q < real ? (q % p.KHW) * ch + q / p.KHW : q;
            } else if (p.mode == 1) {
                R = (int)(i % rows_total);
                qk = (int)(i / rows_total);
            } else {
                qk = (int)(i % cpr);
                R = (int)(i / cpr);
            }
            tile = R / p.n_mma; r = R - tile * p.n_mma;
            kb = qk >> 3; j = qk & 7;
            kbase = qk * 8;
        }
        __align__(16) __nv_bfloat16 v[8];
        int kind = -1, rr = 0;                       // 0 main, 1 sigma, 2 wsum
        if (p.main_col >= 0 && r >= p.main_col && r < p.main_col + p.n_t) { kind = 0; rr = r - p.main_col; }
        else if (p.sig_col >= 0 && r >= p.sig_col && r < p.sig_col + p.n_t) { kind = 1; rr = r - p.sig_col; }
        else if (p.wsum_col >= 0 && r == p.wsum_col) { kind = 2; }
        const int nrows = p.mode == 0 ? p.Cout : p.Cin;   // number of real "output" rows
        const int kdim = p.mode == 0 ? p.Cin : p.Cout;    // real channels inside a tap
        const int tap0 = tma ? tap_t : kbase / p.Cp;                    // Cp % 8 == 0: a chunk never straddles taps
        const int c_first = tma ? c_first_t : kbase - tap0 * p.Cp;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            int tap = tap0, c = c_first + e;
            if (shift) {        // k = kw Cin + c of kernel row kh; past KW Cin: zero
                const int kh = kb / p.sh_planes, k = (kb - kh * p.sh_planes) * 8 + e, kw = k / p.Cin;
                tap = kw < p.sh_kw ? kh * p.sh_kw + kw : p.KHW;
                c = k - kw * p.Cin;
            }
            float f = 0.f;
            if (tap < p.KHW && c < kdim && kind >= 0) {
                if (kind == 2) {
                    const int n_lo = tile * p.n_t, n_hi = min(nrows, n_lo + p.n_t);
                    for (int n = n_lo; n < n_hi; ++n) f += fabsf(__ldg(p.w_raw + ((int64_t)n * p.Cin + c) * p.KHW + tap));
                } else {
                    const int n = tile * p.n_t + rr;
                    if (n < nrows) {
                        if (p.mode == 0) {
                            const int64_t idx = ((int64_t)n * p.Cin + c) * p.KHW + tap;
                            if (kind == 0) {
                                f = pack_main_value(p, rs, idx);
                            } else {
                                const float a = fabsf(__ldg(p.w_raw + idx));
                                f = (p.noise_mode == NN_NOISE_MERGED) ? a : __fadd_rn(__fmul_rn(a, a), a);
                            }
                        } else {
                            const int64_t idx = ((int64_t)c * p.Cin + n) * p.KHW + (p.KHW - 1 - tap);
                            f = pack_main_value(p, rs, idx);
                        }
                    }
                }
            }
            v[e] = __float2bfloat16_rn(f);
        }
        const int64_t blk = ((int64_t)tile * p.num_kb + kb) * p.n_mma * 64;          // elements
        const int64_t off = tma ? (off_t >> 1) : (shift ? i * 8 : blk + (int64_t)r * 64 + (((j ^ (r & 7))) << 3));   // 128B swizzle
        *reinterpret_cast<uint4*>(p.wp + off) = *reinterpret_cast<const uint4*>(v);
    }
}

__global__ void __launch_bounds__(256)
k_pack_w(const PackWP p) {
    pack_w_job(p, blockIdx.x * (int64_t)blockDim.x + threadIdx.x, (int64_t)gridDim.x * blockDim.x);
}

// all weight packs of a training step (forward x layers, dgrad x layers) in ONE launch: blockIdx.y = job
constexpr int UM_MAX_PACK_JOBS = 8;
struct PackJobs { PackWP j[UM_MAX_PACK_JOBS]; };

// The weight quantizer once per parameter: 4 consecutive parameters per thread = ONE Philox call (the pack kernels
// read every parameter from several operand images -- forward rows, dgrad rows -- and were bound by re-drawing Philox
// per packed element: 21 M warp instructions per step).  codes[idx] = 2k - qmax, identical to pack_main_value.
struct CodeJob { const float* w; int8_t* codes; int64_t n; float q_hi, q_scale, q_max, q_stoch; const float* u_inject; nn_rng rng; };
struct CodeJobs { CodeJob j[UM_MAX_PACK_JOBS]; };

__global__ void __launch_bounds__(256)
k_quant_codes(const CodeJobs jobs) {
    const CodeJob& c = jobs.j[blockIdx.y];
    const NnRng rs = nn_rng_load(c.rng);
    const int64_t groups = (c.n + 3) >> 2;
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < groups; g += (int64_t)gridDim.x * blockDim.x) {
        uint4 r = make_uint4(0, 0, 0, 0);
        if (c.q_stoch > 0.f && !c.u_inject) r = nn_philox(rs, (uint64_t)g);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int64_t idx = g * 4 + e;
            if (idx < c.n) {
                float u = 0.f;
                if (c.q_stoch > 0.f) u = c.u_inject ? __ldg(c.u_inject + idx) : nn_usym(rr[e], c.q_stoch);
                float t = __fadd_rn(__fdiv_rn(__fadd_rn(__ldg(c.w + idx), c.q_hi), c.q_scale), u);
                t = rintf(fminf(fmaxf(t, 0.f), c.q_max));
                c.codes[idx] = (int8_t)(2.f * t - c.q_max);
            }
        }
    }
}

__global__ void __launch_bounds__(256)
k_pack_w_batch(const PackJobs jobs) {
    pack_w_job(jobs.j[blockIdx.y], blockIdx.x * (int64_t)blockDim.x + threadIdx.x, (int64_t)gridDim.x * blockDim.x);
}

// ------------------------------------------------------------------ wgrad on the tensor cores (MN-major operands)
//   D[n, kcol] = sum_m gy[m, n] * im2col(x)[m, kcol]      n = output channel (128 tile rows),
//   kcol = tap * Cp + c (up to 256 accumulator columns per CTA), reduction over output pixels m.
// Both operands are read from NHWC bf16 packs, i.e. contiguous along their M / N dimension: they are staged
// as MN-major SWIZZLE_128B tiles  [MN atom of 64 elements][64 reduction rows][128 B]  (LBO = MN-atom stride,
// SBO = 1024 = stride of 8 reduction rows; one UMMA_K = 16 rows = 2048 B).  Split over m across CTAs,
// partial sums to a workspace, fixed-order reduce (deterministic) that also applies the STE mask.
struct WgUP {
    int B, H, W, Cp;                 // xp  [B,H,W,Cp]       (layer input, NHWC bf16)
    int KH, KW, stride, pad, OH, OW;
    int Mpix, Cout, Coutp;           // gyp [Mpix, Coutp]    (grad_output, NHWC bf16)
    int Ktot, NT, ktot_pad;          // Ktot = KH*KW*Cp, NT = accumulator columns per CTA, ktot_pad = tiles * NT
    int num_kb, kb_per_split, stages;
    const __nv_bfloat16 *xp, *gyp;
    float* partial;                  // [splits][Cout][ktot_pad]
    int* err_flag;
};

__global__ void __launch_bounds__(UM_THREADS, 1)
k_wgrad_umma(const WgUP p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int S = p.stages;
    const uint32_t b_stage = (uint32_t)p.NT * 128u;                 // 64 rows x NT bf16
    const uint32_t a_base = base, b_base = base + (uint32_t)S * UM_A_STAGE;
    const uint32_t bar_base = b_base + (uint32_t)S * b_stage;
    const uint32_t full_bar = bar_base, empty_bar = bar_base + 8u * S;
    const uint32_t abort_slot = bar_base + 16u * S, tab_base = (abort_slot + 4 + 15u) & ~15u;
    uint8_t* gen0 = smem_raw + (base - smem_u32(smem_raw));
    volatile uint32_t* abort_g = reinterpret_cast<volatile uint32_t*>(gen0 + (abort_slot - base));
    int4* tab = reinterpret_cast<int4*>(gen0 + (tab_base - base));  // per 16-byte column chunk: {kh, kw, c0, valid}

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);       // warp-uniform for the compiler (see elect_one_sync)
    const int tile_k = blockIdx.x, tile_n = blockIdx.y, split = blockIdx.z;
    const int kb0 = split * p.kb_per_split;
    const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);
    const int nkb = max(0, kb1 - kb0);
    const int nchunk = p.NT >> 3;

    if (tid == 0) {
        for (int s = 0; s < S; ++s) { mbar_init(full_bar + 8 * s, 128); mbar_init(empty_bar + 8 * s, 2); }
        *abort_g = 0;
        fence_mbar_init();
    }
    for (int q = tid; q < nchunk; q += UM_THREADS) {
        const int kcol = tile_k * p.NT + q * 8;
        const int tap = kcol / p.Cp, c0 = kcol - tap * p.Cp;
        const int kh = tap / p.KW, kw = tap - kh * p.KW;
        tab[q] = make_int4(kh, kw, c0, (kcol < p.Ktot) ? 1 : 0);
    }
    __syncthreads();

    if (warp < 4) {
        // Lane mapping (as in the forward producer): consecutive lanes fetch consecutive 16-byte chunks of one
        // pixel row, so a warp instruction touches a few cache lines instead of 32.
        //   A (gy):     16 chunks per pixel row -> tid & 15 = chunk, rows (tid >> 4) + 8 e,  e < 8
        //   B (im2col): nchunk (8/16/32) chunks per pixel row -> tid % nchunk = chunk, rows tid/nchunk + rpp e
        const int ja = tid & 15, rowA0 = tid >> 4;
        const int qB = tid & (nchunk - 1), rppB = 128 / nchunk, rowB0 = tid / nchunk, passesB = 64 / rppB;
        const int4 tb = tab[qB];
        const int koff = tb.x * p.W + tb.y;
        const bool a_col_ok = (tile_n * 128 + ja * 8) < p.Coutp;
        const int ohw = p.OH * p.OW;
        int b0, oh0, ow0;
        {
            const int mf = kb0 * 64 + rowB0;
            b0 = mf / ohw; const int t = mf - b0 * ohw; oh0 = t / p.OW; ow0 = t - oh0 * p.OW;
        }
        auto advance = [&](int& b, int& oh, int& ow, int step) {
            if (ohw == 1) { b += step; return; }
            ow += step;
            while (ow >= p.OW) { ow -= p.OW; if (++oh == p.OH) { oh = 0; ++b; } }
        };
        for (int i = 0; i < nkb; ++i) {
            const int s = i % S;
            if (!mbar_wait(empty_bar + 8 * s, ((i / S) & 1) ^ 1)) { *abort_g = 1; break; }
            if (*abort_g) break;
            const int mblk = (kb0 + i) * 64;
            {
                const uint32_t dstA = a_base + (uint32_t)s * UM_A_STAGE + (uint32_t)(ja >> 3) * (64u * 128u);
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const int r = rowA0 + 8 * e;
                    const int m = mblk + r;
                    const bool ok = a_col_ok && m < p.Mpix;
                    const __nv_bfloat16* src = ok ? p.gyp + (size_t)m * p.Coutp + tile_n * 128 + ja * 8 : p.gyp;
                    cp_async_16(dstA + (uint32_t)r * 128u + ((((uint32_t)(ja & 7)) ^ (uint32_t)(r & 7)) << 4), src, ok ? 16u : 0u);
                }
            }
            {
                const uint32_t dstB = b_base + (uint32_t)s * b_stage + (uint32_t)(qB >> 3) * (64u * 128u);
                int b = b0, oh = oh0, ow = ow0;
                for (int e = 0; e < passesB; ++e) {
                    const int r = rowB0 + rppB * e;
                    const int m = mblk + r;
                    const int ih = oh * p.stride - p.pad + tb.x, iw = ow * p.stride - p.pad + tb.y;
                    const bool ok = tb.w && m < p.Mpix && (unsigned)ih < (unsigned)p.H && (unsigned)iw < (unsigned)p.W;
                    const __nv_bfloat16* src =
                        ok ? p.xp + ((size_t)(b * p.H + oh * p.stride - p.pad) * p.W + (ow * p.stride - p.pad) + koff) * p.Cp + tb.z
                           : p.xp;
                    cp_async_16(dstB + (uint32_t)r * 128u + ((((uint32_t)(qB & 7)) ^ (uint32_t)(r & 7)) << 4), src, ok ? 16u : 0u);
                    advance(b, oh, ow, rppB);
                }
                advance(b0, oh0, ow0, 64);
            }
            cp_async_mbar_arrive_noinc(full_bar + 8 * s);
        }
    } else {
        // MMA warpgroups: MN-major A and B, bf16 x bf16 -> fp32; warpgroup g owns rows (output channels) 64 g .. 64 g + 63 =
        // the second 64-element MN atom of A (+ 8 KB); the 64-column chunks of N are B's MN atoms (LBO = 8192 B)
        const int wg = (warp - 4) >> 2;
        const uint64_t d0 = gmma_desc(0u, (64u * 128u) >> 4, 1024u >> 4, 1u);
        float acc[UM_ACC_CH][32];
        int s = 0, fail = 0;
        uint32_t ph = 0u;
        for (int i = 0; i < nkb; ++i) {
            if (!mbar_wait(full_bar + 8 * s, ph)) { fail = 2; break; }
            fence_proxy_async();
            const uint32_t a_s = (a_base + (uint32_t)s * UM_A_STAGE + (uint32_t)wg * 8192u) >> 4, b_s = (b_base + (uint32_t)s * b_stage) >> 4;
            const uint64_t ad = d0 | (uint64_t)(a_s & 0x3FFFu), bd = d0 | (uint64_t)(b_s & 0x3FFFu);
            wg_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)                                  // 16 reduction rows = 2048 B = 128 units
                wg_mma<UM_ACC_CH, 1, 1>(acc, ad + 128 * k, bd + 128 * k, 512u, p.NT, (i | k) != 0 ? 1 : 0);
            wg_commit();
            wg_wait_all();
            wg_fence_acc(acc);
            __syncwarp();
            if ((warp & 3) == 0 && elect_one_sync()) mbar_arrive(empty_bar + 8 * s);
            __syncwarp();
            if (++s == S) { s = 0; ph ^= 1u; }
        }
        if (fail) *abort_g = (uint32_t)fail;
        if (*abort_g) {
            if (warp == 4 && lane == 0) nn_pipeline_abort(p.err_flag, 200 + (int)*abort_g);
        } else {
            // rows = output channels, columns = this CTA's (tap, channel) columns: partial[split][n][tile_k * NT + col]
            const int wt = tid & 127;
            const int n0 = tile_n * 128 + 64 * wg + 16 * (wt >> 5) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = n0 + 8 * h;
                if (n >= p.Cout) continue;
                float* out = p.partial + ((size_t)split * p.Cout + n) * p.ktot_pad + (size_t)tile_k * p.NT + c0;
#pragma unroll
                for (int c = 0; c < UM_ACC_CH; ++c)
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        if (64 * c + 8 * j < p.NT)
                            *reinterpret_cast<float2*>(out + 64 * c + 8 * j) =
                                nkb > 0 ? make_float2(acc[c][4 * j + 2 * h], acc[c][4 * j + 2 * h + 1]) : make_float2(0.f, 0.f);
            }
        }
    }
}

// ================================================================== shift-GEMM wgrad (narrow-input layers)
//   gw[n][c][kh][kw] = sum over pixels  gy[pixel][n] * x[pixel + kh*W + kw][c]
// with BOTH operands read in place through SWIZZLE_NONE MN-major descriptors (core matrix = 8 reduction rows x
// 16 B, the rows 16 B apart = consecutive pixels):
//   * x is the layer's NHWC pack with 8 channels = 16 B per pixel; the five taps of one kernel row are five
//     "MN atoms" ONE PIXEL (16 B) apart, so one MMA per kernel row covers (kw, c) = N = 48 columns (the sixth
//     atom is a harmless extra tap) from a start address shifted by kh*W pixels;
//   * grad_output comes in the PLANES layout [channel chunk][virtual pixel][8] on the INPUT pixel grid (zeros at
//     positions that are not outputs; written once per step by the stage backward, NN_PACK_SHIFT), so a chunk
//     of 128 pixels is one contiguous 2 KB slab per channel chunk and the M atoms are the planes.
// Nothing is gathered: per 128-pixel reduction chunk the loader issues 9 + 1 bulk copies (23 KB), the two MMA
// warpgroups (64 output channels each) 8 x KH wgmmas, and the CTA (persistent, split over the reduction) keeps its
// accumulators in registers until the end -- kernel rows in passes of up to 256 columns (one pass for 5 x 5).
constexpr int WS_KP = 128;                 // reduction pixels per stage
constexpr int WS_MAX_STAGES = 6;
constexpr int WS_THREADS = 288;            // warps 0-7 MMA warpgroups (then the epilogue), warp 8 loader

struct WgShiftP {
    int H, W, OH, OW, KH, KW, Cout;
    int n_planes, n_row, n_chunks;          // gy channel chunks, accumulator columns per kernel row, reduction chunks
    int b_pixels, a_stage, b_stage, stages;
    long long total_pixels, plane_stride;   // plane_stride = total_pixels rounded up to WS_KP (zeros in the padding)
    const __nv_bfloat16 *xp, *gyv;
    float* partial;                         // [gridDim.x][Cout][row_pitch], column tap * 8 + c
    int row_pitch;
    int* err_flag;
    long long* dbg;                         // optional [cta][32 chunks][4]: before wait, operands landed, MMAs issued
};

__device__ __forceinline__ bool wgshift_chunk_live(const WgShiftP& p, int t) {
    const long long v0 = (long long)t * WS_KP;
    long long v1 = v0 + WS_KP - 1;
    if (v1 >= p.total_pixels) v1 = p.total_pixels - 1;
    const int hw = p.H * p.W;
    const long long b0 = v0 / hw, b1 = v1 / hw;
    if (b0 != b1) return true;
    return (int)((v0 - b0 * hw) / p.W) < p.OH;
}

// NROW: accumulator columns per kernel row (KW taps x 8 channels, padded to 16)
template <int NROW>
__global__ void __launch_bounds__(WS_THREADS, 1)
k_wgrad_shift(const WgShiftP p) {
    constexpr int KHB = 256 / NROW;          // kernel rows per pass (registers: KHB * NROW / 2 <= 128 per thread)
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    const int WS_STAGES = p.stages;
    const uint32_t b_base = base;
    const uint32_t a_base = b_base + (uint32_t)WS_STAGES * (uint32_t)p.b_stage;
    const uint32_t bar_base = a_base + (uint32_t)WS_STAGES * (uint32_t)p.a_stage + 16u * WS_KP * 16u;   // + phantom planes
    const uint32_t full_bar = bar_base, empty_bar = bar_base + 8u * WS_MAX_STAGES;
    const uint32_t abort_slot = bar_base + 16u * WS_MAX_STAGES;
    uint8_t* gen0 = smem_raw + (base - smem_u32(smem_raw));
    volatile uint32_t* abort_g = reinterpret_cast<volatile uint32_t*>(gen0 + (abort_slot - base));
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);       // warp-uniform for the compiler (see elect_one_sync)
    if (tid == 0) {
        for (int s = 0; s < WS_STAGES; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 2); }
        *abort_g = 0;
        fence_mbar_init();
    }
    {   // zero both rings once: x pixels past the end of the pack are never loaded but are multiplied by zero
        // grad_output entries, and the phantom planes beyond the real channel chunks feed unused accumulator rows
        uint4* z = reinterpret_cast<uint4*>(gen0);
        const int n16 = (int)((bar_base - base) / 16);
        for (int i = tid; i < n16; i += WS_THREADS) z[i] = make_uint4(0, 0, 0, 0);
        fence_proxy_async();
    }
    __syncthreads();

    if (warp == 8) {
        int s = 0;
        uint32_t ph = 1u;
        for (int kh0 = 0; kh0 < p.KH; kh0 += KHB)              // one sweep over the reduction per pass
            for (int t = blockIdx.x; t < p.n_chunks; t += gridDim.x) {
                if (!wgshift_chunk_live(p, t)) continue;
                if (!mbar_wait(empty_bar + 8 * s, ph)) { *abort_g = 1; break; }
                if (*abort_g) break;
                const long long v0 = (long long)t * WS_KP;
                const long long pa = WS_KP;              // planes are padded to a multiple of WS_KP pixels
                long long pb = p.total_pixels - v0;
                if (pb > p.b_pixels) pb = p.b_pixels;
                if (elect_one_sync()) {
                    mbar_arrive_expect_tx(full_bar + 8 * s, (uint32_t)(pa * 16 * p.n_planes + pb * 16));
                    bulk_g2s(b_base + (uint32_t)s * p.b_stage, p.xp + v0 * 8, (uint32_t)pb * 16u, full_bar + 8 * s);
                    for (int c = 0; c < p.n_planes; ++c)
                        bulk_g2s(a_base + (uint32_t)s * p.a_stage + (uint32_t)c * (WS_KP * 16u),
                                 p.gyv + ((long long)c * p.plane_stride + v0) * 8, (uint32_t)pa * 16u, full_bar + 8 * s);
                }
                __syncwarp();
                if (++s == WS_STAGES) { s = 0; ph ^= 1u; }
            }
    } else {
        // MN-major A (grad_output planes: SBO = plane stride, LBO = 8 pixels) and B (x: the taps of a kernel row are MN atoms
        // one pixel apart), bf16 x bf16 -> fp32; warpgroup g owns output channels 64 g .. 64 g + 63 (planes 8 g ..)
        const int wg = warp >> 2, wt = tid & 127;
        const int n0 = 64 * wg + 16 * (wt >> 5) + (lane >> 2), c0 = 2 * (lane & 3);
        int s = 0;
        uint32_t ph = 0u;
        for (int kh0 = 0; kh0 < p.KH && !*abort_g; kh0 += KHB) {
            const int nkh = min(KHB, p.KH - kh0);
            float acc[KHB][NROW / 2];
            int i = 0;
            for (int t = blockIdx.x; t < p.n_chunks; t += gridDim.x) {
                if (!wgshift_chunk_live(p, t)) continue;
                if (!mbar_wait(full_bar + 8 * s, ph)) { *abort_g = 2; break; }
                if (*abort_g) break;
                const uint64_t ad0 = gmma_desc_none(a_base + (uint32_t)s * p.a_stage + (uint32_t)wg * 8u * (WS_KP * 16u), 8u, (uint32_t)WS_KP);
                const uint64_t bd0 = gmma_desc_none(b_base + (uint32_t)s * p.b_stage + (uint32_t)kh0 * (uint32_t)p.W * 16u, 8u, 1u);
                wg_fence();
#pragma unroll 1
                for (int k = 0; k < WS_KP / 16; ++k) {
#pragma unroll
                    for (int j = 0; j < KHB; ++j)
                        if (j < nkh)
                            wgmma_c<NROW, 1, 1>(acc[j], ad0 + (uint64_t)(k * 16), bd0 + (uint64_t)(k * 16 + j * p.W), (i | k) != 0);
                }
                wg_commit();
                wg_wait_all();
#pragma unroll
                for (int j = 0; j < KHB; ++j) wg_fence_regs<NROW / 2>(acc[j]);
                __syncwarp();
                if ((warp & 3) == 0 && elect_one_sync()) mbar_arrive(empty_bar + 8 * s);
                __syncwarp();
                ++i;
                if (++s == WS_STAGES) { s = 0; ph ^= 1u; }
            }
            if (*abort_g) break;
            // accumulator rows = output channels; columns (kh, kw, c) -> partial[cta][n][tap * 8 + c] (row pitch 256:
            // k_wgrad_tma_reduce's tail format); a CTA without live chunks contributes zeros
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = n0 + 8 * h;
                if (n >= p.Cout) continue;
                float* dst = p.partial + ((size_t)blockIdx.x * p.Cout + n) * p.row_pitch + c0;
#pragma unroll
                for (int j = 0; j < KHB; ++j)
#pragma unroll
                    for (int kw = 0; kw < NROW / 8; ++kw)
                        if (j < nkh && kw < p.KW)
                            *reinterpret_cast<float2*>(dst + ((kh0 + j) * p.KW + kw) * 8) =
                                i > 0 ? make_float2(acc[j][4 * kw + 2 * h], acc[j][4 * kw + 2 * h + 1]) : make_float2(0.f, 0.f);
            }
        }
    }
    __syncthreads();
    if (*abort_g && tid == 0) nn_pipeline_abort(p.err_flag, 300 + (int)*abort_g);
}

// grad_output NCHW fp32 -> planes layout on the input pixel grid (zeros elsewhere), for callers that did not
// get it from nn_stage_bwd
__global__ void __launch_bounds__(256)
k_pack_gy_planes(const float* __restrict__ gy, __nv_bfloat16* __restrict__ gyv, int B, int C, int H, int W, int OH, int OW,
                 int n_planes, int64_t plane_stride) {
    const int64_t npix = (int64_t)B * H * W, total = plane_stride * n_planes;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pixel = i % plane_stride;
        const int chunk = (int)(i / plane_stride);
        const int b = (int)(pixel / (H * W)), r = (int)(pixel - (int64_t)b * H * W);
        const int ih = r / W, iw = r - ih * W;
        __align__(16) __nv_bfloat16 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = chunk * 8 + j;
            float f = 0.f;
            if (pixel < npix && c < C && ih < OH && iw < OW) f = __ldg(gy + (((int64_t)b * C + c) * OH + ih) * OW + iw);
            v[j] = __float2bfloat16_rn(f);
        }
        *reinterpret_cast<uint4*>(gyv + i * 8) = *reinterpret_cast<const uint4*>(v);
    }
}

// partial [splits][Cout][ktot_pad] (kcol = tap*Cp + c) -> gw [Cout][Cin][KHW], scale, STE mask.  Block = 32 columns
// x 8 split groups: group g sums splits g, g+8, ... (coalesced along kcol), then the 8 group sums are added in a
// fixed order through shared memory -- deterministic, and the serial chain over splits is 8x shorter.
__global__ void __launch_bounds__(256)
k_wgrad_umma_reduce2(const float* __restrict__ partial, int splits, int Cout, int Cin, int KHW, int Cp, int ktot_pad,
                     float scale, float* __restrict__ gw, const float* __restrict__ w_raw, float lo, float hi) {
    __shared__ float sh[8][32];
    const unsigned total = (unsigned)Cout * ktot_pad;
    const size_t zstride = (size_t)Cout * ktot_pad;
    const int col = threadIdx.x & 31, grp = threadIdx.x >> 5;
    for (unsigned base = blockIdx.x * 32u; base < total; base += gridDim.x * 32u) {
        const unsigned i = base + col;
        float s = 0.f;
        if (i < total)
            for (int z = grp; z < splits; z += 8) s += partial[(size_t)z * zstride + i];
        sh[grp][col] = s;
        __syncthreads();
        if (grp == 0 && i < total) {
            float t = sh[0][col];
#pragma unroll
            for (int g = 1; g < 8; ++g) t += sh[g][col];
            const int n = (int)(i / ktot_pad), kcol = (int)(i - (unsigned)n * ktot_pad);
            const int tap = kcol / Cp, c = kcol - tap * Cp;
            if (tap < KHW && c < Cin) {
                t *= scale;
                const size_t o = ((size_t)n * Cin + c) * KHW + tap;
                if (w_raw) { const float w = __ldg(w_raw + o); if (w > hi || w < lo) t = 0.f; }
                gw[o] = t;
            }
        }
        __syncthreads();
    }
}

// few splits / many columns: one thread per (n, kcol), splits summed sequentially (coalesced along kcol)
__global__ void __launch_bounds__(256)
k_wgrad_umma_reduce(const float* __restrict__ partial, int splits, int Cout, int Cin, int KHW, int Cp, int ktot_pad,
                    float scale, float* __restrict__ gw, const float* __restrict__ w_raw, float lo, float hi) {
    const unsigned total = (unsigned)Cout * ktot_pad;
    const size_t zstride = (size_t)Cout * ktot_pad;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int n = (int)(i / ktot_pad), kcol = (int)(i - (unsigned)n * ktot_pad);
        const int tap = kcol / Cp, c = kcol - tap * Cp;
        if (tap >= KHW || c >= Cin) continue;
        float s = 0.f;
        for (int z = 0; z < splits; ++z) s += partial[(size_t)z * zstride + i];
        s *= scale;
        const size_t o = ((size_t)n * Cin + c) * KHW + tap;
        if (w_raw) { const float w = __ldg(w_raw + o); if (w > hi || w < lo) s = 0.f; }
        gw[o] = s;
    }
}

// partials of k_wgrad_tma -> gw [Cout][Cin][KHW], scale, STE mask.  Fixed summation order: deterministic.
//   main [splits][Cout][cols_pad]:       column = (tap * n_c64 + chunk) * 64 + e   <->  channel chunk * 64 + e
//   tail [n_tail][Cout][256] (optional): column = tap * 8 + e                      <->  channel n_c64 * 64 + e
// One thread = four consecutive columns (float4 loads) of one group of partials; a block = (256 / G) column quads x G
// groups, the G group sums are added in fixed order through shared memory.  G is picked per region so that each has
// ~10^5 threads with a handful of independent 16-byte loads each (the partials sit in L2: the kernel is latency-bound).
struct WgRedP {
    const float *main, *tail;
    int splits, n_tail, Cout, Cin, KHW, n_c64, cols_pad, nb_main, g_main, g_tail;
    float scale, lo, hi;
    float* gw;
    const float* w_raw;
};

__global__ void __launch_bounds__(256)
k_wgrad_tma_reduce(const WgRedP p) {
    __shared__ float4 sh[256];
    const bool is_tail = (int)blockIdx.x >= p.nb_main;
    const int G = is_tail ? p.g_tail : p.g_main, qpb = 256 / G;                  // G: power of two <= 32
    const int row = is_tail ? 256 : p.cols_pad, cnt = is_tail ? p.n_tail : p.splits;
    const float* src0 = is_tail ? p.tail : p.main;
    const int g = threadIdx.x / qpb, ql = threadIdx.x - g * qpb;
    const int quad = ((int)blockIdx.x - (is_tail ? p.nb_main : 0)) * qpb + ql;
    const int quads_row = row >> 2, total = p.Cout * quads_row;
    const size_t zstride = (size_t)p.Cout * row;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    int n = 0, col = 0, tap = 0, c0 = 0;
    bool live = false;
    if (quad < total) {
        n = quad / quads_row; col = (quad - n * quads_row) * 4;
        if (is_tail) { tap = col >> 3; c0 = p.n_c64 * 64 + (col & 7); }
        else { const int ga = col >> 6; tap = ga / p.n_c64; c0 = (ga - tap * p.n_c64) * 64 + (col & 63); }
        live = tap < p.KHW && c0 < p.Cin;
    }
    if (live) {
        const float4* src = reinterpret_cast<const float4*>(src0 + (size_t)n * row + col);
        const size_t zs4 = zstride >> 2;
        int z = g;
        for (; z + 3 * G < cnt; z += 4 * G) {
            const float4 a = __ldcg(src + (size_t)z * zs4), b = __ldcg(src + (size_t)(z + G) * zs4);
            const float4 c = __ldcg(src + (size_t)(z + 2 * G) * zs4), d = __ldcg(src + (size_t)(z + 3 * G) * zs4);
            s.x += (a.x + b.x) + (c.x + d.x); s.y += (a.y + b.y) + (c.y + d.y);
            s.z += (a.z + b.z) + (c.z + d.z); s.w += (a.w + b.w) + (c.w + d.w);
        }
        for (; z < cnt; z += G) { const float4 a = __ldcg(src + (size_t)z * zs4); s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w; }
    }
    if (G > 1) {
        sh[threadIdx.x] = s;
        __syncthreads();
        if (g != 0) return;
        for (int k = 1; k < G; ++k) { const float4 a = sh[k * qpb + ql]; s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w; }
    }
    if (!live) return;
    if (p.KHW == 1 && (p.Cin & 3) == 0 && (((uintptr_t)p.gw | (uintptr_t)p.w_raw) & 15) == 0) {
        // fully connected layers: the four columns are contiguous in gw
        const size_t o = (size_t)n * p.Cin + c0;
        float4 t = make_float4(s.x * p.scale, s.y * p.scale, s.z * p.scale, s.w * p.scale);
        if (p.w_raw) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(p.w_raw + o));
            if (w.x > p.hi || w.x < p.lo) t.x = 0.f;
            if (w.y > p.hi || w.y < p.lo) t.y = 0.f;
            if (w.z > p.hi || w.z < p.lo) t.z = 0.f;
            if (w.w > p.hi || w.w < p.lo) t.w = 0.f;
        }
        *reinterpret_cast<float4*>(p.gw + o) = t;
        return;
    }
    const float v[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        if (c0 + e >= p.Cin) break;
        float t = v[e] * p.scale;
        const size_t o = ((size_t)n * p.Cin + c0 + e) * p.KHW + tap;
        if (p.w_raw) { const float w = __ldg(p.w_raw + o); if (w > p.hi || w < p.lo) t = 0.f; }
        p.gw[o] = t;
    }
}

// ------------------------------------------------------------------ host-side planning
struct Plan {
    int Cp, K_total, num_kb, n_tiles, n_t, n_mma, acc_cols, stages, main_col, sig_col, wsum_col, ring_bytes;
    size_t xp_bytes, wp_bytes, smem_bytes;
};

static inline int pad_to(int v, int a) { return (v + a - 1) / a * a; }

static Plan make_plan(int Cin_k, int KHW, int n_out, bool has_main, bool has_sigma, bool has_wsum, int64_t pixels_in,
                      int m_tiles_hint = 0) {
    Plan pl;
    pl.Cp = pad_to(Cin_k, 8);
    pl.K_total = KHW * pl.Cp;
    pl.num_kb = (pl.K_total + UM_BLOCK_K - 1) / UM_BLOCK_K;
    const int env_max_nt = UM_MAX_NT;
    const int max_nt = has_sigma ? (has_main ? env_max_nt : 248) : 256;
    pl.n_tiles = (n_out + max_nt - 1) / max_nt;
    // skinny problems (few 128-row m-tiles, e.g. the fully connected layers at batch 512) are latency-bound:
    // trade operand re-reads for more CTAs by narrowing the n-tile until ~100 CTAs exist
    if (m_tiles_hint > 0) {
        while (m_tiles_hint * pl.n_tiles < 96 && (n_out + pl.n_tiles - 1) / pl.n_tiles > 48) pl.n_tiles *= 2;
    }
    pl.n_t = pad_to((n_out + pl.n_tiles - 1) / pl.n_tiles, 8);
    pl.n_tiles = (n_out + pl.n_t - 1) / pl.n_t;
    int col = 0;
    pl.main_col = pl.sig_col = pl.wsum_col = -1;
    if (has_main) { pl.main_col = col; col += pl.n_t; }
    if (has_sigma) { pl.sig_col = col; col += pl.n_t; }
    if (has_wsum) { pl.wsum_col = col; col += 1; }
    pl.n_mma = pad_to(col, 16);
    if (pl.n_mma < 16) pl.n_mma = 16;
    // the epilogue reads 16-column groups: keep every read inside the allocation
    int need = pl.n_mma;
    if (has_main) need = max(need, pl.main_col + pad_to(pl.n_t, 16));
    if (has_sigma) need = max(need, pl.sig_col + pad_to(pl.n_t, 16));
    if (has_wsum) need = max(need, pl.wsum_col + 16);
    pl.acc_cols = need;
    const int stage_bytes = UM_A_STAGE + pl.n_mma * 128;
    const int max_stages = 4;                           // one CTA per SM (registers of the two MMA warpgroups)
    pl.stages = (192 * 1024) / stage_bytes;
    if (pl.stages > max_stages) pl.stages = max_stages;
    if (pl.stages < 2) pl.stages = 2;
    if (pl.stages > pl.num_kb) pl.stages = pl.num_kb < 1 ? 1 : pl.num_kb;
    // the fp32 accumulator tile (128 rows, acc_cols + 4 floats apart) reuses the operand ring after the main loop
    const int acc_bytes = UM_BLOCK_M * (pl.acc_cols + 4) * 4;
    pl.ring_bytes = pad_to(max(pl.stages * stage_bytes, acc_bytes), 1024);
    pl.smem_bytes = 1024 + (size_t)pl.ring_bytes + 16 * pl.stages + 64;
    pl.xp_bytes = (size_t)pixels_in * pl.Cp * 2;
    pl.wp_bytes = (size_t)pl.n_tiles * pl.num_kb * pl.n_mma * 64 * 2;
    return pl;
}

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---- shift-GEMM forward (k_conv_shift): eligibility and sizes
struct ShiftPlan {
    int n_t, n_mma, main_col, sig_col, n_planes, n_chunks, n_steps, a_pixels, a_plane, a_stage, b_bytes, n_tiles, acc_bufs;
    size_t smem_bytes, wp_bytes;
};
int g_shift_enable = 1;        // test hook: nn_debug_shift_enable

// planes of the row-plane image: K = KW * Cin of a kernel row in whole K = 16 steps of two 8-element planes
static inline int shift_planes(int Cin, int KW) { return 2 * ((KW * Cin + 15) / 16); }

// the weight image [kh][plane][row][8] (nn_prepare_weights sizes it from the same fields)
static void shift_weight_plan(int Cin, int KH, int KW, int Cout, bool noisy, ShiftPlan* sp) {
    sp->n_t = pad_to(Cout, 8);
    sp->main_col = 0;
    sp->sig_col = noisy ? sp->n_t : -1;
    sp->n_mma = pad_to(noisy ? 2 * sp->n_t : sp->n_t, 16);
    sp->n_planes = shift_planes(Cin, KW);
    sp->n_chunks = KH * sp->n_planes;
    sp->n_steps = sp->n_chunks / 2;
    sp->b_bytes = sp->n_chunks * sp->n_mma * 16;
    sp->wp_bytes = (size_t)sp->b_bytes;
}

static bool make_shift_plan(const nn_conv_geom& g, bool noisy, ShiftPlan* out) {
    if (!g_shift_enable) return false;
    if (g.Cin > 8 || g.stride != 1 || g.pad != 0 || g.KH > g.H || g.KW > g.W || g.W >= 4096) return false;
    if ((int64_t)g.B * g.H * g.W >= (int64_t)1 << 31) return false;
    ShiftPlan sp;
    shift_weight_plan(g.Cin, g.KH, g.KW, g.Cout, noisy, &sp);
    if (sp.n_mma > SH_MAX_N || sp.n_steps > SH_MAX_STEPS) return false;
    // pixels per plane of an A stage: 128 positions and KH - 1 rows below them (the horizontal halo is inside K); the
    // block tiles of the pooled launches need 16 + KH - 1 image rows from the tile's column on -- the ring is sized for both
    sp.a_pixels = UM_BLOCK_M + (g.KH - 1) * g.W;
    const int a_pixels_blk = (15 + g.KH - 1) * g.W + 8;
    sp.a_plane = pad_to((a_pixels_blk > sp.a_pixels ? a_pixels_blk : sp.a_pixels) * 16, 128);
    sp.a_stage = sp.n_planes * sp.a_plane;
    sp.n_tiles = (int)(((int64_t)g.B * g.H * g.W + UM_BLOCK_M - 1) / UM_BLOCK_M);
    const size_t acc_tile = (size_t)UM_BLOCK_M * (sp.n_mma + 4) * 4;
    sp.smem_bytes = 128 + (size_t)sp.b_bytes + (size_t)SH_STAGES * sp.a_stage + 16 * SH_STAGES + 96 + 4 * SH_MAX_STEPS + 16 + 12 * 1024 + acc_tile;
    if (sp.smem_bytes > 227 * 1024) return false;
    // a second accumulator tile where it fits (conv1: 222 KB): the MMA warpgroups then store a tile while the epilogue
    // still reads the one before
    sp.acc_bufs = sp.smem_bytes + acc_tile <= 227 * 1024 ? 2 : 1;
    sp.smem_bytes += (sp.acc_bufs - 1) * acc_tile;
    if (out) *out = sp;
    return true;
}

// the row-plane input image of a shift launch: n_planes planes of B*H*W 16-byte pixel records
static size_t shift_planes_bytes(const nn_conv_geom& g) {
    return (size_t)shift_planes(g.Cin, g.KW) * g.B * g.H * g.W * 16;
}

// debug hook: per-CTA phase timestamps of the next forward launches (NN_UMMA_DEBUG=1)
long long* g_dbg_buf = nullptr;
size_t g_dbg_ctas = 0, g_dbg_last = 0;

// measurement hook: CUDA events around the main tensor-core kernel only (excludes the operand packs)
int g_time_main = 0;
cudaEvent_t g_ev0 = nullptr, g_ev1 = nullptr;

static int nn_num_sms_cached() {
    int dev = 0;
    cudaGetDevice(&dev);
    return nn_num_sms(dev);
}

// per-CTA phase stamps of the forward launches (tools/cta_timeline.py): debug builds with NN_UMMA_DEBUG set
static bool umma_cta_dbg() {
#ifdef NN_KDEBUG
    static const bool on = getenv("NN_UMMA_DEBUG") != nullptr;
    return on;
#else
    return false;
#endif
}

// the epilogue k_conv_umma is instantiated with (see k_conv_umma)
static int umma_epi(const UmmaP& p) {
    const bool extras = p.bias || p.mask_x || p.z_inject || p.z_export || p.sigma_export || p.stats;
    if (!extras && p.main_col >= 0 && p.noise_mode != NN_NOISE_NONE && p.y_noisy) return 1;
    if (!extras && p.main_col >= 0 && p.noise_mode == NN_NOISE_NONE && p.y) return 2;
    return 0;
}

// split-K for skinny linear layers (few m-tiles x n-tiles, long K: fc1 forward at batch 512 is 52 CTAs walking 47
// k-blocks each -- a latency chain on a third of the SMs): the k-blocks are dealt to this many CTAs per tile, which dump
// raw accumulators, and k_splitk_epilogue sums them and applies the noise epilogue.  1 = not split (also when the
// split-K workspace, ws_bytes, cannot hold the partial sums)
static int umma_splits(const UmmaP& p, const Plan& pl, size_t ws_bytes) {
    const int epi = umma_epi(p);
    const int m_tiles = (p.M + UM_BLOCK_M - 1) / UM_BLOCK_M;
    if ((epi != 1 && epi != 2) || p.OH * p.OW != 1 || umma_cta_dbg() || m_tiles * pl.n_tiles * 2 > nn_num_sms_cached() ||
        pl.num_kb < 8 || ws_bytes == 0)
        return 1;
    int splits = 4;
    while (splits > 1 && pl.num_kb / splits < 4) --splits;
    const size_t need = (size_t)splits * pl.n_tiles * pl.n_mma * m_tiles * UM_BLOCK_M * sizeof(float);
    return need > ws_bytes ? 1 : splits;
}

static int launch_umma(const UmmaP& p, const Plan& pl, cudaStream_t st, void* splitk_ws = nullptr, size_t splitk_ws_bytes = 0) {
    NN_ONCE_PER_DEVICE({
        NN_CUDA_OK(cudaFuncSetAttribute(k_conv_umma<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        NN_CUDA_OK(cudaFuncSetAttribute(k_conv_umma<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        NN_CUDA_OK(cudaFuncSetAttribute(k_conv_umma<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    });
    const int epi = umma_epi(p);
    UmmaP pd = p;
    // incremental tap tracking saves the producers' divisions on the plain (dgrad) variant; the noisy forward keeps the
    // direct computation
    pd.inc_taps = epi == 2 ? 1 : 0;
    pd.rows_tile = UM_BLOCK_M;
    dim3 grid((p.M + pd.rows_tile - 1) / pd.rows_tile, pl.n_tiles);
#ifdef NN_KDEBUG
    const bool want_dbg = umma_cta_dbg();
    if (want_dbg) {
        const size_t ctas = (size_t)grid.x * grid.y;
        if (ctas > g_dbg_ctas) {
            if (g_dbg_buf) cudaFree(g_dbg_buf);
            cudaMalloc(&g_dbg_buf, ctas * 8 * sizeof(long long));
            g_dbg_ctas = ctas;
        }
        cudaMemsetAsync(g_dbg_buf, 0, ctas * 8 * sizeof(long long), st);
        pd.dbg = g_dbg_buf;
        g_dbg_last = ctas;
    }
#endif
    const int splits = umma_splits(p, pl, splitk_ws ? splitk_ws_bytes : 0);
    if (splits > 1) {
        grid.z = splits;
        pd.partial = (float*)splitk_ws;
        pd.m_pad = (int)grid.x * UM_BLOCK_M;
    }
#ifdef NN_KDEBUG
    static const bool want_kdbg = getenv("NN_UMMA_KDEBUG") != nullptr;
    if (want_kdbg) {
        const size_t rows = ((size_t)grid.x * grid.y * pl.num_kb * 4 + 7) / 8;      // rows of 8 longs, as nn_debug_cta_timeline copies
        if (rows > g_dbg_ctas) {
            if (g_dbg_buf) cudaFree(g_dbg_buf);
            cudaMalloc(&g_dbg_buf, rows * 8 * sizeof(long long));
            g_dbg_ctas = rows;
        }
        cudaMemsetAsync(g_dbg_buf, 0, rows * 8 * sizeof(long long), st);
        pd.kdbg = g_dbg_buf;
        g_dbg_last = rows;
    }
#endif
    if (g_time_main) {
        if (!g_ev0) { cudaEventCreate(&g_ev0); cudaEventCreate(&g_ev1); }
        cudaEventRecord(g_ev0, st);
    }
    UmmaAMap amap;
    memset(&amap, 0, sizeof(amap));
    // linear layers: one output position per sample and the kernel covers the whole (unpadded) input map, so the im2col row of
    // sample m is the sample's packed activation itself = row m of a row-major [B][KH * KW * Cp] matrix
    if (nn_debug_tma_enable(-1) && p.OH * p.OW == 1 && p.pad == 0 && p.KH == p.H && p.KW == p.W && pd.rows_tile == UM_BLOCK_M &&
        (((size_t)p.KH * p.KW * p.Cp * 2) % 16) == 0 && ((uintptr_t)p.xp % 16) == 0) {
        const uint64_t k_total = (uint64_t)p.KH * p.KW * p.Cp;
        if (nn_tma_encode_rows(&amap, p.xp, (uint64_t)p.M, k_total, k_total * 2)) return 1;
        pd.a_tma = 1;
    }
    if (epi == 1) k_conv_umma<1><<<grid, UM_THREADS, pl.smem_bytes, st>>>(pd, amap);
    else if (epi == 2) k_conv_umma<2><<<grid, UM_THREADS, pl.smem_bytes, st>>>(pd, amap);
    else k_conv_umma<0><<<grid, UM_THREADS, pl.smem_bytes, st>>>(pd, amap);
    if (g_time_main) cudaEventRecord(g_ev1, st);
    NN_LAUNCH_OK();
    if (splits > 1) {
        SplitEpiP e;
        memset(&e, 0, sizeof(e));
        e.partial = pd.partial; e.splits = splits; e.n_tiles = pl.n_tiles; e.n_mma = pl.n_mma; e.n_t = pl.n_t;
        e.main_col = pl.main_col; e.sig_col = pl.sig_col; e.m_pad = pd.m_pad; e.M = p.M; e.Cout = p.Cout;
        e.y_scale = p.y_scale; e.s_scale = p.s_scale; e.current = p.current; e.scale_dev = p.scale_dev; e.rng = p.rng;
        e.y = p.y; e.y_noisy = p.y_noisy; e.noisy = epi == 1;
        if (p.bn_fin.mean) {        // (nn_umma_conv_fwd checked M % 256 == 0)
            e.stat_partial = (double*)p.bn_scratch;
            e.stat_counters = (unsigned*)(e.stat_partial + (size_t)p.Cout * 16 * 2);
            e.fin = p.bn_fin; e.fin.count = (double)p.M; e.zero_out = p.zero_out;
        }
        const int total = p.M * ((p.Cout + 3) / 4);
        k_splitk_epilogue<<<(total + 255) / 256, 256, 0, st>>>(e);
        NN_LAUNCH_OK();
    }
    return 0;
}

}  // namespace

// which: 0 forward, 1 dgrad, 2 wgrad
bool nn_umma_supports(const nn_conv_geom* g, int which) {
    if (which == 0) return true;
    if (which == 1) return g->stride == 1 && g->pad <= g->KH - 1 && g->pad <= g->KW - 1;
    return true;
}

int64_t nn_umma_fwd_workspace(const nn_conv_geom* g, int precision) {
    // sized for the larger of forward (input packed) and dgrad (grad_output packed)
    int OH, OW;
    nn_out_hw(*g, OH, OW);
    Plan f = make_plan(g->Cin, g->KH * g->KW, g->Cout, true, true, true, (int64_t)g->B * g->H * g->W,
                       (g->B * OH * OW + 127) / 128);
    Plan d = make_plan(g->Cout, g->KH * g->KW, g->Cin, true, false, false, (int64_t)g->B * OH * OW,
                       (g->B * g->H * g->W + 127) / 128);
    size_t a = align_up(f.xp_bytes, 1024) + align_up(f.wp_bytes, 1024);
    size_t b = align_up(d.xp_bytes, 1024) + align_up(d.wp_bytes, 1024);
    {   // the TMA-im2col path pads every tap to whole channel chunks: its weight image can be the larger one
        TmaPlan tp;
        if (nn_tma_make_plan(g->Cin, g->KH, g->KW, g->stride, g->pad, g->Cout, true, OH, OW, &tp)) {
            const size_t t = align_up((size_t)g->B * g->H * g->W * tp.Cp * 2, 1024) + align_up(tp.wp_bytes, 1024);
            if (t > a) a = t;
        }
        if (g->stride == 1 && nn_tma_make_plan(g->Cout, g->KH, g->KW, 1, g->KH - 1 - g->pad, g->Cin, false, g->H, g->W, &tp)) {
            const size_t t = align_up((size_t)g->B * OH * OW * tp.Cp * 2, 1024) + align_up(tp.wp_bytes, 1024);
            if (t > b) b = t;
        }
    }
    {   // the shift kernel's row-plane image holds P >= 2 planes of the input
        ShiftPlan sp;
        if (make_shift_plan(*g, true, &sp) || make_shift_plan(*g, false, &sp)) {
            const size_t t = align_up(shift_planes_bytes(*g), 1024) + align_up(sp.wp_bytes, 1024);
            if (t > a) a = t;
        }
    }
    if (OH * OW == 1)          // split-K partial sums of a skinny linear forward (up to 4 shares)
        a += (size_t)4 * f.n_tiles * f.n_mma * ((g->B + UM_BLOCK_M - 1) / UM_BLOCK_M * UM_BLOCK_M) * sizeof(float) + 1024;
    return (int64_t)((a > b ? a : b) + 2048);
}


int* nn_umma_err_flag(int device) {
    static int* flags[64] = {nullptr};
    if (device < 0 || device >= 64) return nullptr;
    if (!flags[device]) {
        if (cudaMalloc(&flags[device], sizeof(int)) != cudaSuccess) return nullptr;
        cudaMemset(flags[device], 0, sizeof(int));
    }
    return flags[device];
}

extern "C" int nn_debug_cta_timeline(long long* host_out, int max_ctas) {
    // copies [cta][8] clock64 stamps of the last forward launch (NN_UMMA_DEBUG=1): 0 start, 1 setup done,
    // 2 last MMA issued, 3 accumulators ready, 4 epilogue done, 5 teardown, 6 producers done, 7 smid
    if (!g_dbg_buf) return 0;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    const size_t n = g_dbg_last < (size_t)max_ctas ? g_dbg_last : (size_t)max_ctas;
    if (cudaMemcpy(host_out, g_dbg_buf, n * 8 * sizeof(long long), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return (int)n;
}

extern "C" float nn_debug_main_kernel_ms(int enable) {
    // enable = 1/0: switch the event pair around k_conv_umma on/off; enable < 0: synchronise and return the
    // elapsed milliseconds of the last timed main-kernel launch (-1 if none)
    if (enable >= 0) { g_time_main = enable; return 0.f; }
    if (!g_ev0 || !g_ev1) return -1.f;
    if (cudaEventSynchronize(g_ev1) != cudaSuccess) return -1.f;
    float ms = -1.f;
    if (cudaEventElapsedTime(&ms, g_ev0, g_ev1) != cudaSuccess) return -1.f;
    return ms;
}

extern "C" int nn_debug_error_flag(int device, int reset) {
    int* f = nn_umma_err_flag(device);
    if (!f) return -1;
    int v = 0;
    if (cudaSetDevice(device) != cudaSuccess) return -1;
    if (cudaDeviceSynchronize() != cudaSuccess) return -2;
    if (cudaMemcpy(&v, f, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -3;
    if (reset) cudaMemset(f, 0, sizeof(int));
    return v;
}

extern "C" int nn_conv_pool_fusable(const nn_conv_geom* g, int32_t noise_mode, int32_t precision);

static int shift_conv_fwd(const nn_conv_fwd_args* a, const ShiftPlan& sp, int device, cudaStream_t st) {
    const nn_conv_geom& g = a->g;
    int OH, OW;
    nn_out_hw(g, OH, OW);
    const bool noise = a->noise_mode != NN_NOISE_NONE;
    const size_t xp_bytes = shift_planes_bytes(g);
    uint8_t* ws = (uint8_t*)align_up((size_t)a->workspace, 1024);
    const size_t need = (a->x_packed ? 0 : align_up(xp_bytes, 1024)) + (a->w_packed ? 0 : align_up(sp.wp_bytes, 1024)) + 1024;
    if ((!a->x_packed || !a->w_packed) && (!a->workspace || (size_t)a->workspace_bytes < need))
        return nn_fail("nn_noisy_conv_fwd: workspace too small%s (need %lld bytes)", "", (long long)need);
    const __nv_bfloat16* xp = (const __nv_bfloat16*)a->x_packed;
    const __nv_bfloat16* wp = (const __nv_bfloat16*)a->w_packed;
    if (!xp) {
        const int64_t total = (int64_t)sp.n_planes * g.B * g.H * g.W;
        int grid = (int)((total + 255) / 256);
        if (grid > 16 * nn_num_sms(device)) grid = 16 * nn_num_sms(device);
        k_pack_act_rows<<<grid, 256, 0, st>>>(a->x, (__nv_bfloat16*)ws, g.B, g.Cin, g.H, g.W, g.KW, sp.n_planes, a->a_code_scale);
        NN_LAUNCH_OK();
        xp = (const __nv_bfloat16*)ws;
        ws += align_up(xp_bytes, 1024);
    }
    if (!wp) {
        PackWP pw;
        memset(&pw, 0, sizeof(pw));
        pw.w_eff = a->w_eff; pw.w_raw = a->w_raw; pw.wp = (__nv_bfloat16*)ws;
        pw.Cout = g.Cout; pw.Cin = g.Cin; pw.KHW = g.KH * g.KW; pw.Cp = 8; pw.n_t = sp.n_t; pw.n_mma = sp.n_mma;
        pw.num_kb = sp.n_chunks; pw.n_tiles = 1; pw.main_col = sp.main_col; pw.sig_col = sp.sig_col; pw.wsum_col = -1;
        pw.sh_kw = g.KW; pw.sh_planes = sp.n_planes;
        pw.noise_mode = a->noise_mode; pw.mode = 0; pw.layout = NN_PACK_SHIFT; pw.w_code_scale = a->w_code_scale;
        const int64_t total = (int64_t)sp.n_chunks * sp.n_mma;
        k_pack_w<<<(int)((total + 255) / 256), 256, 0, st>>>(pw);
        NN_LAUNCH_OK();
        wp = (const __nv_bfloat16*)ws;
    }
    ShiftP p;
    memset(&p, 0, sizeof(p));
    p.H = g.H; p.W = g.W; p.OH = OH; p.OW = OW; p.KH = g.KH; p.KW = g.KW; p.Cout = g.Cout;
    p.n_mma = sp.n_mma; p.main_col = sp.main_col; p.sig_col = sp.sig_col; p.n_steps = sp.n_steps; p.n_planes = sp.n_planes;
    p.a_pixels = sp.a_pixels; p.a_plane = sp.a_plane; p.a_stage = sp.a_stage; p.b_bytes = sp.b_bytes; p.n_tiles = sp.n_tiles;
    p.acc_bufs = sp.acc_bufs;
    p.total_pixels = (long long)g.B * g.H * g.W;
    p.xp = xp; p.wp = wp;
    const float as = a->a_code_scale > 0.f ? a->a_code_scale : 1.f;
    const float wsc = a->w_code_scale > 0.f ? a->w_code_scale : 1.f;
    p.y_scale = as * wsc; p.s_scale = as;
    p.y = a->y; p.y_noisy = a->y_noisy; p.z_inject = a->z_inject;
    p.pooled = a->pooled_out; p.pool_arg = a->argmax_out;
    p.current = a->current; p.scale_dev = a->scale_dev; p.rng = a->rng;
    p.err_flag = nn_umma_err_flag(device);
    p.sbo_units = 8; p.zero_out = a->zero_out;
    if (p.pooled) {
        // block tiles (16 rows x 8 columns of the input grid): one stage plane = the rows r0 .. r0 + 15 + KH - 1 from column c0 on
        p.blk = 1; p.tiles_x = g.W / 8; p.tiles_per_img = (g.H / 16) * p.tiles_x; p.sbo_units = g.W;
        p.n_tiles = g.B * p.tiles_per_img;
        p.a_pixels = (15 + g.KH - 1) * g.W + 8;
        if (a->bn_mean) {
            if (!a->bn_invstd || !a->bn_scratch) return nn_fail("nn_noisy_conv_fwd: bn_mean needs bn_invstd and bn_scratch%s", "");
            if (a->bn_eval_mode && (!a->bn_running_mean || !a->bn_running_var))
                return nn_fail("nn_noisy_conv_fwd: bn_eval_mode needs the running statistics%s", "");
            p.stat_ticket = (unsigned*)a->bn_scratch;
            p.stat_partial = (double*)((uint8_t*)a->bn_scratch + 16);
            p.fin.count = (double)g.B * (OH / 2) * (OW / 2);
            p.fin.eps = a->bn_eps; p.fin.momentum = a->bn_momentum; p.fin.mean = a->bn_mean; p.fin.invstd = a->bn_invstd;
            p.fin.running_mean = a->bn_running_mean; p.fin.running_var = a->bn_running_var; p.fin.xmax_out = nullptr;
            p.fin.eval_mode = a->bn_eval_mode;
        }
    } else if (a->bn_mean) {
        return nn_fail("nn_noisy_conv_fwd: bn_mean is served together with pooled_out only%s", "");
    }
    int grid = nn_num_sms(device);
    if (grid > p.n_tiles) grid = p.n_tiles;
    if (p.stat_partial && grid > 256) grid = 256;         // nn_conv_bn_scratch_bytes holds 256 per-CTA partials
#ifdef NN_KDEBUG
    static const bool want_dbg = getenv("NN_UMMA_DEBUG") != nullptr;
#else
    const bool want_dbg = false;
#endif
    if (want_dbg) {
        const size_t rows = (size_t)grid * 32 * SH_DBG / 8;      // 32 tiles x SH_DBG stamps, in rows of 8
        if (rows > g_dbg_ctas) {
            if (g_dbg_buf) cudaFree(g_dbg_buf);
            cudaMalloc(&g_dbg_buf, rows * 8 * sizeof(long long));
            g_dbg_ctas = rows;
        }
        cudaMemsetAsync(g_dbg_buf, 0, rows * 8 * sizeof(long long), st);
        p.dbg = g_dbg_buf;
        g_dbg_last = rows;
    }
    if (g_time_main) {
        if (!g_ev0) { cudaEventCreate(&g_ev0); cudaEventCreate(&g_ev1); }
        cudaEventRecord(g_ev0, st);
    }
    const int mode = !noise ? 0 : (a->z_inject ? 2 : 1);      // 16 epilogue warps
#define NN_SHIFT_LAUNCH(MODE, EW, POOL)                                                                                \
    do {                                                                                                               \
        NN_ONCE_PER_DEVICE({ \
            NN_CUDA_OK(cudaFuncSetAttribute(k_conv_shift<MODE, EW, POOL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); \
        });                                                                                                              \
        k_conv_shift<MODE, EW, POOL><<<grid, (EW + 8) * 32, sp.smem_bytes, st>>>(p);                                    \
    } while (0)
    if (p.pooled) {
        if (mode == 0) NN_SHIFT_LAUNCH(0, 16, true); else if (mode == 1) NN_SHIFT_LAUNCH(1, 16, true); else NN_SHIFT_LAUNCH(2, 16, true);
    } else {
        if (mode == 0) NN_SHIFT_LAUNCH(0, 16, false); else if (mode == 1) NN_SHIFT_LAUNCH(1, 16, false); else NN_SHIFT_LAUNCH(2, 16, false);
    }
#undef NN_SHIFT_LAUNCH
    if (g_time_main) cudaEventRecord(g_ev1, st);
    NN_LAUNCH_OK();
    return 0;
}

extern "C" int nn_conv_pack_layout(const nn_conv_geom* g, int32_t noise_mode, int32_t precision) {
    if (!g || precision != NN_PREC_BF16) return NN_PACK_TILED;
    if (make_shift_plan(*g, noise_mode != NN_NOISE_NONE, nullptr)) return NN_PACK_SHIFT;
    int OH, OW;
    nn_out_hw(*g, OH, OW);
    return nn_tma_make_plan(g->Cin, g->KH, g->KW, g->stride, g->pad, g->Cout, noise_mode != NN_NOISE_NONE, OH, OW, nullptr) ? NN_PACK_TMA
                                                                                                                          : NN_PACK_TILED;
}
extern "C" int nn_conv_dgrad_pack_layout(const nn_conv_geom* g, int32_t precision) {
    if (!g || precision != NN_PREC_BF16 || g->stride != 1) return NN_PACK_TILED;
    return nn_tma_make_plan(g->Cout, g->KH, g->KW, 1, g->KH - 1 - g->pad, g->Cin, false, g->H, g->W, nullptr) ? NN_PACK_TMA : NN_PACK_TILED;
}
extern "C" int nn_conv_pool_fusable(const nn_conv_geom* g, int32_t noise_mode, int32_t precision) {
    if (!g || precision != NN_PREC_BF16) return 0;
    if (!make_shift_plan(*g, noise_mode != NN_NOISE_NONE, nullptr)) return 0;
    int OH, OW;
    nn_out_hw(*g, OH, OW);
    // block tiles of 16 rows x 8 columns; the epilogue keeps SH_POOL_IT 4-channel groups per warp (16 warps)
    const int ngrp = (g->Cout + 3) / 4;      // 16 epilogue warps: 4 per lane quarter; fixed groups + at most one rotating group
    return g->W % 8 == 0 && g->H % 16 == 0 && OH % 2 == 0 && OW % 2 == 0 && ngrp / 4 <= SH_POOL_IT - 1 && ngrp % 4 <= 1;
}
// 1 if nn_noisy_conv_fwd serves bn_mean for this LINEAR layer (its split-K epilogue adds the per-channel sums): the launch must be
// split (few CTAs, >= 8 k-blocks) and the batch a multiple of 256 (<= 4096)
extern "C" int nn_conv_linear_bn_fusable(const nn_conv_geom* g, int32_t noise_mode, int32_t precision, int device) {
    if (!g || precision != NN_PREC_BF16) return 0;
    int OH, OW;
    nn_out_hw(*g, OH, OW);
    const int M = g->B * OH * OW;
    if (OH * OW != 1 || M % 256 || M > 4096) return 0;
    const Plan pl = make_plan(g->Cin, g->KH * g->KW, g->Cout, true, noise_mode != NN_NOISE_NONE, false, (int64_t)g->B * g->H * g->W, (M + 127) / 128);
    const int ctas = ((M + UM_BLOCK_M - 1) / UM_BLOCK_M) * pl.n_tiles;
    return ctas * 2 <= nn_num_sms(device) && pl.num_kb >= 8 && pl.num_kb / 2 >= 4;
}
// [ticket | per-CTA partial sums of the pooled values]: 16 + SMs x Cout x 2 doubles (sized for 256 CTAs)
extern "C" int64_t nn_conv_bn_scratch_bytes(int Cout) { return 16 + (int64_t)256 * Cout * 2 * sizeof(double); }
extern "C" int64_t nn_conv_shift_planes_bytes(const nn_conv_geom* g) {
    if (!g || g->Cin < 1 || g->Cin > 8 || g->KW < 1) return 0;
    return (int64_t)shift_planes_bytes(*g);
}
extern "C" int nn_debug_shift_enable(int enable) {
    const int prev = g_shift_enable;
    if (enable >= 0) g_shift_enable = enable;
    return prev;
}

// ---- TMA-im2col pair kernel (nn_conv_tma.cu): packer parameters of the NN_PACK_TMA weight image
static void fill_pack_tma(PackWP& pw, const TmaPlan& tp) {
    pw.Cp = tp.Cp; pw.n_t = tp.n_t; pw.n_mma = tp.n_mma; pw.num_kb = 0; pw.n_tiles = tp.n_tiles;
    pw.main_col = tp.main_col; pw.sig_col = tp.sig_col; pw.wsum_col = -1; pw.layout = NN_PACK_TMA;
    pw.t_nc64 = tp.n_c64; pw.t_tail = tp.tail_w; pw.t_nc = tp.nc; pw.t_wt = tp.wt; pw.t_nhalf = tp.n_half; pw.t_tapbytes = tp.tap_bytes;
}
static int64_t pack_tma_chunks(const TmaPlan& tp) { return (int64_t)tp.n_tiles * tp.n_mma * tp.taps * (tp.wt >> 3); }

// lean calls only (what the training step issues): no bias / statistics / exports / clean-output copy
static bool tma_fwd_plan(const nn_conv_fwd_args* a, TmaPlan* tp) {
    const nn_conv_geom& g = a->g;
    int OH, OW;
    nn_out_hw(g, OH, OW);
    const bool noise = a->noise_mode != NN_NOISE_NONE;
    const bool has_main = a->w_eff != nullptr || a->w_packed != nullptr;
    const bool lean = has_main && !a->bias && !a->z_export && !a->sigma_export && !a->stats && !a->pooled_out && !a->bn_mean && !(noise && a->y);
    return lean && nn_tma_make_plan(g.Cin, g.KH, g.KW, g.stride, g.pad, g.Cout, noise, OH, OW, tp);
}

static int tma_conv_fwd(const nn_conv_fwd_args* a, const TmaPlan& tp, int device, cudaStream_t st) {
    const nn_conv_geom& g = a->g;
    int OH, OW;
    nn_out_hw(g, OH, OW);
    const size_t xp_bytes = (size_t)g.B * g.H * g.W * tp.Cp * 2;
    const size_t need = (a->x_packed ? 0 : align_up(xp_bytes, 1024)) + (a->w_packed ? 0 : align_up(tp.wp_bytes, 1024)) + 1024;
    if ((!a->x_packed || !a->w_packed) && (!a->workspace || (size_t)a->workspace_bytes < need))
        return nn_fail("nn_noisy_conv_fwd: workspace too small%s (need %lld bytes)", "", (long long)need);
    uint8_t* ws = (uint8_t*)align_up((size_t)a->workspace, 1024);
    const void* xp = a->x_packed;
    const void* wp = a->w_packed;
    if (!xp) {
        const int64_t total = (int64_t)g.B * g.H * g.W * (tp.Cp / 8);
        int grid = (int)((total + 255) / 256);
        if (grid > 16 * nn_num_sms(device)) grid = 16 * nn_num_sms(device);
        k_pack_act<<<grid, 256, 0, st>>>(a->x, (__nv_bfloat16*)ws, g.B, g.Cin, g.H * g.W, tp.Cp, a->a_code_scale);
        NN_LAUNCH_OK();
        xp = ws;
        ws += align_up(xp_bytes, 1024);
    }
    if (!wp) {
        PackWP pw;
        memset(&pw, 0, sizeof(pw));
        pw.w_eff = a->w_eff; pw.w_raw = a->w_raw; pw.wp = (__nv_bfloat16*)ws;
        pw.Cout = g.Cout; pw.Cin = g.Cin; pw.KHW = g.KH * g.KW; pw.noise_mode = a->noise_mode; pw.mode = 0;
        pw.w_code_scale = a->w_code_scale;
        fill_pack_tma(pw, tp);
        const int64_t total = pack_tma_chunks(tp);
        int grid = (int)((total + 255) / 256);
        if (grid > 8 * nn_num_sms(device)) grid = 8 * nn_num_sms(device);
        k_pack_w<<<grid, 256, 0, st>>>(pw);
        NN_LAUNCH_OK();
        wp = ws;
    }
    TmaConvCall c;
    memset(&c, 0, sizeof(c));
    c.pl = tp;
    c.B = g.B; c.H = g.H; c.W = g.W; c.OH = OH; c.OW = OW; c.KH = g.KH; c.KW = g.KW; c.stride = g.stride; c.pad = g.pad; c.Cout = g.Cout;
    c.xp = xp; c.wp = wp;
    const float as = a->a_code_scale > 0.f ? a->a_code_scale : 1.f;
    const float wsc = a->w_code_scale > 0.f ? a->w_code_scale : 1.f;
    c.y_scale = as * wsc; c.s_scale = as;
    c.y = a->y; c.y_noisy = a->y_noisy; c.noise_mode = a->noise_mode; c.current = a->current; c.scale_dev = a->scale_dev; c.rng = a->rng;
    c.z_inject = a->noise_mode != NN_NOISE_NONE ? a->z_inject : nullptr;
    c.err_flag = nn_umma_err_flag(device);
    if (g_time_main) {
        if (!g_ev0) { cudaEventCreate(&g_ev0); cudaEventCreate(&g_ev1); }
        c.ev0 = g_ev0; c.ev1 = g_ev1;
    }
    return nn_tma_conv_launch(c, device, st);
}

int nn_umma_conv_fwd(const nn_conv_fwd_args* a, int device, cudaStream_t st) {
    if (a->precision != NN_PREC_BF16)
        return nn_fail("nn_noisy_conv_fwd: tensor-core path implements NN_PREC_BF16 only%s", "");
    const nn_conv_geom& g = a->g;
    int OH, OW;
    nn_out_hw(g, OH, OW);
    const bool has_main = a->w_eff != nullptr || a->w_packed != nullptr;
    const bool noise = a->noise_mode != NN_NOISE_NONE;
    const bool has_wsum = noise && a->noise_mode == NN_NOISE_EXTERNAL && a->stats != nullptr;
    {   // narrow-input layers: persistent shift-GEMM kernel (weights resident, no im2col gather)
        const bool extras = a->bias || a->z_export || a->sigma_export || a->stats;
        ShiftPlan sp;
        const bool can = has_main && !extras && make_shift_plan(g, noise, &sp);
        if (a->pooled_out) {
            if (!can || !a->argmax_out || !nn_conv_pool_fusable(&g, a->noise_mode, a->precision))
                return nn_fail("nn_noisy_conv_fwd: pooled_out is not served for this call%s (see nn_conv_pool_fusable)", "");
            if (a->w_packed && a->w_packed_layout != NN_PACK_SHIFT)
                return nn_fail("nn_noisy_conv_fwd: pooled_out needs NN_PACK_SHIFT weights%s", "");
        }
        const int layout = a->w_packed ? a->w_packed_layout : (can ? NN_PACK_SHIFT : NN_PACK_TILED);
        if (layout == NN_PACK_SHIFT) {
            if (!can) return nn_fail("nn_noisy_conv_fwd: w_packed_layout = NN_PACK_SHIFT is not served for this call%s", "");
            return shift_conv_fwd(a, sp, device, st);
        }
    }
    {   // conv layers on the lean path: persistent CTA-pair kernel with TMA-im2col operands
        TmaPlan tp;
        const bool can = tma_fwd_plan(a, &tp);
        const int layout = a->w_packed ? a->w_packed_layout : (can ? NN_PACK_TMA : NN_PACK_TILED);
        if (layout == NN_PACK_TMA) {
            if (!can) return nn_fail("nn_noisy_conv_fwd: w_packed_layout = NN_PACK_TMA is not served for this call%s", "");
            return tma_conv_fwd(a, tp, device, st);
        }
    }
    Plan pl = make_plan(g.Cin, g.KH * g.KW, g.Cout, has_main, noise, has_wsum, (int64_t)g.B * g.H * g.W,
                        (g.B * OH * OW + 127) / 128);
    const size_t need = align_up(pl.xp_bytes, 1024) + align_up(pl.wp_bytes, 1024) + 1024;
    if (!a->workspace || (size_t)a->workspace_bytes < need)
        return nn_fail("nn_noisy_conv_fwd: workspace too small%s (need %lld bytes)", "", (long long)need);
    uint8_t* ws = (uint8_t*)align_up((size_t)a->workspace, 1024);
    __nv_bfloat16* xp = a->x_packed ? (__nv_bfloat16*)a->x_packed : (__nv_bfloat16*)ws;
    __nv_bfloat16* wp = a->w_packed ? (__nv_bfloat16*)a->w_packed : (__nv_bfloat16*)(ws + align_up(pl.xp_bytes, 1024));
    int* err = nn_umma_err_flag(device);
    UmmaP p;
    memset(&p, 0, sizeof(p));
    p.B = g.B; p.H = g.H; p.W = g.W; p.Cp = pl.Cp; p.KH = g.KH; p.KW = g.KW; p.stride = g.stride; p.pad = g.pad;
    p.OH = OH; p.OW = OW; p.M = g.B * OH * OW; p.Cout = g.Cout; p.n_t = pl.n_t; p.n_mma = pl.n_mma;
    p.num_kb = pl.num_kb; p.stages = pl.stages; p.acc_cols = pl.acc_cols; p.ring_bytes = pl.ring_bytes;
    p.main_col = pl.main_col; p.sig_col = pl.sig_col; p.wsum_col = pl.wsum_col;
    p.xp = xp; p.wp = wp;
    const float as = a->a_code_scale > 0.f ? a->a_code_scale : 1.f;
    const float wsc = a->w_code_scale > 0.f ? a->w_code_scale : 1.f;
    p.y_scale = as * wsc; p.s_scale = as;
    p.bias = a->bias; p.y = has_main ? a->y : nullptr; p.y_in = has_main ? nullptr : a->y; p.y_noisy = a->y_noisy;
    p.noise_mode = a->noise_mode; p.current = a->current; p.scale_dev = a->scale_dev; p.z_inject = a->z_inject;
    p.z_export = a->z_export; p.sigma_export = a->sigma_export; p.stats = a->stats; p.rng = a->rng;
    p.mask_x = nullptr; p.err_flag = err;
    // what is left of the workspace after the operand packs serves the split-K partial sums
    uint8_t* rest = ws + align_up(pl.xp_bytes, 1024) + align_up(pl.wp_bytes, 1024);
    uint8_t* ws_end = (uint8_t*)a->workspace + a->workspace_bytes;
    void* splitk_ws = rest < ws_end ? rest : nullptr;
    const size_t splitk_bytes = rest < ws_end ? (size_t)(ws_end - rest) : 0;
    if (a->bn_mean && !a->pooled_out) {       // BatchNorm1d statistics of a linear layer's output from the split-K epilogue
        // (every refusal comes before the first launch: a refused call writes nothing)
        if (!a->bn_invstd || !a->bn_scratch) return nn_fail("nn_noisy_conv_fwd: bn_mean needs bn_invstd and bn_scratch%s", "");
        if (a->bn_eval_mode && (!a->bn_running_mean || !a->bn_running_var))
            return nn_fail("nn_noisy_conv_fwd: bn_eval_mode needs the running statistics%s", "");
        if (g.Cout > 0 && ((g.B * OH * OW) >> 8) > 16) return nn_fail("nn_noisy_conv_fwd: bn_mean on a linear layer serves batches up to 4096%s", "");
        if (p.M % 256) return nn_fail("nn_noisy_conv_fwd: bn_mean on a linear layer needs a batch that is a multiple of 256%s", "");
        if (umma_splits(p, pl, splitk_bytes) == 1)
            return nn_fail("nn_noisy_conv_fwd: bn_mean on a linear layer is served by the split-K epilogue only%s (see nn_conv_linear_bn_fusable)", "");
        p.bn_fin.mean = a->bn_mean; p.bn_fin.invstd = a->bn_invstd; p.bn_fin.running_mean = a->bn_running_mean;
        p.bn_fin.running_var = a->bn_running_var; p.bn_fin.eps = a->bn_eps; p.bn_fin.momentum = a->bn_momentum;
        p.bn_fin.eval_mode = a->bn_eval_mode; p.bn_fin.xmax_out = nullptr;
        p.bn_scratch = a->bn_scratch; p.zero_out = a->zero_out;
    }

    if (!a->x_packed) {   // activations -> NHWC bf16 (integer codes when a_code_scale > 0)
        const int64_t total = (int64_t)g.B * g.H * g.W * (pl.Cp / 8);
        int grid = (int)((total + 255) / 256);
        if (grid > 16 * nn_num_sms(device)) grid = 16 * nn_num_sms(device);
        k_pack_act<<<grid, 256, 0, st>>>(a->x, xp, g.B, g.Cin, g.H * g.W, pl.Cp, a->a_code_scale);
        NN_LAUNCH_OK();
    }
    if (!a->w_packed) {
        PackWP pw;
        memset(&pw, 0, sizeof(pw));
        pw.w_eff = a->w_eff; pw.w_raw = a->w_raw; pw.wp = wp;
        pw.Cout = g.Cout; pw.Cin = g.Cin; pw.KHW = g.KH * g.KW; pw.Cp = pl.Cp; pw.n_t = pl.n_t; pw.n_mma = pl.n_mma;
        pw.num_kb = pl.num_kb; pw.n_tiles = pl.n_tiles; pw.main_col = pl.main_col; pw.sig_col = pl.sig_col;
        pw.wsum_col = pl.wsum_col; pw.noise_mode = a->noise_mode; pw.mode = 0; pw.w_code_scale = a->w_code_scale;
        const int64_t total = (int64_t)pl.n_tiles * pl.num_kb * pl.n_mma * 8;
        int grid = (int)((total + 255) / 256);
        if (grid > 8 * nn_num_sms(device)) grid = 8 * nn_num_sms(device);
        k_pack_w<<<grid, 256, 0, st>>>(pw);
        NN_LAUNCH_OK();
    }
    return launch_umma(p, pl, st, splitk_ws, splitk_bytes);
}

static Plan plan_for_job(const nn_wprep_job& jb) {
    if (jb.mode == 0)
        return make_plan(jb.Cin, jb.KHW, jb.Cout, true, jb.noise_mode != NN_NOISE_NONE,
                         jb.noise_mode == NN_NOISE_EXTERNAL && jb.want_wsum, 0, (jb.m_rows + 127) / 128);
    return make_plan(jb.Cout, jb.KHW, jb.Cin, true, false, false, 0, (jb.m_rows + 127) / 128);
}

// shift-layout jobs carry the kernel size as KHW: the kernel is square (KH = KW = sqrt(KHW)), Cin <= 8
static bool shift_plan_for_job(const nn_wprep_job& jb, ShiftPlan* sp, int* k_out) {
    int k = 1;
    while (k * k < jb.KHW) ++k;
    if (k * k != jb.KHW || jb.Cin < 1 || jb.Cin > 8) return false;
    shift_weight_plan(jb.Cin, k, k, jb.Cout, jb.noise_mode != NN_NOISE_NONE, sp);
    if (k_out) *k_out = k;
    return true;
}

// NN_PACK_TMA jobs: the plan depends on the channel counts, the tap count and the sigma rows only
static bool tma_plan_for_job(const nn_wprep_job& jb, TmaPlan* tp) {
    int k = 1;
    while (k * k < jb.KHW) ++k;
    if (k * k != jb.KHW) return false;
    if (jb.mode == 0) return nn_tma_make_plan(jb.Cin, k, k, 1, 0, jb.Cout, jb.noise_mode != NN_NOISE_NONE, 2, 2, tp);
    return nn_tma_make_plan(jb.Cout, k, k, 1, 0, jb.Cin, false, 2, 2, tp);
}

extern "C" int64_t nn_weight_pack_bytes(const nn_wprep_job* jb) {
    if (!jb) return 0;
    if (jb->layout == NN_PACK_TMA) { TmaPlan tp; return tma_plan_for_job(*jb, &tp) ? (int64_t)align_up(tp.wp_bytes, 1024) : 0; }
    if (jb->layout == NN_PACK_SHIFT) { ShiftPlan sp; return shift_plan_for_job(*jb, &sp, nullptr) ? (int64_t)align_up(sp.wp_bytes, 1024) : 0; }
    return (int64_t)align_up(plan_for_job(*jb).wp_bytes, 1024);
}

extern "C" int nn_prepare_weights(const nn_wprep_job* jobs, int count, int device, void* stream) {
    if (count <= 0) return 0;
    if (count > UM_MAX_PACK_JOBS) return nn_fail("nn_prepare_weights: too many jobs%s (%lld)", "", count);
    NN_SET_DEVICE(device);
    PackJobs pj;
    memset(&pj, 0, sizeof(pj));
    int64_t max_total = 0;
    for (int i = 0; i < count; ++i) {
        const nn_wprep_job& jb = jobs[i];
        if (!jb.w_raw || !jb.packed_out) return nn_fail("nn_prepare_weights: null pointer%s", "");
        if (jb.q_bits > 0 && !(jb.q_hi > 0)) return nn_fail("nn_prepare_weights: symmetric range needs q_hi > 0%s", "");
        Plan pl = plan_for_job(jb);
        TmaPlan tp;
        if (jb.layout == NN_PACK_TMA) {
            if (jb.want_wsum || !tma_plan_for_job(jb, &tp))
                return nn_fail("nn_prepare_weights: NN_PACK_TMA is not served for this job%s (see nn_conv_pack_layout)", "");
        }
        ShiftPlan sp;
        int sk = 0;
        if (jb.layout == NN_PACK_SHIFT) {
            if (jb.mode != 0 || jb.want_wsum || !shift_plan_for_job(jb, &sp, &sk))
                return nn_fail("nn_prepare_weights: NN_PACK_SHIFT needs a forward job with Cin <= 8, a square kernel and no colsum row%s", "");
            pl.Cp = 8; pl.n_t = sp.n_t; pl.n_mma = sp.n_mma; pl.num_kb = sp.n_chunks; pl.n_tiles = 1;
            pl.main_col = sp.main_col; pl.sig_col = sp.sig_col; pl.wsum_col = -1;
        }
        PackWP& pw = pj.j[i];
        pw.w_eff = jb.w_raw; pw.w_raw = jb.w_raw; pw.wp = (__nv_bfloat16*)jb.packed_out;
        pw.Cout = jb.Cout; pw.Cin = jb.Cin; pw.KHW = jb.KHW; pw.Cp = pl.Cp; pw.n_t = pl.n_t; pw.n_mma = pl.n_mma;
        pw.num_kb = pl.num_kb; pw.n_tiles = pl.n_tiles; pw.main_col = pl.main_col; pw.sig_col = pl.sig_col;
        pw.wsum_col = pl.wsum_col; pw.noise_mode = jb.noise_mode; pw.mode = jb.mode; pw.w_code_scale = 0.f;
        pw.layout = jb.layout;
        if (jb.layout == NN_PACK_SHIFT) { pw.sh_kw = sk; pw.sh_planes = sp.n_planes; }
        pw.q_bits = jb.q_bits;
        if (jb.q_bits > 0) {
            const double qmax = (double)((1u << jb.q_bits) - 1u);
            double sc = 2.0 * jb.q_hi / qmax;
            if (sc < 1e-6) sc = 1e-6;
            pw.q_hi = (float)jb.q_hi; pw.q_scale = (float)sc; pw.q_max = (float)qmax; pw.q_stoch = jb.stochastic;
            pw.u_inject = jb.u_inject; pw.rng = jb.rng;
        }
        int64_t total = jb.layout == NN_PACK_SHIFT ? (int64_t)pl.num_kb * pl.n_mma
                                                   : (int64_t)pl.n_tiles * pl.num_kb * pl.n_mma * 8;
        if (jb.layout == NN_PACK_TMA) { fill_pack_tma(pw, tp); total = pack_tma_chunks(tp); }
        if (total > max_total) max_total = total;
    }
    {   // quantizer codes once per distinct (parameter, scratch) pair
        CodeJobs cj;
        memset(&cj, 0, sizeof(cj));
        int nc = 0;
        int64_t max_groups = 0;
        for (int i = 0; i < count; ++i) {
            const nn_wprep_job& jb = jobs[i];
            if (!jb.codes || jb.q_bits <= 0) continue;
            if (jb.q_bits > 7) return nn_fail("nn_prepare_weights: the code scratch serves q_bits <= 7%s", "");
            pj.j[i].codes = (const int8_t*)jb.codes;
            bool seen = false;
            for (int k = 0; k < nc; ++k) seen = seen || cj.j[k].codes == (int8_t*)jb.codes;
            if (seen) continue;
            CodeJob& c = cj.j[nc++];
            c.w = jb.w_raw; c.codes = (int8_t*)jb.codes; c.n = (int64_t)jb.Cout * jb.Cin * jb.KHW;
            c.q_hi = pj.j[i].q_hi; c.q_scale = pj.j[i].q_scale; c.q_max = pj.j[i].q_max; c.q_stoch = pj.j[i].q_stoch;
            c.u_inject = jb.u_inject; c.rng = jb.rng;
            if ((c.n + 3) / 4 > max_groups) max_groups = (c.n + 3) / 4;
        }
        if (nc > 0) {
            int gx = (int)((max_groups + 255) / 256);
            if (gx > 4 * nn_num_sms(device)) gx = 4 * nn_num_sms(device);
            k_quant_codes<<<dim3(gx, nc), 256, 0, (cudaStream_t)stream>>>(cj);
            NN_LAUNCH_OK();
        }
    }
    int gx = (int)((max_total + 255) / 256);
    if (gx > 4 * nn_num_sms(device)) gx = 4 * nn_num_sms(device);
    dim3 grid(gx, count);
    k_pack_w_batch<<<grid, 256, 0, (cudaStream_t)stream>>>(pj);
    NN_LAUNCH_OK();
    return 0;
}

int nn_umma_conv_dgrad(const nn_conv_dgrad_args* a, int device, cudaStream_t st) {
    if (a->precision != NN_PREC_BF16)
        return nn_fail("nn_noisy_conv_dgrad: tensor-core path implements NN_PREC_BF16 only%s", "");
    const nn_conv_geom& g = a->g;
    int OH, OW;
    nn_out_hw(g, OH, OW);
    // dgrad(stride 1) == forward conv of gy [B,Cout,OH,OW] with the transposed, tap-flipped weights and
    // padding K-1-pad, producing [B,Cin,H,W]
    {   // conv layers without an STE mask: persistent CTA-pair kernel with TMA-im2col operands over grad_output
        TmaPlan tp;
        const bool can = !a->x_pre && g.stride == 1 &&
                         nn_tma_make_plan(g.Cout, g.KH, g.KW, 1, g.KH - 1 - g.pad, g.Cin, false, g.H, g.W, &tp);
        const int layout = a->w_packed ? a->w_packed_layout : (can ? NN_PACK_TMA : NN_PACK_TILED);
        if (layout == NN_PACK_TMA) {
            if (!can) return nn_fail("nn_noisy_conv_dgrad: w_packed_layout = NN_PACK_TMA is not served for this call%s", "");
            const size_t xp_bytes = (size_t)g.B * OH * OW * tp.Cp * 2;
            const size_t need = (a->gy_packed ? 0 : align_up(xp_bytes, 1024)) + (a->w_packed ? 0 : align_up(tp.wp_bytes, 1024)) + 1024;
            if ((!a->gy_packed || !a->w_packed) && (!a->workspace || (size_t)a->workspace_bytes < need))
                return nn_fail("nn_noisy_conv_dgrad: workspace too small%s (need %lld bytes)", "", (long long)need);
            uint8_t* ws = (uint8_t*)align_up((size_t)a->workspace, 1024);
            const void* xp = a->gy_packed;
            const void* wp = a->w_packed;
            if (!xp) {
                const int64_t total = (int64_t)g.B * OH * OW * (tp.Cp / 8);
                int grid = (int)((total + 255) / 256);
                if (grid > 16 * nn_num_sms(device)) grid = 16 * nn_num_sms(device);
                k_pack_act<<<grid, 256, 0, st>>>(a->gy, (__nv_bfloat16*)ws, g.B, g.Cout, OH * OW, tp.Cp, 0.f);
                NN_LAUNCH_OK();
                xp = ws;
                ws += align_up(xp_bytes, 1024);
            }
            if (!wp) {
                PackWP pw;
                memset(&pw, 0, sizeof(pw));
                pw.w_eff = a->w_eff; pw.w_raw = nullptr; pw.wp = (__nv_bfloat16*)ws;
                pw.Cout = g.Cout; pw.Cin = g.Cin; pw.KHW = g.KH * g.KW; pw.noise_mode = 0; pw.mode = 1; pw.w_code_scale = a->w_code_scale;
                fill_pack_tma(pw, tp);
                const int64_t total = pack_tma_chunks(tp);
                int grid = (int)((total + 255) / 256);
                if (grid > 8 * nn_num_sms(device)) grid = 8 * nn_num_sms(device);
                k_pack_w<<<grid, 256, 0, st>>>(pw);
                NN_LAUNCH_OK();
                wp = ws;
            }
            TmaConvCall c;
            memset(&c, 0, sizeof(c));
            c.pl = tp;
            c.B = g.B; c.H = OH; c.W = OW; c.OH = g.H; c.OW = g.W; c.KH = g.KH; c.KW = g.KW; c.stride = 1; c.pad = g.KH - 1 - g.pad;
            c.Cout = g.Cin; c.xp = xp; c.wp = wp;
            c.y_scale = a->w_code_scale > 0.f ? a->w_code_scale : 1.f; c.s_scale = 1.f;
            c.y = a->gx; c.noise_mode = NN_NOISE_NONE; c.err_flag = nn_umma_err_flag(device);
            return nn_tma_conv_launch(c, device, st);
        }
    }
    Plan pl = make_plan(g.Cout, g.KH * g.KW, g.Cin, true, false, false, (int64_t)g.B * OH * OW,
                        (g.B * g.H * g.W + 127) / 128);
    const size_t need = align_up(pl.xp_bytes, 1024) + align_up(pl.wp_bytes, 1024) + 1024;
    if (!a->workspace || (size_t)a->workspace_bytes < need)
        return nn_fail("nn_noisy_conv_dgrad: workspace too small%s (need %lld bytes)", "", (long long)need);
    uint8_t* ws = (uint8_t*)align_up((size_t)a->workspace, 1024);
    __nv_bfloat16* xp = (__nv_bfloat16*)ws;
    __nv_bfloat16* wp = (__nv_bfloat16*)(ws + align_up(pl.xp_bytes, 1024));
    if (a->gy_packed) {
        xp = (__nv_bfloat16*)a->gy_packed;
    } else {
        const int64_t total = (int64_t)g.B * OH * OW * (pl.Cp / 8);
        int grid = (int)((total + 255) / 256);
        if (grid > 16 * nn_num_sms(device)) grid = 16 * nn_num_sms(device);
        k_pack_act<<<grid, 256, 0, st>>>(a->gy, xp, g.B, g.Cout, OH * OW, pl.Cp, 0.f);
        NN_LAUNCH_OK();
    }
    if (a->w_packed) {
        wp = (__nv_bfloat16*)a->w_packed;
    } else {
        PackWP pw;
        memset(&pw, 0, sizeof(pw));
        pw.w_eff = a->w_eff; pw.w_raw = nullptr; pw.wp = wp;
        pw.Cout = g.Cout; pw.Cin = g.Cin; pw.KHW = g.KH * g.KW; pw.Cp = pl.Cp; pw.n_t = pl.n_t; pw.n_mma = pl.n_mma;
        pw.num_kb = pl.num_kb; pw.n_tiles = pl.n_tiles; pw.main_col = pl.main_col; pw.sig_col = -1; pw.wsum_col = -1;
        pw.noise_mode = 0; pw.mode = 1; pw.w_code_scale = a->w_code_scale;
        const int64_t total = (int64_t)pl.n_tiles * pl.num_kb * pl.n_mma * 8;
        int grid = (int)((total + 255) / 256);
        if (grid > 8 * nn_num_sms(device)) grid = 8 * nn_num_sms(device);
        k_pack_w<<<grid, 256, 0, st>>>(pw);
        NN_LAUNCH_OK();
    }
    UmmaP p;
    memset(&p, 0, sizeof(p));
    p.B = g.B; p.H = OH; p.W = OW; p.Cp = pl.Cp; p.KH = g.KH; p.KW = g.KW; p.stride = 1; p.pad = g.KH - 1 - g.pad;
    p.OH = g.H; p.OW = g.W; p.M = g.B * g.H * g.W; p.Cout = g.Cin; p.n_t = pl.n_t; p.n_mma = pl.n_mma;
    p.num_kb = pl.num_kb; p.stages = pl.stages; p.acc_cols = pl.acc_cols; p.ring_bytes = pl.ring_bytes;
    p.main_col = pl.main_col; p.sig_col = -1; p.wsum_col = -1;
    p.xp = xp; p.wp = wp; p.y_scale = a->w_code_scale > 0.f ? a->w_code_scale : 1.f; p.s_scale = 1.f;
    p.y = a->gx; p.noise_mode = NN_NOISE_NONE;
    p.mask_x = a->x_pre; p.mask_lo = (float)a->x_lo; p.mask_hi = (float)a->x_hi;
    p.err_flag = nn_umma_err_flag(device);
    if (g.KH != g.KW && (g.KH - 1 - g.pad) != (g.KW - 1 - g.pad))
        return nn_fail("nn_noisy_conv_dgrad: non-square kernels not supported on the tensor-core path%s", "");
    return launch_umma(p, pl, st);
}

namespace {
struct WgPlan {
    int Cp, Coutp, Ktot, n_tiles_k, NT, ktot_pad, m_tiles_n, num_kb, splits, kb_per_split, stages;
    size_t xp_bytes, gyp_bytes, partial_bytes, smem_bytes;
};
WgPlan make_wg_plan(const nn_conv_geom& g, int device) {
    WgPlan w;
    int OH, OW;
    nn_out_hw(g, OH, OW);
    const int64_t Mpix = (int64_t)g.B * OH * OW;
    w.Cp = pad_to(g.Cin, 8);
    w.Coutp = pad_to(g.Cout, 8);
    w.Ktot = g.KH * g.KW * w.Cp;
    w.n_tiles_k = (w.Ktot + 255) / 256;
    w.NT = 64;
    while (w.NT < (w.Ktot + w.n_tiles_k - 1) / w.n_tiles_k) w.NT <<= 1;      // 64 / 128 / 256 (lane mapping needs 2^k chunks)
    w.ktot_pad = w.n_tiles_k * w.NT;
    w.m_tiles_n = (g.Cout + 127) / 128;
    w.num_kb = (int)((Mpix + 63) / 64);
    const int tiles = w.n_tiles_k * w.m_tiles_n;
    int splits = (nn_num_sms(device) + tiles - 1) / tiles;
    if (splits > w.num_kb) splits = w.num_kb;
    if (splits < 1) splits = 1;
    w.kb_per_split = (w.num_kb + splits - 1) / splits;
    w.splits = (w.num_kb + w.kb_per_split - 1) / w.kb_per_split;
    const int stage_bytes = UM_A_STAGE + w.NT * 128;
    w.stages = (192 * 1024) / stage_bytes;
    if (w.stages > 4) w.stages = 4;
    if (w.stages < 2) w.stages = 2;
    w.smem_bytes = 1024 + (size_t)w.stages * stage_bytes + 16 * w.stages + 64 + (size_t)(w.NT / 8) * 16 + 16;
    w.xp_bytes = (size_t)g.B * g.H * g.W * w.Cp * 2;
    w.gyp_bytes = (size_t)Mpix * w.Coutp * 2;
    w.partial_bytes = (size_t)w.splits * g.Cout * w.ktot_pad * 4;
    return w;
}
}  // namespace



namespace {
struct WgShiftPlan {
    int n_planes, n_row, n_chunks, b_pixels, a_stage, b_stage, stages, grid;
    int64_t plane_stride;
    size_t smem_bytes, xp_bytes, gyv_bytes, partial_bytes;
};
bool make_wg_shift_plan(const nn_conv_geom& g, int device, WgShiftPlan* out) {
    if (!g_shift_enable) return false;
    if (g.Cin > 8 || g.stride != 1 || g.pad != 0 || g.KH > g.H || g.KW > g.W || g.W >= 2048 || g.Cout > 128) return false;
    WgShiftPlan w;
    w.n_planes = (g.Cout + 7) / 8;
    w.n_row = pad_to(g.KW * 8, 16);
    if (w.n_row > 64) return false;                     // k_wgrad_shift<16 / 32 / 48 / 64>
    const int64_t total = (int64_t)g.B * g.H * g.W;
    w.plane_stride = (total + WS_KP - 1) / WS_KP * WS_KP;
    w.n_chunks = (int)(w.plane_stride / WS_KP);
    w.b_pixels = pad_to(WS_KP + (g.KH - 1) * g.W + w.n_row / 8, 8);
    w.a_stage = w.n_planes * WS_KP * 16;
    w.b_stage = pad_to(w.b_pixels * 16, 128);
    const int fixed = 128 + 16 * WS_KP * 16 + 16 * WS_MAX_STAGES + 64;
    w.stages = (190 * 1024 - fixed) / (w.a_stage + w.b_stage);         // one CTA per SM (accumulator registers)
    if (w.stages > WS_MAX_STAGES) w.stages = WS_MAX_STAGES;
    if (w.stages < 2) return false;
    w.smem_bytes = (size_t)fixed + (size_t)w.stages * (w.a_stage + w.b_stage);
    w.grid = nn_num_sms(device);
    if (w.grid > w.n_chunks) w.grid = w.n_chunks;
    w.xp_bytes = (size_t)total * 16;
    w.gyv_bytes = (size_t)w.n_planes * w.plane_stride * 16;
    {   // rows of 256 columns (k_wgrad_tma_reduce's remainder format) when the taps fit, else packed rows
        const int kc = g.KH * g.KW * 8;
        w.partial_bytes = (size_t)w.grid * g.Cout * (kc <= 256 ? 256 : kc) * sizeof(float);
    }
    if (out) *out = w;
    return true;
}
}  // namespace

int64_t nn_umma_wgrad_workspace(const nn_conv_geom* g, int, int device) {
    WgPlan w = make_wg_plan(*g, device);
    size_t partial_bytes = w.partial_bytes;
    {
        int OH, OW;
        nn_out_hw(*g, OH, OW);
        TmaWgradPlan tw;
        if (nn_tma_wgrad_plan(g->Cin, g->KH, g->KW, g->stride, g->pad, g->Cout, (int64_t)g->B * OH * OW, device, &tw) &&
            tw.partial_bytes > partial_bytes)
            partial_bytes = tw.partial_bytes;
    }
    size_t need = align_up(w.xp_bytes, 1024) + align_up(w.gyp_bytes, 1024) + align_up(partial_bytes, 1024) + 2048;
    WgShiftPlan sw;
    if (make_wg_shift_plan(*g, device, &sw)) {
        const size_t ns = align_up(sw.xp_bytes, 1024) + align_up(sw.gyv_bytes, 1024) + align_up(sw.partial_bytes, 1024) + 2048;
        if (ns > need) need = ns;
    }
    return (int64_t)need;
}

extern "C" int nn_conv_wgrad_pack_layout(const nn_conv_geom* g, int32_t precision, int device) {
    if (!g || precision != NN_PREC_BF16) return NN_PACK_TILED;
    return make_wg_shift_plan(*g, device, nullptr) ? NN_PACK_SHIFT : NN_PACK_TILED;
}
extern "C" int64_t nn_conv_gy_planes_bytes(const nn_conv_geom* g) {
    if (!g) return 0;
    const int64_t total = (int64_t)g->B * g->H * g->W;
    return (int64_t)((g->Cout + 7) / 8) * ((total + WS_KP - 1) / WS_KP * WS_KP) * 16;
}

static int shift_conv_wgrad(const nn_conv_wgrad_args* a, const WgShiftPlan& w, int device, cudaStream_t st) {
    const nn_conv_geom& g = a->g;
    int OH, OW;
    nn_out_hw(g, OH, OW);
    const bool gy_ready = a->gy_packed && a->gy_packed_layout == NN_PACK_SHIFT;
    const size_t need = (a->x_packed ? 0 : align_up(w.xp_bytes, 1024)) + (gy_ready ? 0 : align_up(w.gyv_bytes, 1024)) +
                        align_up(w.partial_bytes, 1024) + 1024;
    if (!a->workspace || (size_t)a->workspace_bytes < need)
        return nn_fail("nn_noisy_conv_wgrad: workspace too small%s (need %lld bytes)", "", (long long)need);
    uint8_t* ws = (uint8_t*)align_up((size_t)a->workspace, 1024);
    const int sms = nn_num_sms(device);
    const __nv_bfloat16* xp = (const __nv_bfloat16*)a->x_packed;
    if (!xp) {
        const int64_t total = (int64_t)g.B * g.H * g.W;
        int grid = (int)((total + 255) / 256);
        if (grid > 16 * sms) grid = 16 * sms;
        k_pack_act<<<grid, 256, 0, st>>>(a->x, (__nv_bfloat16*)ws, g.B, g.Cin, g.H * g.W, 8, a->a_code_scale);
        NN_LAUNCH_OK();
        xp = (const __nv_bfloat16*)ws;
        ws += align_up(w.xp_bytes, 1024);
    }
    const __nv_bfloat16* gyv = (const __nv_bfloat16*)a->gy_packed;
    if (!gy_ready) {
        if (!a->gy) return nn_fail("nn_noisy_conv_wgrad: the shift path needs gy (fp32) or a NN_PACK_SHIFT gy_packed%s", "");
        const int64_t total = w.plane_stride * w.n_planes;
        int grid = (int)((total + 255) / 256);
        if (grid > 16 * sms) grid = 16 * sms;
        k_pack_gy_planes<<<grid, 256, 0, st>>>(a->gy, (__nv_bfloat16*)ws, g.B, g.Cout, g.H, g.W, OH, OW, w.n_planes, w.plane_stride);
        NN_LAUNCH_OK();
        gyv = (const __nv_bfloat16*)ws;
        ws += align_up(w.gyv_bytes, 1024);
    }
    float* partial = (float*)ws;
    WgShiftP p;
    memset(&p, 0, sizeof(p));
    p.H = g.H; p.W = g.W; p.OH = OH; p.OW = OW; p.KH = g.KH; p.KW = g.KW; p.Cout = g.Cout;
    p.n_planes = w.n_planes; p.n_row = w.n_row; p.n_chunks = w.n_chunks; p.b_pixels = w.b_pixels;
    p.a_stage = w.a_stage; p.b_stage = w.b_stage; p.stages = w.stages;
    p.total_pixels = (long long)g.B * g.H * g.W; p.plane_stride = w.plane_stride;
    p.xp = xp; p.gyv = gyv; p.partial = partial; p.err_flag = nn_umma_err_flag(device);
    NN_ONCE_PER_DEVICE({
        NN_CUDA_OK(cudaFuncSetAttribute(k_wgrad_shift<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        NN_CUDA_OK(cudaFuncSetAttribute(k_wgrad_shift<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        NN_CUDA_OK(cudaFuncSetAttribute(k_wgrad_shift<48>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        NN_CUDA_OK(cudaFuncSetAttribute(k_wgrad_shift<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    });
#ifdef NN_KDEBUG
    static const bool want_dbg = getenv("NN_UMMA_DEBUG") != nullptr;
#else
    const bool want_dbg = false;
#endif
    if (want_dbg) {
        const size_t rows = (size_t)w.grid * 16;
        if (rows > g_dbg_ctas) {
            if (g_dbg_buf) cudaFree(g_dbg_buf);
            cudaMalloc(&g_dbg_buf, rows * 8 * sizeof(long long));
            g_dbg_ctas = rows;
        }
        cudaMemsetAsync(g_dbg_buf, 0, rows * 8 * sizeof(long long), st);
        p.dbg = g_dbg_buf;
        g_dbg_last = rows;
    }
    const int kcols = g.KH * g.KW * 8;
    p.row_pitch = kcols <= 256 ? 256 : kcols;
    if (w.n_row == 16) k_wgrad_shift<16><<<w.grid, WS_THREADS, w.smem_bytes, st>>>(p);
    else if (w.n_row == 32) k_wgrad_shift<32><<<w.grid, WS_THREADS, w.smem_bytes, st>>>(p);
    else if (w.n_row == 48) k_wgrad_shift<48><<<w.grid, WS_THREADS, w.smem_bytes, st>>>(p);
    else k_wgrad_shift<64><<<w.grid, WS_THREADS, w.smem_bytes, st>>>(p);
    NN_LAUNCH_OK();
    const float scale = a->a_code_scale > 0.f ? a->a_code_scale : 1.f;
    if (kcols <= 256) {
        // the per-CTA partials are [grid][Cout][256] with column tap * 8 + c: the remainder format of k_wgrad_tma_reduce
        // (float4 loads, groups of partials per block; w.grid = 2 x SMs partials is a long chain for one thread)
        WgRedP r;
        memset(&r, 0, sizeof(r));
        r.tail = partial; r.n_tail = w.grid; r.Cout = g.Cout; r.Cin = g.Cin; r.KHW = g.KH * g.KW; r.n_c64 = 0; r.cols_pad = 0;
        r.scale = scale; r.lo = (float)a->w_lo; r.hi = (float)a->w_hi; r.gw = a->gw; r.w_raw = a->w_raw;
        r.nb_main = 0; r.g_main = 1;
        const int64_t q_tail = (int64_t)g.Cout * 64;
        int G = 1;
        while (G < 32 && q_tail * G < 131072 && r.n_tail >= 8 * G) G <<= 1;
        r.g_tail = G;
        k_wgrad_tma_reduce<<<(int)((q_tail + 256 / G - 1) / (256 / G)), 256, 0, st>>>(r);
        NN_LAUNCH_OK();
        return 0;
    }
    const int64_t n = (int64_t)g.Cout * kcols;
    int rb = (int)((n + 31) / 32);
    if (rb > 16 * sms) rb = 16 * sms;
    k_wgrad_umma_reduce2<<<rb, 256, 0, st>>>(partial, w.grid, g.Cout, g.Cin, g.KH * g.KW, 8, kcols, scale, a->gw, a->w_raw,
                                             (float)a->w_lo, (float)a->w_hi);
    NN_LAUNCH_OK();
    return 0;
}

int nn_umma_conv_wgrad(const nn_conv_wgrad_args* a, int device, cudaStream_t st) {
    if (a->precision != NN_PREC_BF16)
        return nn_fail("nn_noisy_conv_wgrad: tensor-core path implements NN_PREC_BF16 only%s", "");
    const nn_conv_geom& g = a->g;
    int OH, OW;
    nn_out_hw(g, OH, OW);
    {   // narrow-input layers: both operands read in place (no im2col gather)
        WgShiftPlan sw;
        const bool can = make_wg_shift_plan(g, device, &sw);
        const bool want = a->gy_packed ? a->gy_packed_layout == NN_PACK_SHIFT : can;
        if (want) {
            if (!can) return nn_fail("nn_noisy_conv_wgrad: gy_packed_layout = NN_PACK_SHIFT is not served for this geometry%s", "");
            return shift_conv_wgrad(a, sw, device, st);
        }
    }
    WgPlan w = make_wg_plan(g, device);
    TmaWgradPlan tw;
    const bool use_tma = nn_tma_wgrad_plan(g.Cin, g.KH, g.KW, g.stride, g.pad, g.Cout, (int64_t)g.B * OH * OW, device, &tw);
    if (use_tma) w.partial_bytes = tw.partial_bytes;
    const size_t need = align_up(w.xp_bytes, 1024) + align_up(w.gyp_bytes, 1024) + align_up(w.partial_bytes, 1024) + 1024;
    if (!a->workspace || (size_t)a->workspace_bytes < need)
        return nn_fail("nn_noisy_conv_wgrad: workspace too small%s (need %lld bytes)", "", (long long)need);
    uint8_t* ws = (uint8_t*)align_up((size_t)a->workspace, 1024);
    __nv_bfloat16* xp = (__nv_bfloat16*)ws;
    __nv_bfloat16* gyp = (__nv_bfloat16*)(ws + align_up(w.xp_bytes, 1024));
    float* partial = (float*)(ws + align_up(w.xp_bytes, 1024) + align_up(w.gyp_bytes, 1024));
    const int sms = nn_num_sms(device);
    if (a->x_packed) {
        xp = (__nv_bfloat16*)a->x_packed;
    } else {
        int64_t total = (int64_t)g.B * g.H * g.W * (w.Cp / 8);
        int grid = (int)((total + 255) / 256);
        if (grid > 16 * sms) grid = 16 * sms;
        k_pack_act<<<grid, 256, 0, st>>>(a->x, xp, g.B, g.Cin, g.H * g.W, w.Cp, a->a_code_scale);
        NN_LAUNCH_OK();
    }
    if (a->gy_packed) {
        gyp = (__nv_bfloat16*)a->gy_packed;
    } else {
        int64_t total = (int64_t)g.B * OH * OW * (w.Coutp / 8);
        int grid = (int)((total + 255) / 256);
        if (grid > 16 * sms) grid = 16 * sms;
        k_pack_act<<<grid, 256, 0, st>>>(a->gy, gyp, g.B, g.Cout, OH * OW, w.Coutp, 0.f);
        NN_LAUNCH_OK();
    }
    const float scale = a->a_code_scale > 0.f ? a->a_code_scale : 1.f;
    if (use_tma) {      // both operands staged by the copy engine (im2col / tiled tensor maps)
        TmaWgradCall c;
        memset(&c, 0, sizeof(c));
        c.pl = tw;
        c.B = g.B; c.H = g.H; c.W = g.W; c.OH = OH; c.OW = OW; c.KH = g.KH; c.KW = g.KW; c.stride = g.stride; c.pad = g.pad;
        c.Cout = g.Cout; c.xp = xp; c.gyp = gyp; c.partial = partial; c.err_flag = nn_umma_err_flag(device);
        if (nn_tma_wgrad_launch(c, device, st)) return 1;
        WgRedP r;
        memset(&r, 0, sizeof(r));
        r.main = partial;
        r.tail = tw.tail_w ? reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(partial) + tw.main_bytes) : nullptr;
        r.splits = tw.splits; r.n_tail = tw.splits; r.Cout = g.Cout; r.Cin = g.Cin; r.KHW = g.KH * g.KW; r.n_c64 = tw.n_c64;
        r.cols_pad = tw.cols_pad; r.scale = scale; r.lo = (float)a->w_lo; r.hi = (float)a->w_hi; r.gw = a->gw; r.w_raw = a->w_raw;
        auto groups = [](int64_t quads, int cnt) {      // ~128 k threads, at least ~4 partials per thread
            int G = 1;
            while (G < 32 && quads * G < 131072 && cnt >= 8 * G) G <<= 1;
            return G;
        };
        const int64_t q_main = (int64_t)g.Cout * (tw.cols_pad / 4), q_tail = (int64_t)g.Cout * 64;
        r.g_main = groups(q_main, r.splits);
        r.g_tail = tw.tail_w ? groups(q_tail, r.n_tail) : 1;
        r.nb_main = (int)((q_main + 256 / r.g_main - 1) / (256 / r.g_main));
        const int nb_tail = tw.tail_w ? (int)((q_tail + 256 / r.g_tail - 1) / (256 / r.g_tail)) : 0;
        k_wgrad_tma_reduce<<<r.nb_main + nb_tail, 256, 0, st>>>(r);
        NN_LAUNCH_OK();
        return 0;
    }
    WgUP p;
    memset(&p, 0, sizeof(p));
    p.B = g.B; p.H = g.H; p.W = g.W; p.Cp = w.Cp; p.KH = g.KH; p.KW = g.KW; p.stride = g.stride; p.pad = g.pad;
    p.OH = OH; p.OW = OW; p.Mpix = g.B * OH * OW; p.Cout = g.Cout; p.Coutp = w.Coutp;
    p.Ktot = w.Ktot; p.NT = w.NT; p.ktot_pad = w.ktot_pad; p.num_kb = w.num_kb; p.kb_per_split = w.kb_per_split;
    p.stages = w.stages; p.xp = xp; p.gyp = gyp; p.partial = partial;
    p.err_flag = nn_umma_err_flag(device);
    NN_ONCE_PER_DEVICE({
        NN_CUDA_OK(cudaFuncSetAttribute(k_wgrad_umma, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    });
    dim3 grid(w.n_tiles_k, w.m_tiles_n, w.splits);
    k_wgrad_umma<<<grid, UM_THREADS, w.smem_bytes, st>>>(p);
    NN_LAUNCH_OK();
    const int64_t n = (int64_t)g.Cout * w.ktot_pad;
    if (w.splits >= 64) {       // many splits, few columns (conv1): shorten the serial chain over splits 8x
        int rb = (int)((n + 31) / 32);
        if (rb > 16 * sms) rb = 16 * sms;
        k_wgrad_umma_reduce2<<<rb, 256, 0, st>>>(partial, w.splits, g.Cout, g.Cin, g.KH * g.KW, w.Cp, w.ktot_pad, scale,
                                                 a->gw, a->w_raw, (float)a->w_lo, (float)a->w_hi);
    } else {
        int rb = (int)((n + 255) / 256);
        if (rb > 8 * sms) rb = 8 * sms;
        k_wgrad_umma_reduce<<<rb, 256, 0, st>>>(partial, w.splits, g.Cout, g.Cin, g.KH * g.KW, w.Cp, w.ktot_pad, scale,
                                                a->gw, a->w_raw, (float)a->w_lo, (float)a->w_hi);
    }
    NN_LAUNCH_OK();
    return 0;
}
