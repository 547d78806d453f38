// Persistent implicit-GEMM conv with TMA-staged operands (sm_90a): the tiled noisy-conv forward and the dgrad of the
// layers whose im2col rows cannot be read in place (conv2 of NoisyNet, the ResNet 3x3 layers).
//
//   D[m, n] = sum_{tap, c} X[pixel(m) + tap, c] * Wp[n, tap, c]      m = output pixel, n = accumulator column
//
// * A operand: ONE cp.async.bulk.tensor (im2col-mode tensor map, cuTensorMapEncodeIm2col) per (tap, channel chunk)
//   lands 128 output pixels x 64 channels as a SWIZZLE_128B K-major tile; the channel remainder of a tap is a second,
//   narrower box (16 / 32 channels -> SWIZZLE_32B / 64B tile, its own descriptor kind) instead of padding every tap to
//   a multiple of 64 channels (65 channels -> K = 80 per tap, not 128).  Padding taps and tile rows past the tensor are
//   zero-filled by the TMA unit: no thread computes an address.
// * B operand: pre-swizzled weight image [n-tile][tap][group][half][chunk rows]; per stage and chunk two tiled
//   tensor-map copies (the two row halves) land the chunk's n_mma rows contiguously.
// * CTA pairs: clusters of two CTAs walk adjacent 128-pixel tiles of one n-tile in lockstep; each multicasts one of the
//   two weight row halves to both, so the weights (65 % of the operand bytes of conv2's forward) cross L2 once per pair.
// * Persistent: a pair walks (two 128-pixel tiles, n-tile) items.  Two MMA warpgroups (64 pixels each) accumulate the
//   main and sigma^2 columns in registers with ONE wgmma per k16 step over the full width (m64n240k16 for conv2), keep
//   one ring stage's wgmmas in flight, and run the epilogue (scale, Philox / Box-Muller current noise -> NCHW stores)
//   straight from the wgmma fragments, while the producers already fill the ring with the next item's operands.
// * Warp roles: warps 0-7 the two MMA / epilogue warpgroups, warps 8 .. 8 + P - 1 producers (one elected thread each; a
//   thread owns whole stages round-robin, since a tensor-map copy keeps its issuing thread busy for hundreds of cycles).
#include "nn_conv_tma.h"

#include <cuda.h>

#include "nn_wgmma.cuh"

namespace {

constexpr int TC_MAX_STAGES = 8;

struct TmaConvP {
    CUtensorMap map64, map_tail;         // im2col maps: 64-channel SWIZZLE_128B box, tail box
    CUtensorMap mapb64, mapb_tail;       // weight image as rows of 128 B / of the tail width: boxes of n_half rows
    int M, OH, OW, Cout, stride, pad, KW, taps;
    int n_c64, tail_w, nc, gpt, n_groups;
    int n_mma, n_half, n_tiles;
    int stages, a_stage, b_stage, n_prod, tap_bytes;
    float y_scale, s_scale;
    float *y, *y_noisy;
    float current;
    const float* scale_dev;
    const float* z_inject;               // EPI 3: N(0,1) draws of the caller (parity hook), [B, Cout, OH, OW]
    nn_rng rng;
    int* err_flag;
};

// The wgmmas of one ring stage of k_conv_tma: KA k16 steps of the stage's first channel chunk, KB of its second (0: none),
// committed as one group; returns when the previous stage's group has completed.  scale_d of the first one: 0 starts the
// accumulators of an item.
template <int N, int KA, int KB>
__device__ __forceinline__ void conv_stage_mma(float* acc, uint64_t ad_a, uint64_t bd_a, uint64_t ad_b, uint64_t bd_b, int acc0) {
    wg_fence();
#pragma unroll
    for (int k = 0; k < KA; ++k) wgmma_c<N, 0, 0>(acc, ad_a + 2 * k, bd_a + 2 * k, k == 0 ? acc0 : 1);
#pragma unroll
    for (int k = 0; k < KB; ++k) wgmma_c<N, 0, 0>(acc, ad_b + 2 * k, bd_b + 2 * k, 1);
    wg_commit();
    wg_wait_1();            // this stage's wgmmas stay in flight; the previous stage's have completed
}

// EPI 1: noisy (main + sigma accumulators, Philox z), EPI 2: plain, EPI 3: noisy with injected z (parity tests).
// NT = main accumulator columns of an n-tile (the plan's n_t); the MMA width is NT, or 2 NT with the sigma^2 columns.
// Launched as clusters of two CTAs (rank r = 0 / 1) that walk adjacent m-tiles (2 mp + r) of the same n-tile in lockstep:
// each producer copies its own A and multicasts weight row half r to both CTAs, so a weight stage crosses L2 once per pair.
template <int EPI, int NT>
__global__ void __launch_bounds__((8 + 2) * 32, 1)
k_conv_tma(const __grid_constant__ TmaConvP p) {
    constexpr bool noise = EPI != 2;
    constexpr int N = noise ? 2 * NT : NT;       // one wgmma per k16 step: [main | sigma^2] columns (fragment offset NT / 2)
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int S = p.stages;
    const uint32_t stage_bytes = (uint32_t)(p.a_stage + p.b_stage);
    const uint32_t bar_base = base + (uint32_t)S * stage_bytes;
    const uint32_t full_bar = bar_base, empty_bar = bar_base + 8u * TC_MAX_STAGES;

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);          // warp-uniform for the compiler: role branches are convergent
    const int P = p.n_prod;
    const uint32_t rank = cluster_ctarank(), peer = rank ^ 1u;
    const int n_mt = (p.M + 127) >> 7, pairs = ((n_mt + 1) >> 1) * p.n_tiles;
    const int cl0 = blockIdx.x >> 1, n_cl = gridDim.x >> 1;

    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full_bar + 8 * s, 1);          // the producer's arrive.expect_tx (A + both weight halves)
            mbar_init(empty_bar + 8 * s, 4);         // both MMA warpgroups of both CTAs have read the stage
        }
        fence_mbar_init();
        tma_prefetch_desc(&p.map64);
        tma_prefetch_desc(&p.map_tail);
        tma_prefetch_desc(&p.mapb64);
        tma_prefetch_desc(&p.mapb_tail);
    }
    cluster_sync();                                  // the peer's barriers are initialised before any copy or arrival reaches them
    const int ohw = p.OH * p.OW;

    if (warp >= 8 && warp < 8 + P) {
        // ---------------------------------------------------------------- producers
        const int pw = warp - 8;
        int s = 0, turn = 0;                                 // ring stage and producer turn of the current group (no div / mod)
        uint32_t eph = 1u;                                   // parity to wait for on the stage's empty barrier
        // (no function call inside the role loops: uniform registers do not survive calls -- the loops break out instead)
        int fail = 0;
        for (int pi = cl0; pi < pairs && !fail; pi += n_cl) {
            const int mp = pi / p.n_tiles, nt = pi - mp * p.n_tiles;
            // the odd last m-tile: rank 1 reloads its partner's A (no stores follow) because the partner needs its weight half
            const int mt = min(2 * mp + (int)rank, n_mt - 1);
            const int m0 = mt * 128;
            const int b0 = m0 / ohw, r0 = m0 - b0 * ohw, oh0 = r0 / p.OW, ow0 = r0 - oh0 * p.OW;
            const int iw0 = ow0 * p.stride - p.pad, ih0 = oh0 * p.stride - p.pad;
            const long long wt = (long long)nt * p.taps * p.tap_bytes;           // byte offset of this n-tile's weight image
            int kh = 0, kw = 0, gi = 0;
            for (int g = 0; g < p.n_groups; ++g) {
                if (turn == pw) {
                    if (!mbar_wait_backoff(empty_bar + 8 * s, eph)) { fail = 401; break; }
                    const int ca = 2 * gi, cb = 2 * gi + 1;
                    const int wa = ca < p.n_c64 ? 64 : p.tail_w;
                    const int wb = cb < p.nc ? (cb < p.n_c64 ? 64 : p.tail_w) : 0;
                    const uint32_t half_bytes = (uint32_t)(p.n_half * 2 * (wa + wb));      // one row half of the group's weights
                    const uint32_t a_dst = base + (uint32_t)s * stage_bytes, b_dst = a_dst + (uint32_t)p.a_stage;
                    const uint32_t bar = full_bar + 8 * s;
                    if (elect_one_sync()) {
                        mbar_arrive_expect_tx(bar, (uint32_t)(256 * (wa + wb)) + 2u * half_bytes);
                        tma_im2col_4d(a_dst, ca < p.n_c64 ? &p.map64 : &p.map_tail, bar, 64 * ca, iw0, ih0, b0, (uint16_t)kw, (uint16_t)kh);
                        if (wb) tma_im2col_4d(a_dst + 256u * (uint32_t)wa, cb < p.n_c64 ? &p.map64 : &p.map_tail, bar, 64 * cb, iw0, ih0, b0,
                                              (uint16_t)kw, (uint16_t)kh);
                        const int tap = kh * p.KW + kw;
                        // chunk a of the group: rows [half 0 | half 1] at b_dst; chunk b after all n_mma rows of chunk a.
                        // This CTA's half (h = rank) goes to both CTAs of the pair.
                        const int h = (int)rank;
                        const long long boff = wt + (long long)tap * p.tap_bytes + (long long)gi * (p.n_half * 512) + (long long)h * half_bytes;
                        const uint32_t da = b_dst + (uint32_t)(h * p.n_half * 2 * wa);
                        if (wa == 64) tma_tile_2d_mc(da, &p.mapb64, bar, 0, (int)(boff >> 7), 0x3);
                        else tma_tile_2d_mc(da, &p.mapb_tail, bar, 0, (int)(boff / (2 * wa)), 0x3);
                        if (wb) {
                            const long long boff2 = boff + (long long)p.n_half * 2 * wa;
                            const uint32_t db = b_dst + (uint32_t)(p.n_mma * 2 * wa + h * p.n_half * 2 * wb);
                            if (wb == 64) tma_tile_2d_mc(db, &p.mapb64, bar, 0, (int)(boff2 >> 7), 0x3);
                            else tma_tile_2d_mc(db, &p.mapb_tail, bar, 0, (int)(boff2 / (2 * wb)), 0x3);
                        }
                    }
                    __syncwarp();
                }
                if (++gi == p.gpt) { gi = 0; if (++kw == p.KW) { kw = 0; ++kh; } }
                if (++turn == P) turn = 0;
                if (++s == S) { s = 0; eph ^= 1u; }
            }
        }
        if (fail) nn_pipeline_abort(p.err_flag, fail);
        __syncwarp();
    } else if (warp < 8) {
        // ---------------------------------------------------------------- MMA warpgroups + epilogue
        const int wg = warp >> 2, wt = tid & 127;
        float coef = 0.f;
        NnRng rs = {0, 0, 0, 0};
        if (noise) { coef = nn_noise_coef(*p.scale_dev, p.current); rs = nn_rng_load(p.rng); }
        const int ngrp = (p.Cout + 3) >> 2;
        const float y_scale = p.y_scale, s_scale = p.s_scale;
        const int kt = p.tail_w >> 4;
        const bool releaser = (warp & 3) == 0;
        int s = 0, fail = 0;
        uint32_t fph = 0u;                                   // parity to wait for on the stage's full barrier
        for (int pi = cl0; pi < pairs && !fail; pi += n_cl) {
            const int mp = pi / p.n_tiles, nt = pi - mp * p.n_tiles;
            const int mt = 2 * mp + (int)rank;
            float acc[N / 2];
            int gi = 0, prev = 0;
            for (int g = 0; g < p.n_groups; ++g) {
                if (!mbar_wait(full_bar + 8 * s, fph)) { fail = 403; break; }
                const int ca = 2 * gi, cb = 2 * gi + 1;
                const bool has_b = cb < p.nc;
                const int wa = ca < p.n_c64 ? 64 : p.tail_w, wb = has_b ? (cb < p.n_c64 ? 64 : p.tail_w) : 0;
                const uint32_t a_s = base + (uint32_t)s * stage_bytes, b_s = a_s + (uint32_t)p.a_stage;
                // chunk a: A at a_s, B at b_s (main rows, then the sigma^2 rows); chunk b: A after chunk a's 128 rows, B after
                // its n_mma rows.  K-major tiles with rows of 2 w bytes.
                const uint64_t ad_a = gmma_desc_kmajor(a_s + (uint32_t)(wg * 64 * 2 * wa), 2u * (uint32_t)wa);
                const uint64_t bd_a = gmma_desc_kmajor(b_s, 2u * (uint32_t)wa);
                const uint32_t a_b = a_s + 256u * (uint32_t)wa, b_b = b_s + (uint32_t)(p.n_mma * 2 * wa);
                const uint64_t ad_b = has_b ? gmma_desc_kmajor(a_b + (uint32_t)(wg * 64 * 2 * wb), 2u * (uint32_t)wb) : 0;
                const uint64_t bd_b = has_b ? gmma_desc_kmajor(b_b, 2u * (uint32_t)wb) : 0;
                const int ka = wa == 64 ? 4 : kt, kb = wb == 64 ? 4 : (wb ? kt : 0);
                const int acc0 = g != 0 ? 1 : 0;
                // one straight-line sequence per stage shape (k16 steps of chunks a, b), fence to wait: a branch or a loop back
                // edge between two wgmmas, or between them and the wait, makes ptxas insert a warpgroup.arrive there
                switch (8 * ka + kb) {
                    case 8 * 4 + 4: conv_stage_mma<N, 4, 4>(acc, ad_a, bd_a, ad_b, bd_b, acc0); break;
                    case 8 * 4 + 2: conv_stage_mma<N, 4, 2>(acc, ad_a, bd_a, ad_b, bd_b, acc0); break;
                    case 8 * 4 + 1: conv_stage_mma<N, 4, 1>(acc, ad_a, bd_a, ad_b, bd_b, acc0); break;
                    case 8 * 4: conv_stage_mma<N, 4, 0>(acc, ad_a, bd_a, ad_b, bd_b, acc0); break;
                    case 8 * 2: conv_stage_mma<N, 2, 0>(acc, ad_a, bd_a, ad_b, bd_b, acc0); break;
                    default: conv_stage_mma<N, 1, 0>(acc, ad_a, bd_a, ad_b, bd_b, acc0); break;      // 8 * 1: a 16-channel tail alone
                }
                // the previous stage's operands may be refilled
                if (g != 0 && releaser && elect_one_sync()) {
                    mbar_arrive(empty_bar + 8 * prev);
                    mbar_arrive_cluster(cluster_map(empty_bar + 8 * prev, peer));
                }
                __syncwarp();
                prev = s;
                if (++gi == p.gpt) gi = 0;
                if (++s == S) { s = 0; fph ^= 1u; }
            }
            if (fail) break;
            wg_wait_all();
            wg_fence_regs<N / 2>(acc);
            if (releaser && elect_one_sync()) {
                mbar_arrive(empty_bar + 8 * prev);
                mbar_arrive_cluster(cluster_map(empty_bar + 8 * prev, peer));
            }
            __syncwarp();
            if (mt >= n_mt) continue;                        // rank 1's copy of the odd last m-tile: nothing to store
            // ---- epilogue from the fragments: rows r0, r0 + 8; columns 8 i + 2 (l % 4) + {0, 1} (registers 4 i + 2 h + j;
            // the sigma^2 partner of a main column NT / 2 registers later).  The two lanes l, l ^ 1 share the 4-channel
            // Philox groups of both rows: each draws one and hands over half of it.
            const int r_top = 64 * wg + 16 * (wt >> 5) + (lane >> 2);
            const int m_a = mt * 128 + r_top, m_b = m_a + 8;
            const bool odd = (lane & 1) != 0;
            const int m_own = odd ? m_b : m_a;
            size_t orow[2];
            bool ok[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = h ? m_b : m_a;
                ok[h] = m < p.M;
                const int b = ok[h] ? m / ohw : 0, pix = ok[h] ? m - b * ohw : 0;
                orow[h] = (size_t)b * p.Cout * ohw + pix;
            }
            float* const out = EPI != 2 ? p.y_noisy : p.y;
            const int n_base = nt * NT;
#pragma unroll
            for (int i = 0; i < NT / 8; ++i) {
                const int n = n_base + 8 * i + 2 * (lane & 3);        // column of register 4 i (+1: next column)
                float z[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
                if (EPI == 1) {
                    float zz[4];
                    nn_normal4(rs, (uint64_t)m_own * ngrp + (uint64_t)(n >> 2), zz);
                    // even lane keeps z[0..1] of row a, gets z[0..1] of row b; odd lane keeps z[2..3] of row b, gets those of row a
                    const float o0 = __shfl_xor_sync(0xffffffffu, odd ? zz[0] : zz[2], 1);
                    const float o1 = __shfl_xor_sync(0xffffffffu, odd ? zz[1] : zz[3], 1);
                    if (odd) { z[0][0] = o0; z[0][1] = o1; z[1][0] = zz[2]; z[1][1] = zz[3]; }
                    else { z[0][0] = zz[0]; z[0][1] = zz[1]; z[1][0] = o0; z[1][1] = o1; }
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!ok[h]) continue;
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        if (n + j >= p.Cout) continue;
                        const size_t o = orow[h] + (size_t)(n + j) * ohw;
                        const float yv = acc[4 * i + 2 * h + j] * y_scale;
                        if (EPI == 2) {
                            out[o] = yv;
                        } else {
                            const float zv = EPI == 3 ? __ldg(p.z_inject + o) : z[h][j];
                            out[o] = __fadd_rn(yv, __fmul_rn(zv, nn_sigma(coef, acc[N / 4 + 4 * i + 2 * h + j] * s_scale)));
                        }
                    }
                }
            }
        }
        if (fail) nn_pipeline_abort(p.err_flag, fail);
    }
    cluster_sync();                                  // neither CTA exits while its peer can still write to it or arrive on it
}

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const int*,
                                   const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeIm2colFn get_encode_im2col() {
    static EncodeIm2colFn fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeIm2colFn)f;
    }
    return fn;
}

int encode_map(CUtensorMap* map, const TmaConvCall& c, int box_c) {
    EncodeIm2colFn enc = get_encode_im2col();
    if (!enc) return nn_fail("nn_conv_tma: cuTensorMapEncodeIm2col is not available%s", "");
    const cuuint64_t Cp = (cuuint64_t)c.pl.Cp;
    cuuint64_t dims[4] = {Cp, (cuuint64_t)c.W, (cuuint64_t)c.H, (cuuint64_t)c.B};
    cuuint64_t strides[3] = {Cp * 2, (cuuint64_t)c.W * Cp * 2, (cuuint64_t)c.H * c.W * Cp * 2};
    int lower[2] = {-c.pad, -c.pad};
    int upper[2] = {c.pad - (c.KW - 1), c.pad - (c.KH - 1)};
    cuuint32_t estr[4] = {1, (cuuint32_t)c.stride, (cuuint32_t)c.stride, 1};
    const CUtensorMapSwizzle sw = box_c == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (box_c == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(c.xp), dims, strides, lower, upper, (cuuint32_t)box_c, 128,
                           estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return nn_fail("nn_conv_tma: cuTensorMapEncodeIm2col failed%s (CUresult %lld)", "", (long long)r);
    // (as CUTLASS does for drivers <= 13.1: small tensors must not carry bit 21 of descriptor word 1)
    int drv = 0;
    cudaDriverGetVersion(&drv);
    if (drv <= 13010 && (size_t)c.B * c.H * c.W * Cp * 2 < 131072) reinterpret_cast<uint64_t*>(map)[1] &= ~(1ull << 21);
    return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_tiled() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)f;
    }
    return fn;
}

// the pre-swizzled weight image viewed as rows of `row_elems` bf16: a box = the n_half rows of one chunk of one CTA rank
int encode_weight_map(CUtensorMap* map, const void* wp, size_t wp_bytes, int row_elems, int box_rows) {
    EncodeTiledFn enc = get_encode_tiled();
    if (!enc) return nn_fail("nn_conv_tma: cuTensorMapEncodeTiled is not available%s", "");
    cuuint64_t dims[2] = {(cuuint64_t)row_elems, (cuuint64_t)(wp_bytes / ((size_t)row_elems * 2))};
    cuuint64_t strides[1] = {(cuuint64_t)row_elems * 2};
    cuuint32_t box[2] = {(cuuint32_t)row_elems, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(wp), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return nn_fail("nn_conv_tma: cuTensorMapEncodeTiled failed%s (CUresult %lld)", "", (long long)r);
    return 0;
}

int g_tma_enable = 1;

typedef void (*TmaConvKernel)(const TmaConvP);

// k_conv_tma<EPI, NT> for NT = nt: every n-tile width a plan can produce (multiples of 8 up to NMAX)
template <int EPI, int NT, int NMAX>
TmaConvKernel tma_conv_kernel(int nt) {
    if (nt == NT) return k_conv_tma<EPI, NT>;
    if constexpr (NT + 8 <= NMAX) return tma_conv_kernel<EPI, NT + 8, NMAX>(nt);
    else return nullptr;
}

// once per (device, kernel): the shared-memory opt-in; once per (device, shared-memory size): the number of co-resident
// clusters (an occupancy query of one kernel stands for all: same block size, one CTA per SM whatever the width)
template <typename Kernel>
int tma_conv_prepare(Kernel kern, int device, const cudaLaunchConfig_t& cfg, int* n_cl) {
    struct Seen { int device; Kernel kern; };
    struct Occ { int device; size_t smem; int clusters; };
    static Seen seen[256];
    static Occ occ[32];
    static int n_seen = 0, n_occ = 0;
    bool done = false;
    for (int i = 0; i < n_seen && !done; ++i) done = seen[i].device == device && seen[i].kern == kern;
    if (!done) {
        NN_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        if (n_seen < 256) seen[n_seen++] = {device, kern};
    }
    for (int i = 0; i < n_occ; ++i)
        if (occ[i].device == device && occ[i].smem == cfg.dynamicSmemBytes) { *n_cl = occ[i].clusters; return 0; }
    cudaLaunchConfig_t q = cfg;
    q.gridDim = dim3(2 * nn_num_sms(device));
    int n = 0;
    NN_CUDA_OK(cudaOccupancyMaxActiveClusters(&n, kern, &q));
    if (n < 1) return nn_fail("nn_conv_tma: no cluster of two CTAs fits on the device%s", "");
    if (n_occ < 32) occ[n_occ++] = {device, cfg.dynamicSmemBytes, n};
    *n_cl = n;
    return 0;
}

}  // namespace

extern "C" int nn_debug_tma_enable(int enable) {
    const int prev = g_tma_enable;
    if (enable >= 0) g_tma_enable = enable;
    return prev;
}

static inline int tc_pad_to(int v, int a) { return (v + a - 1) / a * a; }

bool nn_tma_make_plan(int Cin_k, int KH, int KW, int stride, int pad, int n_out, bool has_sigma, int OH, int OW, TmaPlan* out) {
    if (!g_tma_enable) return false;
    if (KH != KW || stride < 1 || stride > 8 || pad < 0 || pad > 127 || (KH - 1) > 127 + pad || KH > 200) return false;
    if (OH * OW <= 1) return false;                 // linear layers: the split-K path of the tiled kernel
    TmaPlan pl;
    memset(&pl, 0, sizeof(pl));
    pl.Cp = tc_pad_to(Cin_k, 8);
    if (pl.Cp <= 8) return false;                   // narrow inputs: the shift kernels
    pl.taps = KH * KW;
    pl.n_c64 = pl.Cp / 64;
    const int rem = pl.Cp - 64 * pl.n_c64;
    pl.tail_w = rem == 0 ? 0 : (rem <= 16 ? 16 : (rem <= 32 ? 32 : 64));
    pl.nc = pl.n_c64 + (pl.tail_w ? 1 : 0);
    pl.wt = 64 * pl.n_c64 + pl.tail_w;
    pl.gpt = (pl.nc + 1) / 2;
    pl.n_groups = pl.taps * pl.gpt;
    const int max_nt = has_sigma ? 120 : 256;
    pl.n_tiles = (n_out + max_nt - 1) / max_nt;
    pl.n_t = tc_pad_to((n_out + pl.n_tiles - 1) / pl.n_tiles, 8);
    pl.n_tiles = (n_out + pl.n_t - 1) / pl.n_t;
    pl.main_col = 0;
    pl.sig_col = has_sigma ? pl.n_t : -1;
    pl.n_mma = tc_pad_to(has_sigma ? 2 * pl.n_t : pl.n_t, 16);
    if (pl.n_mma < 32) pl.n_mma = 32;
    if (pl.n_mma > 256) return false;
    pl.n_half = pl.n_mma / 2;
    if (pl.n_t > (has_sigma ? 120 : 256)) return false;     // register accumulators of the MMA warpgroups
    int gw = 0;                                     // widest group of a tap (channels)
    for (int gi = 0; gi < pl.gpt; ++gi) {
        const int ca = 2 * gi, cb = 2 * gi + 1;
        const int wa = ca < pl.n_c64 ? 64 : pl.tail_w, wb = cb < pl.nc ? (cb < pl.n_c64 ? 64 : pl.tail_w) : 0;
        if (wa + wb > gw) gw = wa + wb;
    }
    pl.a_stage = tc_pad_to(256 * gw, 1024);
    pl.b_stage = tc_pad_to(pl.n_mma * 2 * gw, 1024);
    const int budget = 222 * 1024 - 2048;
    pl.stages = budget / (pl.a_stage + pl.b_stage);
    if (pl.stages > TC_MAX_STAGES) pl.stages = TC_MAX_STAGES;
    if (pl.stages < 2) return false;
    pl.n_prod = 2;          // two producer warps (<= stages: a producer may run at most one ring revolution ahead)
    pl.threads = (8 + pl.n_prod) * 32;
    pl.tap_bytes = 2 * pl.n_half * 2 * pl.wt;
    pl.smem_bytes = 1024 + (size_t)pl.stages * (pl.a_stage + pl.b_stage) + 16 * TC_MAX_STAGES + 64;
    pl.wp_bytes = (size_t)pl.n_tiles * pl.taps * pl.tap_bytes;
    if (out) *out = pl;
    return true;
}

int nn_tma_conv_launch(const TmaConvCall& c, int device, cudaStream_t st) {
    const TmaPlan& pl = c.pl;
    TmaConvP p;
    memset(&p, 0, sizeof(p));
    if (pl.n_c64 > 0) { if (int e = encode_map(&p.map64, c, 64)) return e; }
    if (pl.tail_w > 0) { if (int e = encode_map(&p.map_tail, c, pl.tail_w)) return e; }
    if (pl.n_c64 == 0) p.map64 = p.map_tail;
    if (pl.tail_w == 0) p.map_tail = p.map64;
    if (((uintptr_t)c.wp & 15) != 0) return nn_fail("nn_conv_tma: the weight image must be 16-byte aligned%s", "");
    if (pl.n_c64 > 0) { if (int e = encode_weight_map(&p.mapb64, c.wp, pl.wp_bytes, 64, pl.n_half)) return e; }
    if (pl.tail_w > 0) { if (int e = encode_weight_map(&p.mapb_tail, c.wp, pl.wp_bytes, pl.tail_w, pl.n_half)) return e; }
    if (pl.n_c64 == 0) p.mapb64 = p.mapb_tail;
    if (pl.tail_w == 0) p.mapb_tail = p.mapb64;
    p.M = c.B * c.OH * c.OW; p.OH = c.OH; p.OW = c.OW; p.Cout = c.Cout; p.stride = c.stride; p.pad = c.pad; p.KW = c.KW; p.taps = pl.taps;
    p.n_c64 = pl.n_c64; p.tail_w = pl.tail_w; p.nc = pl.nc; p.gpt = pl.gpt; p.n_groups = pl.n_groups;
    p.n_mma = pl.n_mma; p.n_half = pl.n_half; p.n_tiles = pl.n_tiles;
    p.stages = pl.stages; p.a_stage = pl.a_stage; p.b_stage = pl.b_stage; p.n_prod = pl.n_prod; p.tap_bytes = pl.tap_bytes;
    p.y_scale = c.y_scale; p.s_scale = c.s_scale; p.y = c.y; p.y_noisy = c.y_noisy;
    p.current = c.current; p.scale_dev = c.scale_dev; p.z_inject = c.z_inject; p.rng = c.rng; p.err_flag = c.err_flag;
    const bool noise = c.noise_mode != NN_NOISE_NONE;
    const int epi = noise ? (c.z_inject ? 3 : 1) : 2;
    const TmaConvKernel kern = epi == 3 ? tma_conv_kernel<3, 8, 120>(pl.n_t) : epi == 1 ? tma_conv_kernel<1, 8, 120>(pl.n_t)
                                                                             : tma_conv_kernel<2, 8, 256>(pl.n_t);
    if (!kern) return nn_fail("nn_conv_tma: no kernel for an n-tile of%s %lld columns", "", (long long)pl.n_t);
    // persistent clusters of two CTAs (one CTA per SM): as many as fit at once, at most one per pair of m-tiles and n-tile
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.blockDim = dim3(pl.threads);
    cfg.dynamicSmemBytes = pl.smem_bytes;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n_cl = 0;
    if (int e = tma_conv_prepare(kern, device, cfg, &n_cl)) return e;
    const int pairs = ((p.M + 255) / 256) * pl.n_tiles;
    if (n_cl > pairs) n_cl = pairs;
    cfg.gridDim = dim3(2 * n_cl);
    if (c.ev0) cudaEventRecord((cudaEvent_t)c.ev0, st);          // measurement hook: brackets the kernel, not the host-side descriptor encoding
    NN_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, p));
    if (c.ev1) cudaEventRecord((cudaEvent_t)c.ev1, st);
    NN_LAUNCH_OK();
    return 0;
}

// Tiled 2-D map of a row-major bf16 matrix [rows][cols] (row pitch in bytes, a multiple of 16), box = 64 columns x 128 rows,
// SWIZZLE_128B: the K-major A tile of the gathered kernels when the layer is linear (out-of-range rows / columns read as 0).
int nn_tma_encode_rows(void* map_out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t pitch_bytes) {
    EncodeTiledFn enc = get_encode_tiled();
    if (!enc) return nn_fail("nn_conv_tma: cuTensorMapEncodeTiled is not available%s", "");
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)pitch_bytes};
    cuuint32_t box[2] = {64, 128};
    cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(reinterpret_cast<CUtensorMap*>(map_out), CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box,
                           estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return nn_fail("nn_conv_tma: cuTensorMapEncodeTiled (matrix rows) failed%s (CUresult %lld)", "", (long long)r);
    return 0;
}

// ================================================================== dgrad on a resident row-plane image of grad_output
//   gx[b, n, oh, ow] = sum_{tap, c} gyp[b, oh + kh - pad', ow + kw - pad', c] * Wp[n, tap, c]       (pad' = K - 1 - pad)
// k_conv_tma loads one im2col tile per (128-pixel tile, tap): 25 x 32 KB per tile for conv2's dgrad, ~600 MB of L2 -> SM
// traffic per step to read a 12 MB grad_output.  k_dgrad_planes loads each image ONCE and takes all taps from it:
// * A operand: the image zero-padded by pad' on every side (GH x GW pixels, 18 x 18 for conv2) as row planes -- plane q
//   holds channels 8 q .. 8 q + 7, one 16-byte row per pixel (the SWIZZLE_NONE K-major core-matrix row).  One tiled
//   tensor-map copy per plane (box {8, GW, GH, 1} from (8 q, -pad', -pad', b)) lands it, the TMA unit zero-filling the
//   halo.  Outputs live on a virtual grid r = oh * GW + ow (OH x GW rows, 4 m64 blocks); tap (kh, kw) is the same planes
//   read kh * GW + kw rows later: the descriptor's start address moves, SBO = 8 rows (128 B), LBO = the plane stride.
//   Planes past the channels and rows past the grid that the last block's taps reach are zeroed once at kernel start.
// * B operand: the NN_PACK_TMA dgrad image and weight maps of k_conv_tma, one ring stage per tap, each CTA of a pair
//   multicasting one row half.
// * Work item: one image per CTA, clusters of two CTAs on images 2 i, 2 i + 1 in lockstep (an odd last image: rank 1
//   reloads its partner's and stores nothing).  k16 step j of a tap is channels 16 j .. 16 j + 15 and the taps run in
//   k_conv_tma's order, so every output receives the same products in the same k16 groups in the same order: gx is
//   bit-identical to k_conv_tma<2, NT>'s.
// * Warp roles: warps 0-7 two MMA warpgroups (m64 blocks 2 g, 2 g + 1 each; epilogue from the fragments), warp 8 the
//   weight ring, warp 9 the A image (refilled once both warpgroups' chains over the previous image have completed, so
//   it lands during their epilogue; one full barrier per plane pair lets the first tap start on the first planes).
namespace {

constexpr int DP_MAX_STAGES = 8;
constexpr int DP_MAX_PAIRS = 8;              // 16 planes: up to 128 channels

struct DgPlanesP {
    CUtensorMap map_gy;                      // tiled {Cp, W, H, B} over grad_output, box {8, GW, GH, 1}: one plane of one image
    CUtensorMap mapb64, mapb_tail;           // the weight image as in k_conv_tma
    int B, OH, OW, Cout, pad, KW, taps, GW, GH;
    int n_c64, tail_w, nc, n_mma, n_half, tap_bytes;
    int n_load, n_pairs, plane_bytes, stages, b_stage;
    float y_scale;
    float* gx;
    int* err_flag;
};

// the wgmmas of one tap over m64 blocks 0 and 1 of the warpgroup (block 1: 64 rows = 64 descriptor units later): k16 step k
// reads plane pair k (`pstep` units apart) and weight columns 16 k .. of chunk a, then of chunk b; committed as one group,
// returning when the previous tap's group has completed.  scale_d of the first step: 0 starts the accumulators of an image.
template <int N, int KA, int KB>
__device__ __forceinline__ void planes_tap_mma(float* acc0, float* acc1, uint64_t ad, uint64_t pstep, uint64_t bd_a, uint64_t bd_b, int acc_in) {
    wg_fence();
#pragma unroll
    for (int k = 0; k < KA + KB; ++k) {
        const uint64_t a = ad + (uint64_t)k * pstep, b = k < KA ? bd_a + 2 * k : bd_b + 2 * (k - KA);
        wgmma_c<N, 0, 0>(acc0, a, b, k == 0 ? acc_in : 1);
        wgmma_c<N, 0, 0>(acc1, a + 64, b, k == 0 ? acc_in : 1);
    }
    wg_commit();
    wg_wait_1();
}

template <int NT>
__global__ void __launch_bounds__((8 + 2) * 32, 1)
k_dgrad_planes(const __grid_constant__ DgPlanesP p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int S = p.stages;
    const uint32_t a_base = base + (uint32_t)S * (uint32_t)p.b_stage;
    const uint32_t a_bytes = (uint32_t)(2 * p.n_pairs * p.plane_bytes);
    const uint32_t bar_base = a_base + a_bytes;
    const uint32_t full_bar = bar_base, empty_bar = bar_base + 8u * DP_MAX_STAGES;
    const uint32_t a_full = bar_base + 16u * DP_MAX_STAGES, a_empty = a_full + 8u * DP_MAX_PAIRS;

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const uint32_t rank = cluster_ctarank(), peer = rank ^ 1u;
    const int pairs = (p.B + 1) >> 1;
    const int cl0 = blockIdx.x >> 1, n_cl = gridDim.x >> 1;
    // chunk widths of a tap (one ring stage: k_conv_tma's single group of <= 128 channels)
    const int wa = p.n_c64 > 0 ? 64 : p.tail_w;
    const int wb = p.nc > 1 ? (p.n_c64 > 1 ? 64 : p.tail_w) : 0;

    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full_bar + 8 * s, 1);          // the weight producer's arrive.expect_tx (both row halves)
            mbar_init(empty_bar + 8 * s, 4);         // both MMA warpgroups of both CTAs have read the stage
        }
        for (int j = 0; j < p.n_pairs; ++j) mbar_init(a_full + 8 * j, 1);
        mbar_init(a_empty, 2);                       // both MMA warpgroups of this CTA are done with the image
        fence_mbar_init();
        tma_prefetch_desc(&p.map_gy);
        tma_prefetch_desc(&p.mapb64);
        tma_prefetch_desc(&p.mapb_tail);
    }
    {   // zeros the copies never write: rows past the padded grid of the loaded planes, and whole planes past the channels
        const int grid_bytes = p.GH * p.GW * 16;
        uint8_t* const a_gen = smem_raw + (a_base - smem_u32(smem_raw));
        const int tail_bytes = p.plane_bytes - grid_bytes;
        const int n_tail = p.n_load * (tail_bytes >> 4), n_rest = (2 * p.n_pairs - p.n_load) * (p.plane_bytes >> 4);
        for (int i = tid; i < n_tail + n_rest; i += blockDim.x) {
            const int off = i < n_tail ? (i / (tail_bytes >> 4)) * p.plane_bytes + grid_bytes + 16 * (i % (tail_bytes >> 4))
                                       : p.n_load * p.plane_bytes + 16 * (i - n_tail);
            *reinterpret_cast<uint4*>(a_gen + off) = make_uint4(0u, 0u, 0u, 0u);
        }
        fence_proxy_async();                         // visible to the wgmmas (async proxy)
    }
    cluster_sync();                                  // barriers initialised and zeros written before any copy, arrival or wgmma

    if (warp == 8) {
        // ---------------------------------------------------------------- weight ring: one stage per tap
        int s = 0, fail = 0;
        uint32_t eph = 1u;
        const uint32_t half_bytes = (uint32_t)(p.n_half * 2 * (wa + wb));
        const int h = (int)rank;                             // this CTA's row half goes to both CTAs of the pair
        for (int pi = cl0; pi < pairs && !fail; pi += n_cl) {
            for (int t = 0; t < p.taps; ++t) {
                if (!mbar_wait_backoff(empty_bar + 8 * s, eph)) { fail = 601; break; }
                if (elect_one_sync()) {
                    const uint32_t bar = full_bar + 8 * s, b_dst = base + (uint32_t)s * (uint32_t)p.b_stage;
                    mbar_arrive_expect_tx(bar, 2u * half_bytes);
                    const long long boff = (long long)t * p.tap_bytes + (long long)h * half_bytes;
                    const uint32_t da = b_dst + (uint32_t)(h * p.n_half * 2 * wa);
                    if (wa == 64) tma_tile_2d_mc(da, &p.mapb64, bar, 0, (int)(boff >> 7), 0x3);
                    else tma_tile_2d_mc(da, &p.mapb_tail, bar, 0, (int)(boff / (2 * wa)), 0x3);
                    if (wb) {
                        const long long boff2 = boff + (long long)p.n_half * 2 * wa;
                        const uint32_t db = b_dst + (uint32_t)(p.n_mma * 2 * wa + h * p.n_half * 2 * wb);
                        if (wb == 64) tma_tile_2d_mc(db, &p.mapb64, bar, 0, (int)(boff2 >> 7), 0x3);
                        else tma_tile_2d_mc(db, &p.mapb_tail, bar, 0, (int)(boff2 / (2 * wb)), 0x3);
                    }
                }
                __syncwarp();
                if (++s == S) { s = 0; eph ^= 1u; }
            }
        }
        if (fail) nn_pipeline_abort(p.err_flag, fail);
        __syncwarp();
    } else if (warp == 9) {
        // ---------------------------------------------------------------- A image: one copy per plane, a barrier per pair
        int fail = 0;
        uint32_t eph = 1u;
        const uint32_t box_bytes = (uint32_t)(p.GH * p.GW * 16);
        for (int pi = cl0; pi < pairs; pi += n_cl) {
            const int b = min(2 * pi + (int)rank, p.B - 1);
            if (!mbar_wait_backoff(a_empty, eph)) { fail = 602; break; }
            eph ^= 1u;
            if (elect_one_sync()) {
                for (int j = 0; j < p.n_pairs; ++j) {
                    const int nq = max(0, min(2, p.n_load - 2 * j));
                    mbar_arrive_expect_tx(a_full + 8 * j, (uint32_t)nq * box_bytes);
                    for (int q = 2 * j; q < 2 * j + nq; ++q)
                        tma_tile_4d(a_base + (uint32_t)(q * p.plane_bytes), &p.map_gy, a_full + 8 * j, 8 * q, -p.pad, -p.pad, b);
                }
            }
            __syncwarp();
        }
        if (fail) nn_pipeline_abort(p.err_flag, fail);
        __syncwarp();
    } else if (warp < 8) {
        // ---------------------------------------------------------------- MMA warpgroups + epilogue
        const int wg = warp >> 2, wt = tid & 127;
        const bool releaser = (warp & 3) == 0;
        const int kt = p.tail_w >> 4;
        const int shape = 8 * (wa == 64 ? 4 : kt) + (wb == 64 ? 4 : (wb ? kt : 0));
        const uint32_t plane_units = (uint32_t)p.plane_bytes >> 4;
        const uint64_t pstep = 2ull * plane_units;
        const int ohw = p.OH * p.OW;
        const float y_scale = p.y_scale;
        int s = 0, prev = 0, fail = 0;
        uint32_t fph = 0u, aph = 0u;
        for (int pi = cl0; pi < pairs && !fail; pi += n_cl) {
            const int b = 2 * pi + (int)rank;
            float acc[2][NT / 2];
            int kh = 0, kw = 0;
            for (int t = 0; t < p.taps; ++t) {
                if (!mbar_wait(full_bar + 8 * s, fph)) { fail = 603; break; }
                const uint32_t b_s = base + (uint32_t)s * (uint32_t)p.b_stage;
                const uint64_t bd_a = gmma_desc_kmajor(b_s, 2u * (uint32_t)wa);
                const uint64_t bd_b = wb ? gmma_desc_kmajor(b_s + (uint32_t)(p.n_mma * 2 * wa), 2u * (uint32_t)wb) : 0;
                const uint64_t ad = gmma_desc_none(a_base + 16u * (uint32_t)(128 * wg + kh * p.GW + kw), plane_units, 8u);
                if (t == 0) {                                // the image (this item's A phase)
                    for (int j = 0; j < p.n_pairs && !fail; ++j)
                        if (!mbar_wait(a_full + 8 * j, aph)) fail = 604;
                    if (fail) break;
                }
                const int acc_in = t != 0 ? 1 : 0;
                // one straight-line sequence per tap shape, as in k_conv_tma
                switch (shape) {
                    case 8 * 4 + 4: planes_tap_mma<NT, 4, 4>(acc[0], acc[1], ad, pstep, bd_a, bd_b, acc_in); break;
                    case 8 * 4 + 2: planes_tap_mma<NT, 4, 2>(acc[0], acc[1], ad, pstep, bd_a, bd_b, acc_in); break;
                    case 8 * 4 + 1: planes_tap_mma<NT, 4, 1>(acc[0], acc[1], ad, pstep, bd_a, bd_b, acc_in); break;
                    case 8 * 4: planes_tap_mma<NT, 4, 0>(acc[0], acc[1], ad, pstep, bd_a, bd_b, acc_in); break;
                    case 8 * 2: planes_tap_mma<NT, 2, 0>(acc[0], acc[1], ad, pstep, bd_a, bd_b, acc_in); break;
                    default: planes_tap_mma<NT, 1, 0>(acc[0], acc[1], ad, pstep, bd_a, bd_b, acc_in); break;
                }
                if (t != 0 && releaser && elect_one_sync()) {      // the previous tap's weights may be refilled
                    mbar_arrive(empty_bar + 8 * prev);
                    mbar_arrive_cluster(cluster_map(empty_bar + 8 * prev, peer));
                }
                __syncwarp();
                prev = s;
                if (++kw == p.KW) { kw = 0; ++kh; }
                if (++s == S) { s = 0; fph ^= 1u; }
            }
            if (fail) break;
            wg_wait_all();
            wg_fence_regs<NT / 2>(acc[0]);
            wg_fence_regs<NT / 2>(acc[1]);
            if (releaser && elect_one_sync()) {
                mbar_arrive(empty_bar + 8 * prev);
                mbar_arrive_cluster(cluster_map(empty_bar + 8 * prev, peer));
                mbar_arrive(a_empty);                        // the next image may land while this one's outputs are stored
            }
            __syncwarp();
            aph ^= 1u;
            if (b >= p.B) continue;                          // rank 1's copy of an odd last image: nothing to store
            // ---- epilogue from the fragments: virtual row r -> (oh, ow) = (r / GW, r % GW), real where ow < OW, oh < OH
            float* const out = p.gx + (size_t)b * p.Cout * ohw;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = 128 * wg + 64 * i + 16 * (wt >> 5) + (lane >> 2) + 8 * h;
                    const int oh = r / p.GW, ow = r - oh * p.GW;
                    if (oh >= p.OH || ow >= p.OW) continue;
                    float* const o = out + oh * p.OW + ow;
#pragma unroll
                    for (int ii = 0; ii < NT / 8; ++ii) {
#pragma unroll
                        for (int j = 0; j < 2; ++j) {
                            const int n = 8 * ii + 2 * (lane & 3) + j;
                            if (n < p.Cout) o[(size_t)n * ohw] = acc[i][4 * ii + 2 * h + j] * y_scale;
                        }
                    }
                }
            }
        }
        if (fail) nn_pipeline_abort(p.err_flag, fail);
    }
    cluster_sync();                                  // neither CTA exits while its peer can still write to it or arrive on it
}

typedef void (*DgPlanesKernel)(const DgPlanesP);

// k_dgrad_planes<NT> for NT = nt (multiples of 8 up to NMAX)
template <int NT, int NMAX>
DgPlanesKernel dgrad_planes_kernel(int nt) {
    if (nt == NT) return k_dgrad_planes<NT>;
    if constexpr (NT + 8 <= NMAX) return dgrad_planes_kernel<NT + 8, NMAX>(nt);
    else return nullptr;
}

}  // namespace

bool nn_dgrad_planes_plan(const nn_conv_geom& g, DgPlanesPlan* out) {
    if (g.stride != 1 || g.KH != g.KW || g.pad > g.KH - 1 || g.Cout > 128) return false;
    DgPlanesPlan d;
    memset(&d, 0, sizeof(d));
    d.pad = g.KH - 1 - g.pad;
    if (!nn_tma_make_plan(g.Cout, g.KH, g.KW, 1, d.pad, g.Cin, false, g.H, g.W, &d.tp)) return false;
    const TmaPlan& tp = d.tp;
    if (tp.n_tiles != 1 || tp.n_t > 120 || tp.gpt != 1) return false;
    int OH, OW;                                      // grad_output
    nn_out_hw(g, OH, OW);
    d.GW = OW + 2 * d.pad;
    d.GH = OH + 2 * d.pad;
    if (g.H * d.GW > 256 || d.GH > 256) return false;       // four m64 blocks of virtual rows; one tensor-map box per plane
    const int reach = 256 + (g.KH - 1) * (d.GW + 1);        // rows the last block's last tap reads
    d.rows = tc_pad_to(d.GH * d.GW > reach ? d.GH * d.GW : reach, 8);
    d.n_planes = tp.wt / 8;
    d.n_load = tp.Cp / 8;
    d.plane_bytes = d.rows * 16;
    const int a_bytes = d.n_planes * d.plane_bytes;
    d.stages = (222 * 1024 - 2048 - a_bytes) / tp.b_stage;
    if (d.stages > DP_MAX_STAGES) d.stages = DP_MAX_STAGES;
    if (d.stages < 2) return false;
    d.smem_bytes = 1024 + (size_t)d.stages * tp.b_stage + a_bytes + 8 * (2 * DP_MAX_STAGES + DP_MAX_PAIRS + 1);
    if (out) *out = d;
    return true;
}

int nn_dgrad_planes_launch(const nn_conv_dgrad_args& a, const DgPlanesPlan& d, int device, cudaStream_t st) {
    const TmaPlan& pl = d.tp;
    const nn_conv_geom& g = a.g;
    int OH, OW;
    nn_out_hw(g, OH, OW);
    DgPlanesP p;
    memset(&p, 0, sizeof(p));
    {   // grad_output [B][OH][OW][Cp] bf16: boxes of one plane (8 channels) of the zero-padded GH x GW grid of one image
        EncodeTiledFn enc = get_encode_tiled();
        if (!enc) return nn_fail("nn_conv_tma: cuTensorMapEncodeTiled is not available%s", "");
        const cuuint64_t Cp = (cuuint64_t)pl.Cp;
        cuuint64_t dims[4] = {Cp, (cuuint64_t)OW, (cuuint64_t)OH, (cuuint64_t)g.B};
        cuuint64_t strides[3] = {Cp * 2, (cuuint64_t)OW * Cp * 2, (cuuint64_t)OH * OW * Cp * 2};
        cuuint32_t box[4] = {8, (cuuint32_t)d.GW, (cuuint32_t)d.GH, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        const CUresult r = enc(&p.map_gy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(a.gy_packed), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return nn_fail("nn_conv_dgrad_planes: cuTensorMapEncodeTiled (grad_output planes) failed%s (CUresult %lld)", "",
                                              (long long)r);
    }
    if (((uintptr_t)a.w_packed & 15) != 0) return nn_fail("nn_conv_dgrad_planes: the weight image must be 16-byte aligned%s", "");
    if (pl.n_c64 > 0) { if (int e = encode_weight_map(&p.mapb64, a.w_packed, pl.wp_bytes, 64, pl.n_half)) return e; }
    if (pl.tail_w > 0) { if (int e = encode_weight_map(&p.mapb_tail, a.w_packed, pl.wp_bytes, pl.tail_w, pl.n_half)) return e; }
    if (pl.n_c64 == 0) p.mapb64 = p.mapb_tail;
    if (pl.tail_w == 0) p.mapb_tail = p.mapb64;
    p.B = g.B; p.OH = g.H; p.OW = g.W; p.Cout = g.Cin; p.pad = d.pad; p.KW = g.KW; p.taps = pl.taps; p.GW = d.GW; p.GH = d.GH;
    p.n_c64 = pl.n_c64; p.tail_w = pl.tail_w; p.nc = pl.nc; p.n_mma = pl.n_mma; p.n_half = pl.n_half; p.tap_bytes = pl.tap_bytes;
    p.n_load = d.n_load; p.n_pairs = d.n_planes / 2; p.plane_bytes = d.plane_bytes; p.stages = d.stages; p.b_stage = pl.b_stage;
    p.y_scale = a.w_code_scale > 0.f ? a.w_code_scale : 1.f;
    p.gx = a.gx; p.err_flag = nn_umma_err_flag(device);
    const DgPlanesKernel kern = dgrad_planes_kernel<8, 120>(pl.n_t);
    if (!kern) return nn_fail("nn_conv_dgrad_planes: no kernel for an n-tile of%s %lld columns", "", (long long)pl.n_t);
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.blockDim = dim3((8 + 2) * 32);
    cfg.dynamicSmemBytes = d.smem_bytes;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n_cl = 0;
    if (int e = tma_conv_prepare(kern, device, cfg, &n_cl)) return e;
    const int pairs = (g.B + 1) / 2;
    if (n_cl > pairs) n_cl = pairs;
    cfg.gridDim = dim3(2 * n_cl);
    NN_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, p));
    NN_LAUNCH_OK();
    return 0;
}

// ================================================================== weight gradient with TMA-staged operands
//   D[n, (tap, c)] = sum over output pixels m of gy[m, n] * x[pixel(m) + tap, c]
// Both operands are NHWC bf16, i.e. contiguous along their M / N dimension: they are staged as MN-major SWIZZLE_128B atoms
// [64 reduction rows (pixels)][128 B = 64 channels] -- exactly what ONE tensor-map copy delivers: a tiled 2-D box of
// grad_output (64 pixels x 64 output channels) and an im2col box of the layer input (64 pixels x 64 channels of one tap).
// A CTA owns up to four (tap, 64-channel chunk) atoms = 256 accumulator columns and a share of the pixels; per 64-pixel
// k-block six copies (48 KB) replace the 3072 cp.async gathers of the thread-gathered kernel.  An 8-channel remainder of
// each tap (the 65 -> 72 channels of NoisyNet's conv2) is a second launch of the same kernel (TAIL): its B operand is a slab
// of one {8 channels, 64 pixels} im2col copy per tap (SWIZZLE_NONE MN-major core matrices, taps 1 KB apart), 8 columns
// per tap.  Two MMA warpgroups (64 output channels each) accumulate in registers and store the partial sums.
namespace {

struct WgTmaP {
    CUtensorMap map_gy;              // tiled {Coutp, Mpix}, box {64, 64}, SWIZZLE_128B
    CUtensorMap map_x;               // im2col {Cp, W, H, B}, box {64 channels, 64 pixels}, SWIZZLE_128B
    CUtensorMap map_xt;              // im2col, box {8 channels, 64 pixels}, SWIZZLE_NONE: the channel remainder of a tap
    int OH, OW, stride, pad, KW, n_c64, n_atoms, Mpix, Cout;
    int taps;
    int num_kb, kb_per_split, stages, cols_pad;
    float* partial;                  // [splits][Cout][cols_pad]
    float* partial_tail;             // [splits][Cout][256]: column tap * 8 + e <-> channel 64 * n_c64 + e
    int* err_flag;
};

constexpr int WT_STAGE = 16384 + 32768;        // A: 2 atoms, B: 4 atoms of 8 KB (or the remainder slab: 1 KB per tap, <= 32 taps)
constexpr int WT_PROD = 4;                     // producer warps (warps 0-7 MMA warpgroups, 8-11 producers)
constexpr int WT_THREADS = (8 + WT_PROD) * 32;

// the MMA warpgroups' k-block loop at a compile-time width N (one wgmma per k16 step); returns a watchdog code or 0
template <int N, bool TAIL>
__device__ __forceinline__ int wgrad_mma_loop(float* acc, int nkb, uint32_t base, uint32_t full_bar, uint32_t empty_bar, int S, int wg,
                                              bool releaser) {
    // A: SWIZZLE_128B MN-major atoms (LBO = atom stride 8192 B, 16 pixels = 2048 B); B: main -- the same; remainder slab --
    // LBO = 8-pixel groups 128 B apart, SBO = the taps' slabs 1 KB apart, 16 pixels = 256 B
    const uint64_t da = gmma_desc(0u, 8192u >> 4, 1024u >> 4, 1u);
    const uint64_t db = TAIL ? gmma_desc(0u, 8u, 64u, 0u) : da;
    constexpr uint32_t k_step_b = TAIL ? 16u : 128u;
    int s = 0, prev = 0;
    uint32_t ph = 0u;
    for (int i = 0; i < nkb; ++i) {
        if (!mbar_wait(full_bar + 8 * s, ph)) return 502;
        const uint32_t a_s = (base + (uint32_t)s * WT_STAGE + (uint32_t)wg * 8192u) >> 4, b_s = (base + (uint32_t)s * WT_STAGE + 16384u) >> 4;
        const uint64_t ad = da | (uint64_t)(a_s & 0x3FFFu), bd = db | (uint64_t)(b_s & 0x3FFFu);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_c<N, 1, 1>(acc, ad + 128 * k, bd + k_step_b * k, (i | k) != 0 ? 1 : 0);
        wg_commit();
        wg_wait_1();                     // this k-block's wgmmas stay in flight; the previous block's stage is released
        if (i != 0 && releaser && elect_one_sync()) mbar_arrive(empty_bar + 8 * prev);
        __syncwarp();
        prev = s;
        if (++s == S) { s = 0; ph ^= 1u; }
    }
    wg_wait_all();
    wg_fence_regs<N / 2>(acc);
    if (nkb > 0 && releaser && elect_one_sync()) mbar_arrive(empty_bar + 8 * prev);
    __syncwarp();
    return 0;
}

// TW: the MMA width of the remainder launch (TAIL; 16 * ceil(taps / 2) columns), 0 for the main launch, whose column
// tiles have 1 .. 4 atoms of 64 columns (the last tile of a layer is narrower): one compile-time width per case
template <bool TAIL, int TW>
__global__ void __launch_bounds__(WT_THREADS, 1)
k_wgrad_tma(const __grid_constant__ WgTmaP p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int S = p.stages;
    const uint32_t bar_base = base + (uint32_t)S * WT_STAGE;
    const uint32_t full_bar = bar_base, empty_bar = bar_base + 64u;
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int tile_k = blockIdx.x, tile_n = blockIdx.y, split = blockIdx.z;
    const int kb0 = split * p.kb_per_split, kb1 = min(p.num_kb, kb0 + p.kb_per_split);
    const int nkb = max(0, kb1 - kb0);
    const int atoms = TAIL ? 0 : min(4, p.n_atoms - tile_k * 4);  // (tap, chunk) atoms of this column tile
    const int n_cols = TAIL ? (p.taps * 8 + 15) & ~15 : 64 * atoms;
    if (tid == 0) {
        for (int s = 0; s < S; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 2); }
        fence_mbar_init();
        tma_prefetch_desc(&p.map_gy);
        if (TAIL) tma_prefetch_desc(&p.map_xt);
        else tma_prefetch_desc(&p.map_x);
    }
    __syncthreads();
    int fail = 0;

    if (warp >= 8) {
        // ---- producers: one elected lane per warp issues its share of a stage's copies (an im2col copy occupies its issuing
        // thread for hundreds of cycles, so the copies of a stage go out from several warps); warp 8 also posts the byte count.
        const int pw = warp - 8;
        const int ohw = p.OH * p.OW;
        for (int i = 0; i < nkb; ++i) {
            const int s = i % S;
            if (!mbar_wait_backoff(empty_bar + 8 * s, (((uint32_t)(i / S)) & 1u) ^ 1u)) { fail = 501; break; }
            const int m0 = (kb0 + i) * 64;
            const int b0 = m0 / ohw, r0 = m0 - b0 * ohw, oh0 = r0 / p.OW, ow0 = r0 - oh0 * p.OW;
            const int n_copy = 2 + (TAIL ? p.taps : atoms);
            if (elect_one_sync()) {
                const uint32_t dst = base + (uint32_t)s * WT_STAGE, bar = full_bar + 8 * s;
                if (pw == 0) mbar_arrive_expect_tx(bar, 16384u + (TAIL ? 1024u * (uint32_t)p.taps : 8192u * (uint32_t)atoms));
                for (int j = pw; j < n_copy; j += WT_PROD) {
                    if (j < 2) {
                        tma_tile_2d(dst + 8192u * (uint32_t)j, &p.map_gy, bar, tile_n * 128 + 64 * j, m0);
                    } else if (TAIL) {
                        const int tap = j - 2, kh = tap / p.KW, kw = tap - kh * p.KW;
                        tma_im2col_4d(dst + 16384u + 1024u * (uint32_t)tap, &p.map_xt, bar, 64 * p.n_c64, ow0 * p.stride - p.pad,
                                      oh0 * p.stride - p.pad, b0, (uint16_t)kw, (uint16_t)kh);
                    } else {
                        const int a = j - 2, ga = tile_k * 4 + a, tap = ga / p.n_c64, ch = ga - tap * p.n_c64;
                        const int kh = tap / p.KW, kw = tap - kh * p.KW;
                        tma_im2col_4d(dst + 16384u + 8192u * (uint32_t)a, &p.map_x, bar, 64 * ch, ow0 * p.stride - p.pad, oh0 * p.stride - p.pad, b0,
                                      (uint16_t)kw, (uint16_t)kh);
                    }
                }
            }
            __syncwarp();
        }
    } else {
        // ---- MMA warpgroups: MN-major A and B; warpgroup g owns output channels 64 g .. 64 g + 63 (the second atom of A, + 8 KB).
        const int wg = warp >> 2;
        const bool releaser = (warp & 3) == 0;
        float acc[128];
        if constexpr (TAIL) fail = wgrad_mma_loop<TW, true>(acc, nkb, base, full_bar, empty_bar, S, wg, releaser);
        else if (atoms == 4) fail = wgrad_mma_loop<256, TAIL>(acc, nkb, base, full_bar, empty_bar, S, wg, releaser);
        else if (atoms == 3) fail = wgrad_mma_loop<192, TAIL>(acc, nkb, base, full_bar, empty_bar, S, wg, releaser);
        else if (atoms == 2) fail = wgrad_mma_loop<128, TAIL>(acc, nkb, base, full_bar, empty_bar, S, wg, releaser);
        else fail = wgrad_mma_loop<64, TAIL>(acc, nkb, base, full_bar, empty_bar, S, wg, releaser);
        if (!fail) {
            // ---- epilogue: rows = output channels, columns = (atom, channel) [or (tap, remainder channel)]
            const int wt = tid & 127;
            const int n0 = tile_n * 128 + 64 * wg + 16 * (wt >> 5) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = n0 + 8 * h;
                if (n >= p.Cout) continue;
                float* out = TAIL ? p.partial_tail + ((size_t)split * p.Cout + n) * 256 + c0
                                  : p.partial + ((size_t)split * p.Cout + n) * p.cols_pad + (size_t)tile_k * 256 + c0;
#pragma unroll
                for (int c = 0; c < 4; ++c)
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        if (64 * c + 8 * j < n_cols)
                            *reinterpret_cast<float2*>(out + 64 * c + 8 * j) =
                                nkb > 0 ? make_float2(acc[32 * c + 4 * j + 2 * h], acc[32 * c + 4 * j + 2 * h + 1]) : make_float2(0.f, 0.f);
            }
        }
    }
    if (fail) nn_pipeline_abort(p.err_flag, fail);
}

}  // namespace

bool nn_tma_wgrad_plan(int Cin, int KH, int KW, int stride, int pad, int Cout, int64_t Mpix, int device, TmaWgradPlan* out) {
    if (!g_tma_enable) return false;
    if (KH != KW || stride < 1 || stride > 8 || pad < 0 || pad > 127 || (KH - 1) > 127 + pad) return false;
    TmaWgradPlan w;
    memset(&w, 0, sizeof(w));
    w.Cp = tc_pad_to(Cin, 8);
    w.n_c64 = w.Cp / 64;
    w.tail_w = w.Cp - 64 * w.n_c64;
    if (w.n_c64 == 0) return false;                     // narrow inputs: the shift kernel / the gathered kernel
    // an 8-channel remainder (65 -> 72 channels) is its own column tile of 8 columns per tap; wider ones are one more
    // (zero-filled) 64-channel chunk
    if (w.tail_w > 8 || (w.tail_w == 8 && KH * KW > 31)) { w.n_c64 += 1; w.tail_w = 0; }
    w.stages = 4;
    w.Coutp = tc_pad_to(Cout, 8);
    w.taps = KH * KW;
    w.n_atoms = w.taps * w.n_c64;
    w.tiles_k = (w.n_atoms + 3) / 4;
    w.cols_pad = w.tiles_k * 256;
    w.m_tiles_n = (Cout + 127) / 128;
    w.num_kb = (int)((Mpix + 63) / 64);
    const int tiles = w.tiles_k * w.m_tiles_n;
    int splits = nn_num_sms(device) / tiles;            // one CTA per SM (four 48 KB stages)
    if (splits > w.num_kb) splits = w.num_kb;
    if (splits < 1) splits = 1;
    w.kb_per_split = (w.num_kb + splits - 1) / splits;
    w.splits = (w.num_kb + w.kb_per_split - 1) / w.kb_per_split;
    w.smem_bytes = 1024 + (size_t)w.stages * WT_STAGE + 256;
    w.main_bytes = ((size_t)w.splits * Cout * w.cols_pad * 4 + 1023) / 1024 * 1024;
    w.partial_bytes = w.main_bytes + (w.tail_w ? (size_t)w.splits * Cout * 256 * 4 : 0);
    if (out) *out = w;
    return true;
}

int nn_tma_wgrad_launch(const TmaWgradCall& c, int device, cudaStream_t st) {
    const TmaWgradPlan& w = c.pl;
    WgTmaP p;
    memset(&p, 0, sizeof(p));
    {   // grad_output [Mpix, Coutp] bf16: boxes of 64 pixels x 64 channels
        EncodeTiledFn enc = get_encode_tiled();
        if (!enc) return nn_fail("nn_conv_tma: cuTensorMapEncodeTiled is not available%s", "");
        const cuuint64_t Mpix = (cuuint64_t)c.B * c.OH * c.OW;
        cuuint64_t dims[2] = {(cuuint64_t)w.Coutp, Mpix};
        cuuint64_t strides[1] = {(cuuint64_t)w.Coutp * 2};
        cuuint32_t box[2] = {64, 64};
        cuuint32_t estr[2] = {1, 1};
        const CUresult r = enc(&p.map_gy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(c.gyp), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return nn_fail("nn_conv_tma: cuTensorMapEncodeTiled (grad_output) failed%s (CUresult %lld)", "", (long long)r);
    }
    {   // layer input: im2col boxes of 64 pixels x 64 channels of one tap
        EncodeIm2colFn enc = get_encode_im2col();
        if (!enc) return nn_fail("nn_conv_tma: cuTensorMapEncodeIm2col is not available%s", "");
        const cuuint64_t Cp = (cuuint64_t)w.Cp;
        cuuint64_t dims[4] = {Cp, (cuuint64_t)c.W, (cuuint64_t)c.H, (cuuint64_t)c.B};
        cuuint64_t strides[3] = {Cp * 2, (cuuint64_t)c.W * Cp * 2, (cuuint64_t)c.H * c.W * Cp * 2};
        int lower[2] = {-c.pad, -c.pad};
        int upper[2] = {c.pad - (c.KW - 1), c.pad - (c.KH - 1)};
        cuuint32_t estr[4] = {1, (cuuint32_t)c.stride, (cuuint32_t)c.stride, 1};
        const CUresult r = enc(&p.map_x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(c.xp), dims, strides, lower, upper, 64, 64, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return nn_fail("nn_conv_tma: cuTensorMapEncodeIm2col (wgrad) failed%s (CUresult %lld)", "", (long long)r);
        int drv = 0;
        cudaDriverGetVersion(&drv);
        if (drv <= 13010 && (size_t)c.B * c.H * c.W * Cp * 2 < 131072) reinterpret_cast<uint64_t*>(&p.map_x)[1] &= ~(1ull << 21);
        if (w.tail_w) {
            const CUresult r2 = enc(&p.map_xt, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(c.xp), dims, strides, lower, upper, 8, 64,
                                    estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r2 != CUDA_SUCCESS) return nn_fail("nn_conv_tma: cuTensorMapEncodeIm2col (wgrad remainder) failed%s (CUresult %lld)", "", (long long)r2);
            if (drv <= 13010 && (size_t)c.B * c.H * c.W * Cp * 2 < 131072) reinterpret_cast<uint64_t*>(&p.map_xt)[1] &= ~(1ull << 21);
        }
    }
    p.taps = w.taps;
    p.partial_tail = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(c.partial) + w.main_bytes);
    p.OH = c.OH; p.OW = c.OW; p.stride = c.stride; p.pad = c.pad; p.KW = c.KW; p.n_c64 = w.n_c64; p.n_atoms = w.n_atoms;
    p.Mpix = c.B * c.OH * c.OW; p.Cout = c.Cout; p.num_kb = w.num_kb; p.kb_per_split = w.kb_per_split; p.stages = w.stages;
    p.cols_pad = w.cols_pad; p.partial = c.partial; p.err_flag = c.err_flag;
    typedef void (*WgradKernel)(const WgTmaP);
    // remainder launch: 8 columns per tap padded to 16 -- square filters of up to 5 x 5 (the plan's limit of 31 taps)
    const int tw = w.tail_w ? (w.taps * 8 + 15) & ~15 : 0;
    const WgradKernel tail = tw == 16 ? k_wgrad_tma<true, 16> : tw == 32 ? k_wgrad_tma<true, 32> : tw == 80 ? k_wgrad_tma<true, 80>
                           : tw == 128 ? k_wgrad_tma<true, 128> : tw == 208 ? k_wgrad_tma<true, 208> : nullptr;
    if (w.tail_w && !tail) return nn_fail("nn_conv_tma: no remainder weight-gradient kernel for%s %lld taps", "", (long long)w.taps);
    NN_ONCE_PER_DEVICE({
        NN_CUDA_OK(cudaFuncSetAttribute(k_wgrad_tma<false, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        for (WgradKernel k : {k_wgrad_tma<true, 16>, k_wgrad_tma<true, 32>, k_wgrad_tma<true, 80>, k_wgrad_tma<true, 128>, k_wgrad_tma<true, 208>})
            NN_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    });
    k_wgrad_tma<false, 0><<<dim3(w.tiles_k, w.m_tiles_n, w.splits), WT_THREADS, w.smem_bytes, st>>>(p);
    NN_LAUNCH_OK();
    if (w.tail_w) {         // the 8-channel remainder columns of every tap: one column tile
        tail<<<dim3(1, w.m_tiles_n, w.splits), WT_THREADS, w.smem_bytes, st>>>(p);
        NN_LAUNCH_OK();
    }
    return 0;
}
