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
// * Persistent: a CTA walks (128-pixel tile, n-tile) items.  Two MMA warpgroups (64 pixels each) accumulate the main
//   and sigma^2 columns in registers and run the epilogue (scale, Philox / Box-Muller current noise -> NCHW stores)
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
    int n_t, n_mma, n_half, n_tiles;
    int items, stages, a_stage, b_stage, n_prod, tap_bytes;
    float y_scale, s_scale;
    float *y, *y_noisy;
    float current;
    const float* scale_dev;
    const float* z_inject;               // EPI 3: N(0,1) draws of the caller (parity hook), [B, Cout, OH, OW]
    nn_rng rng;
    int* err_flag;
};

// EPI 1: noisy (main + sigma accumulators, Philox z), EPI 2: plain, EPI 3: noisy with injected z (parity tests)
template <int EPI>
__global__ void __launch_bounds__((8 + 2) * 32, 1)
k_conv_tma(const __grid_constant__ TmaConvP p) {
    constexpr int MCH = EPI == 2 ? 4 : 2;        // 64-column register chunks of the main / sigma accumulators
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int S = p.stages;
    const uint32_t stage_bytes = (uint32_t)(p.a_stage + p.b_stage);
    const uint32_t bar_base = base + (uint32_t)S * stage_bytes;
    const uint32_t full_bar = bar_base, empty_bar = bar_base + 8u * TC_MAX_STAGES;

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);          // warp-uniform for the compiler: role branches are convergent
    const int P = p.n_prod;

    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full_bar + 8 * s, 1);          // the producer's arrive.expect_tx
            mbar_init(empty_bar + 8 * s, 2);         // both MMA warpgroups have read the stage
        }
        fence_mbar_init();
        tma_prefetch_desc(&p.map64);
        tma_prefetch_desc(&p.map_tail);
        tma_prefetch_desc(&p.mapb64);
        tma_prefetch_desc(&p.mapb_tail);
    }
    __syncthreads();
    const int ohw = p.OH * p.OW;

    if (warp >= 8 && warp < 8 + P) {
        // ---------------------------------------------------------------- producers
        const int pw = warp - 8;
        int s = 0, turn = 0;                                 // ring stage and producer turn of the current group (no div / mod)
        uint32_t eph = 1u;                                   // parity to wait for on the stage's empty barrier
        // (no function call inside the role loops: uniform registers do not survive calls -- the loops break out instead)
        int fail = 0;
        for (int it = blockIdx.x; it < p.items && !fail; it += gridDim.x) {
            const int mt = it / p.n_tiles, nt = it - mt * p.n_tiles;
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
                        // chunk a of the group: rows [half 0 | half 1] at b_dst; chunk b after all n_mma rows of chunk a
                        for (int h = 0; h < 2; ++h) {
                            const long long boff = wt + (long long)tap * p.tap_bytes + (long long)gi * (p.n_half * 512) + (long long)h * half_bytes;
                            const uint32_t da = b_dst + (uint32_t)(h * p.n_half * 2 * wa);
                            if (wa == 64) tma_tile_2d(da, &p.mapb64, bar, 0, (int)(boff >> 7));
                            else tma_tile_2d(da, &p.mapb_tail, bar, 0, (int)(boff / (2 * wa)));
                            if (wb) {
                                const long long boff2 = boff + (long long)p.n_half * 2 * wa;
                                const uint32_t db = b_dst + (uint32_t)(p.n_mma * 2 * wa + h * p.n_half * 2 * wb);
                                if (wb == 64) tma_tile_2d(db, &p.mapb64, bar, 0, (int)(boff2 >> 7));
                                else tma_tile_2d(db, &p.mapb_tail, bar, 0, (int)(boff2 / (2 * wb)));
                            }
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
        constexpr bool noise = EPI != 2;
        float coef = 0.f;
        NnRng rs = {0, 0, 0, 0};
        if (noise) { coef = nn_noise_coef(*p.scale_dev, p.current); rs = nn_rng_load(p.rng); }
        const int ngrp = (p.Cout + 3) >> 2;
        const float y_scale = p.y_scale, s_scale = p.s_scale;
        const int kt = p.tail_w >> 4;
        int s = 0, fail = 0;
        uint32_t fph = 0u;                                   // parity to wait for on the stage's full barrier
        for (int it = blockIdx.x; it < p.items && !fail; it += gridDim.x) {
            const int mt = it / p.n_tiles, nt = it - mt * p.n_tiles;
            float accm[MCH][32], accs[2][32];
            int gi = 0;
            for (int g = 0; g < p.n_groups; ++g) {
                if (!mbar_wait(full_bar + 8 * s, fph)) { fail = 403; break; }
                const int ca = 2 * gi, cb = 2 * gi + 1;
                const bool has_b = cb < p.nc;
                const uint32_t a_s = base + (uint32_t)s * stage_bytes, b_s = a_s + (uint32_t)p.a_stage;
                wg_fence();
#pragma unroll 1
                for (int ch = 0; ch < (has_b ? 2 : 1); ++ch) {
                    const int w = (ch == 0 ? ca : cb) < p.n_c64 ? 64 : p.tail_w;      // channels of this chunk (row = 2 w bytes)
                    const uint32_t a_c = a_s + (ch == 0 ? 0u : 256u * (uint32_t)(ca < p.n_c64 ? 64 : p.tail_w));
                    const uint32_t b_c = b_s + (ch == 0 ? 0u : (uint32_t)(p.n_mma * 2 * (ca < p.n_c64 ? 64 : p.tail_w)));
                    const uint64_t ad = gmma_desc_kmajor(a_c + (uint32_t)(wg * 64 * 2 * w), 2u * (uint32_t)w);
                    const uint64_t bm = gmma_desc_kmajor(b_c, 2u * (uint32_t)w);
                    const uint64_t bsg = gmma_desc_kmajor(b_c + (uint32_t)(p.n_t * 2 * w), 2u * (uint32_t)w);    // sigma rows follow the main rows
                    const uint32_t step = 8u * (uint32_t)w;               // 64 rows of B in descriptor units
                    const int ks = w == 64 ? 4 : kt;
#pragma unroll 1
                    for (int k = 0; k < ks; ++k) {
                        const int acc_on = (g != 0 || ch != 0 || k != 0) ? 1 : 0;
                        wg_mma<MCH, 0, 0>(accm, ad + 2 * k, bm + 2 * k, step, p.n_t, acc_on);
                        if (noise) wg_mma<2, 0, 0>(accs, ad + 2 * k, bsg + 2 * k, step, p.n_t, acc_on);
                    }
                }
                wg_commit();
                wg_wait_all();
                wg_fence_acc(accm);
                if (noise) wg_fence_acc(accs);
                __syncwarp();
                if ((warp & 3) == 0 && elect_one_sync()) mbar_arrive(empty_bar + 8 * s);      // the stage may be refilled
                __syncwarp();
                if (++gi == p.gpt) gi = 0;
                if (++s == S) { s = 0; fph ^= 1u; }
            }
            if (fail) break;
            // ---- epilogue from the fragments: rows r0, r0 + 8; columns 8 i + 2 (l % 4) + {0, 1} of each chunk.  The two
            // lanes l, l ^ 1 share the 4-channel Philox groups of both rows: each draws one and hands over half of it.
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
            const int n_base = nt * p.n_t;
#pragma unroll
            for (int c = 0; c < MCH; ++c)
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int nl = 64 * c + 8 * i + 2 * (lane & 3);        // local column of register 4 i (+1: next column)
                    if (64 * c + 8 * i >= p.n_t) continue;                 // warp-uniform
                    const int n = n_base + nl;
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
                            if (nl + j >= p.n_t || n + j >= p.Cout) continue;
                            const size_t o = orow[h] + (size_t)(n + j) * ohw;
                            const float yv = accm[c][4 * i + 2 * h + j] * y_scale;
                            if (EPI == 2) {
                                out[o] = yv;
                            } else {
                                const float zv = EPI == 3 ? __ldg(p.z_inject + o) : z[h][j];
                                out[o] = __fadd_rn(yv, __fmul_rn(zv, nn_sigma(coef, accs[c & 1][4 * i + 2 * h + j] * s_scale)));      // (MCH == 2)
                            }
                        }
                    }
                }
        }
        if (fail) nn_pipeline_abort(p.err_flag, fail);
    }
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
    if (pl.n_t > (has_sigma ? 128 : 256)) return false;     // register accumulators of the MMA warpgroups
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
    p.n_t = pl.n_t; p.n_mma = pl.n_mma; p.n_half = pl.n_half; p.n_tiles = pl.n_tiles;
    p.items = ((p.M + 127) / 128) * pl.n_tiles;
    p.stages = pl.stages; p.a_stage = pl.a_stage; p.b_stage = pl.b_stage; p.n_prod = pl.n_prod; p.tap_bytes = pl.tap_bytes;
    p.y_scale = c.y_scale; p.s_scale = c.s_scale; p.y = c.y; p.y_noisy = c.y_noisy;
    p.current = c.current; p.scale_dev = c.scale_dev; p.z_inject = c.z_inject; p.rng = c.rng; p.err_flag = c.err_flag;
    int grid = nn_num_sms(device);          // persistent: one CTA per SM
    if (grid > p.items) grid = p.items;
    NN_ONCE_PER_DEVICE({
        NN_CUDA_OK(cudaFuncSetAttribute(k_conv_tma<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        NN_CUDA_OK(cudaFuncSetAttribute(k_conv_tma<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        NN_CUDA_OK(cudaFuncSetAttribute(k_conv_tma<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    });
    if (c.ev0) cudaEventRecord((cudaEvent_t)c.ev0, st);          // measurement hook: brackets the kernel, not the host-side descriptor encoding
    if (c.noise_mode != NN_NOISE_NONE && c.z_inject) k_conv_tma<3><<<grid, pl.threads, pl.smem_bytes, st>>>(p);
    else if (c.noise_mode != NN_NOISE_NONE) k_conv_tma<1><<<grid, pl.threads, pl.smem_bytes, st>>>(p);
    else k_conv_tma<2><<<grid, pl.threads, pl.smem_bytes, st>>>(p);
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

template <bool TAIL>
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
        // B: main -- SWIZZLE_128B atoms (LBO = atom stride 8192 B, 16 pixels = 2048 B); remainder slab -- LBO = 8-pixel groups
        // 128 B apart, SBO = the taps' slabs 1 KB apart, 16 pixels = 256 B
        const int wg = warp >> 2;
        const uint64_t da = gmma_desc(0u, 8192u >> 4, 1024u >> 4, 1u);
        const uint64_t db = TAIL ? gmma_desc(0u, 8u, 64u, 0u) : da;
        const uint32_t b_step = 512u, k_step_b = TAIL ? 16u : 128u;
        float acc[4][32];
        int s = 0;
        uint32_t ph = 0u;
        for (int i = 0; i < nkb; ++i) {
            if (!mbar_wait(full_bar + 8 * s, ph)) { fail = 502; break; }
            const uint32_t a_s = (base + (uint32_t)s * WT_STAGE + (uint32_t)wg * 8192u) >> 4, b_s = (base + (uint32_t)s * WT_STAGE + 16384u) >> 4;
            const uint64_t ad = da | (uint64_t)(a_s & 0x3FFFu), bd = db | (uint64_t)(b_s & 0x3FFFu);
            wg_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) wg_mma<4, 1, 1>(acc, ad + 128 * k, bd + k_step_b * k, b_step, n_cols, (i | k) != 0 ? 1 : 0);
            wg_commit();
            wg_wait_all();
            wg_fence_acc(acc);
            __syncwarp();
            if ((warp & 3) == 0 && elect_one_sync()) mbar_arrive(empty_bar + 8 * s);
            __syncwarp();
            if (++s == S) { s = 0; ph ^= 1u; }
        }
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
                                nkb > 0 ? make_float2(acc[c][4 * j + 2 * h], acc[c][4 * j + 2 * h + 1]) : make_float2(0.f, 0.f);
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
    NN_ONCE_PER_DEVICE({
        NN_CUDA_OK(cudaFuncSetAttribute(k_wgrad_tma<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        NN_CUDA_OK(cudaFuncSetAttribute(k_wgrad_tma<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    });
    k_wgrad_tma<false><<<dim3(w.tiles_k, w.m_tiles_n, w.splits), WT_THREADS, w.smem_bytes, st>>>(p);
    NN_LAUNCH_OK();
    if (w.tail_w) {         // the 8-channel remainder columns of every tap: one column tile
        k_wgrad_tma<true><<<dim3(1, w.m_tiles_n, w.splits), WT_THREADS, w.smem_bytes, st>>>(p);
        NN_LAUNCH_OK();
    }
    return 0;
}
