// CUDA-core fp32 implicit-GEMM kernels (NN_PREC_FP32): the reference-arithmetic path.
// Any stride / padding; conv and linear (H=W=KH=KW=1).  These kernels define the exact-fp32
// behaviour the tensor-core kernels (nn_conv_umma.cu) are checked against on the device, and
// serve geometries the tensor-core path does not take.
//
//  forward : M = B*OH*OW, N = Cout, K = Cin*KH*KW.  Two (three) accumulators per output:
//            Y = x (*) w_eff,  S = x (*) g(|w_raw|)  [, P = x (*) |w_raw| for the power stat],
//            epilogue adds bias, draws Philox normals, writes y and y + z*sqrt(c*S).
//  dgrad   : M = B*H*W,   N = Cin,  K = Cout*KH*KW, STE mask fused in the store.
//  wgrad   : M = Cout,    N = Cin*KH*KW, reduction over B*OH*OW, deterministic split +
//            reduce kernel with the weight-quantizer STE mask fused.
#include "nn_common.cuh"

namespace {

constexpr int BM = 64, BN = 64, BK = 16, PAD = 4, NT = 256;

struct FwdP {
    nn_conv_geom g;
    int OH, OW, M, K;
    const float *x, *w_eff, *w_raw, *bias, *scale_dev, *z_inject;
    float *y, *y_noisy, *z_export, *sigma_export, *stats;
    float current;
    nn_rng rng;
};

// NOISE: 0 none, 1 merged (|w|), 2 external (|w|^2+|w|).  PLAIN: also accumulate x (*) |w| (power stat
// of the external-DAC branch, hardware_model.py:67-68,74-79).
template <int NOISE, bool PLAIN>
__global__ void __launch_bounds__(NT)
k_conv_fwd_simt(const FwdP p) {
    __shared__ __align__(16) float As[BK][BM + PAD];
    __shared__ __align__(16) float Bs[BK][BN + PAD];
    __shared__ __align__(16) float Bs2[NOISE ? BK : 1][BN + PAD];
    __shared__ __align__(16) float Bs3[PLAIN ? BK : 1][BN + PAD];
    __shared__ float red[3][NT / 32];

    const int t = threadIdx.x;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const nn_conv_geom g = p.g;
    const int KHW = g.KH * g.KW, OHW = p.OH * p.OW;

    // A loader: m_local = t % 64, k_local = t / 64 + 4 j
    const int am = t & 63, ak = t >> 6;
    const int gm = m0 + am;
    const bool am_ok = gm < p.M;
    int ab = 0, aoh = 0, aow = 0;
    if (am_ok) { ab = gm / OHW; int r = gm - ab * OHW; aoh = r / p.OW; aow = r - aoh * p.OW; }
    const int ih0 = aoh * g.stride - g.pad, iw0 = aow * g.stride - g.pad;
    const float* xb = p.x + (int64_t)ab * g.Cin * g.H * g.W;
    // B loader: k_local = t % 16, n_local = t / 16 + 16 j
    const int bk = t & 15, bn = t >> 4;

    const int tm = t & 15, tn = t >> 4;      // micro tile: rows tm*4.., cols tn*4..
    float acc[4][4] = {}, acc2[4][4] = {}, acc3[4] = {};

    for (int k0 = 0; k0 < p.K; k0 += BK) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int kl = ak + 4 * j, k = k0 + kl;
            float v = 0.f;
            if (am_ok && k < p.K) {
                int c = k / KHW, r = k - c * KHW, kh = r / g.KW, kw = r - kh * g.KW;
                int ih = ih0 + kh, iw = iw0 + kw;
                if ((unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W)
                    v = __ldg(xb + ((int64_t)c * g.H + ih) * g.W + iw);
            }
            As[kl][am] = v;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int nl = bn + 16 * j, n = n0 + nl, k = k0 + bk;
            float v = 0.f, v2 = 0.f, v3 = 0.f;
            if (n < g.Cout && k < p.K) {
                if (p.w_eff) v = __ldg(p.w_eff + (int64_t)n * p.K + k);
                if (NOISE) {
                    float a = fabsf(__ldg(p.w_raw + (int64_t)n * p.K + k));
                    v3 = a;
                    v2 = (NOISE == 1) ? a : __fadd_rn(__fmul_rn(a, a), a);   // abs_weights.pow(2) + abs_weights (:62)
                }
            }
            Bs[bk][nl] = v;
            if (NOISE) Bs2[bk][nl] = v2;
            if (PLAIN) Bs3[bk][nl] = v3;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a4 = *reinterpret_cast<const float4*>(&As[k][tm * 4]);
            const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tn * 4]);
            const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            if (NOISE) {
                const float4 c4 = *reinterpret_cast<const float4*>(&Bs2[k][tn * 4]);
                const float c[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc2[i][j] = fmaf(a[i], c[j], acc2[i][j]);
            }
            if (PLAIN) {
                const float4 d4 = *reinterpret_cast<const float4*>(&Bs3[k][tn * 4]);
                const float ds = (d4.x + d4.y) + (d4.z + d4.w);
#pragma unroll
                for (int i = 0; i < 4; ++i) acc3[i] = fmaf(a[i], ds, acc3[i]);
            }
        }
        __syncthreads();
    }

    // ---------------- epilogue
    float coef = 0.f;
    NnRng rs = {0, 0, 0, 0};
    if (NOISE) { coef = nn_noise_coef(*p.scale_dev, p.current); rs = nn_rng_load(p.rng); }
    const int ngrp = (g.Cout + 3) >> 2;
    float s_plain = 0.f, s_abs = 0.f, s_max = __int_as_float(0xff800000);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + tm * 4 + i;
        if (m >= p.M) continue;
        const int b = m / OHW, pix = m - b * OHW;
        float z[4] = {0.f, 0.f, 0.f, 0.f};
        const int nbase = n0 + tn * 4;
        if (NOISE && !p.z_inject && nbase < g.Cout) nn_normal4(rs, (uint64_t)m * ngrp + (nbase >> 2), z);
        if (PLAIN) s_plain += acc3[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = nbase + j;
            if (n >= g.Cout) continue;
            const int64_t o = ((int64_t)b * g.Cout + n) * OHW + pix;
            float yv;
            if (p.w_eff) {
                yv = acc[i][j];
                if (p.bias) yv = __fadd_rn(yv, __ldg(p.bias + n));
                if (p.y) p.y[o] = yv;
            } else {
                yv = p.y[o];          // noise-only mode: the clean output is an input
            }
            if (NOISE) {
                const float S = acc2[i][j];
                const float sg = nn_sigma(coef, S);
                const float zz = p.z_inject ? __ldg(p.z_inject + o) : z[j];
                const float nz = __fmul_rn(zz, sg);
                p.y_noisy[o] = __fadd_rn(yv, nz);
                if (p.z_export) p.z_export[o] = zz;
                if (p.sigma_export) p.sigma_export[o] = sg;
                if (NOISE == 1) s_plain += S;
                s_abs += fabsf(nz);
                s_max = fmaxf(s_max, yv);
            }
        }
    }
    if (NOISE && p.stats) {
        s_plain = nn_warp_sum(s_plain); s_abs = nn_warp_sum(s_abs); s_max = nn_warp_max(s_max);
        const int w = t >> 5, l = t & 31;
        if (l == 0) { red[0][w] = s_plain; red[1][w] = s_abs; red[2][w] = s_max; }
        __syncthreads();
        if (w == 0) {
            s_plain = l < NT / 32 ? red[0][l] : 0.f;
            s_abs = l < NT / 32 ? red[1][l] : 0.f;
            s_max = l < NT / 32 ? red[2][l] : __int_as_float(0xff800000);
            s_plain = nn_warp_sum(s_plain); s_abs = nn_warp_sum(s_abs); s_max = nn_warp_max(s_max);
            if (l == 0) {
                atomicAdd(p.stats + 0, s_plain);
                atomicAdd(p.stats + 1, s_abs);
                nn_atomic_max_float(p.stats + 2, s_max);
            }
        }
    }
}

// ------------------------------------------------------------------ dgrad
struct DgP {
    nn_conv_geom g;
    int OH, OW, M, K;   // M = B*H*W, K = Cout*KH*KW
    const float *gy, *w, *x_pre;
    float* gx;
    float lo, hi;
};

__global__ void __launch_bounds__(NT)
k_conv_dgrad_simt(const DgP p) {
    __shared__ __align__(16) float As[BK][BM + PAD];
    __shared__ __align__(16) float Bs[BK][BN + PAD];
    const int t = threadIdx.x;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const nn_conv_geom g = p.g;
    const int KHW = g.KH * g.KW, HW = g.H * g.W, OHW = p.OH * p.OW;

    const int am = t & 63, ak = t >> 6;
    const int gm = m0 + am;
    const bool am_ok = gm < p.M;
    int ab = 0, ah = 0, aw = 0;
    if (am_ok) { ab = gm / HW; int r = gm - ab * HW; ah = r / g.W; aw = r - ah * g.W; }
    const float* gyb = p.gy + (int64_t)ab * g.Cout * OHW;
    const int bk = t & 15, bn = t >> 4;
    const int tm = t & 15, tn = t >> 4;
    float acc[4][4] = {};

    for (int k0 = 0; k0 < p.K; k0 += BK) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int kl = ak + 4 * j, k = k0 + kl;
            float v = 0.f;
            if (am_ok && k < p.K) {
                int n = k / KHW, r = k - n * KHW, kh = r / g.KW, kw = r - kh * g.KW;
                int th = ah + g.pad - kh, tw = aw + g.pad - kw;
                if (th >= 0 && tw >= 0) {
                    int oh = th / g.stride, ow = tw / g.stride;
                    if (oh * g.stride == th && ow * g.stride == tw && oh < p.OH && ow < p.OW)
                        v = __ldg(gyb + (int64_t)n * OHW + oh * p.OW + ow);
                }
            }
            As[kl][am] = v;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int cl = bn + 16 * j, c = n0 + cl, k = k0 + bk;
            float v = 0.f;
            if (c < g.Cin && k < p.K) {
                int n = k / KHW, r = k - n * KHW;
                v = __ldg(p.w + ((int64_t)n * g.Cin + c) * KHW + r);
            }
            Bs[bk][cl] = v;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a4 = *reinterpret_cast<const float4*>(&As[k][tm * 4]);
            const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tn * 4]);
            const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + tm * 4 + i;
        if (m >= p.M) continue;
        const int b = m / HW, pix = m - b * HW;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = n0 + tn * 4 + j;
            if (c >= g.Cin) continue;
            const int64_t o = ((int64_t)b * g.Cin + c) * HW + pix;
            float v = acc[i][j];
            if (p.x_pre) { float xv = __ldg(p.x_pre + o); if (xv > p.hi || xv < p.lo) v = 0.f; }
            p.gx[o] = v;
        }
    }
}

// ------------------------------------------------------------------ wgrad (split reduction)
struct WgP {
    nn_conv_geom g;
    int OH, OW, R, K, r_per_split;   // R = B*OH*OW
    const float *gy, *x;
    float* partial;                  // [splits][Cout][K]
};

__global__ void __launch_bounds__(NT)
k_conv_wgrad_simt(const WgP p) {
    __shared__ __align__(16) float As[BK][BM + PAD];   // [r][n]
    __shared__ __align__(16) float Bs[BK][BN + PAD];   // [r][k]
    const int t = threadIdx.x;
    const int n0 = blockIdx.y * BM, k0 = blockIdx.x * BN;
    const nn_conv_geom g = p.g;
    const int KHW = g.KH * g.KW, OHW = p.OH * p.OW;
    const int r_begin = blockIdx.z * p.r_per_split;
    const int r_end = min(p.R, r_begin + p.r_per_split);

    const int lr = t & 15, lc = t >> 4;     // loaders: r_local = t%16, col = t/16 + 16 j
    // per-thread constant decomposition of the 4 k columns this thread loads
    int kc[4], kkh[4], kkw[4];
    bool kok[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        int k = k0 + lc + 16 * j;
        kok[j] = k < p.K;
        int kk = kok[j] ? k : 0;
        kc[j] = kk / KHW; int r = kk - kc[j] * KHW; kkh[j] = r / g.KW; kkw[j] = r - kkh[j] * g.KW;
    }
    const int tm = t & 15, tn = t >> 4;      // micro tile: n rows tm*4.., k cols tn*4..
    float acc[4][4] = {};

    for (int r0 = r_begin; r0 < r_end; r0 += BK) {
        const int r = r0 + lr;
        const bool rok = r < r_end;
        int b = 0, oh = 0, ow = 0;
        if (rok) { b = r / OHW; int q = r - b * OHW; oh = q / p.OW; ow = q - oh * p.OW; }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int nl = lc + 16 * j, n = n0 + nl;
            float v = 0.f;
            if (rok && n < g.Cout) v = __ldg(p.gy + ((int64_t)b * g.Cout + n) * OHW + oh * p.OW + ow);
            As[lr][nl] = v;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float v = 0.f;
            if (rok && kok[j]) {
                int ih = oh * g.stride - g.pad + kkh[j], iw = ow * g.stride - g.pad + kkw[j];
                if ((unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W)
                    v = __ldg(p.x + (((int64_t)b * g.Cin + kc[j]) * g.H + ih) * g.W + iw);
            }
            Bs[lr][lc + 16 * j] = v;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a4 = *reinterpret_cast<const float4*>(&As[k][tm * 4]);
            const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tn * 4]);
            const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* out = p.partial + (int64_t)blockIdx.z * g.Cout * p.K;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n0 + tm * 4 + i;
        if (n >= g.Cout) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0 + tn * 4 + j;
            if (k < p.K) out[(int64_t)n * p.K + k] = acc[i][j];
        }
    }
}

}  // namespace

// Shared with the tensor-core path: sums split partials in a fixed order and applies the STE mask.
__global__ void __launch_bounds__(256)
k_wgrad_reduce(const float* __restrict__ partial, int splits, int64_t n, float* __restrict__ gw,
               const float* __restrict__ w_raw, float lo, float hi) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int z = 0; z < splits; ++z) s += partial[(int64_t)z * n + i];
        if (w_raw) { float w = __ldg(w_raw + i); if (w > hi || w < lo) s = 0.f; }
        gw[i] = s;
    }
}

static int simt_wgrad_splits(const nn_conv_geom& g, int device) {
    int OH, OW; nn_out_hw(g, OH, OW);
    const int K = g.Cin * g.KH * g.KW;
    const int64_t R = (int64_t)g.B * OH * OW;
    const int tiles = ((K + BN - 1) / BN) * ((g.Cout + BM - 1) / BM);
    int splits = (4 * nn_num_sms(device) + tiles - 1) / tiles;
    int64_t max_splits = (R + 4 * BK - 1) / (4 * BK);
    if (splits > max_splits) splits = (int)max_splits;
    if (splits < 1) splits = 1;
    if (splits > 256) splits = 256;
    return splits;
}

int64_t nn_simt_wgrad_workspace(const nn_conv_geom* g, int device) {
    return (int64_t)simt_wgrad_splits(*g, device) * g->Cout * g->Cin * g->KH * g->KW * sizeof(float);
}

int nn_simt_conv_fwd(const nn_conv_fwd_args* a, int device, cudaStream_t st) {
    FwdP p;
    p.g = a->g;
    nn_out_hw(a->g, p.OH, p.OW);
    p.M = a->g.B * p.OH * p.OW;
    p.K = a->g.Cin * a->g.KH * a->g.KW;
    p.x = a->x; p.w_eff = a->w_eff; p.w_raw = a->w_raw; p.bias = a->bias; p.scale_dev = a->scale_dev;
    p.z_inject = a->z_inject; p.y = a->y; p.y_noisy = a->y_noisy; p.z_export = a->z_export;
    p.sigma_export = a->sigma_export; p.stats = a->stats; p.current = a->current; p.rng = a->rng;
    dim3 grid((p.M + BM - 1) / BM, (a->g.Cout + BN - 1) / BN);
    const bool plain = a->noise_mode == NN_NOISE_EXTERNAL && a->stats != nullptr;
    switch (a->noise_mode) {
        case NN_NOISE_NONE: k_conv_fwd_simt<0, false><<<grid, NT, 0, st>>>(p); break;
        case NN_NOISE_MERGED: k_conv_fwd_simt<1, false><<<grid, NT, 0, st>>>(p); break;
        default:
            if (plain) k_conv_fwd_simt<2, true><<<grid, NT, 0, st>>>(p);
            else k_conv_fwd_simt<2, false><<<grid, NT, 0, st>>>(p);
    }
    NN_LAUNCH_OK();
    return 0;
}

int nn_simt_conv_dgrad(const nn_conv_dgrad_args* a, int device, cudaStream_t st) {
    DgP p;
    p.g = a->g;
    nn_out_hw(a->g, p.OH, p.OW);
    p.M = a->g.B * a->g.H * a->g.W;
    p.K = a->g.Cout * a->g.KH * a->g.KW;
    p.gy = a->gy; p.w = a->w_eff; p.x_pre = a->x_pre; p.gx = a->gx;
    p.lo = (float)a->x_lo; p.hi = (float)a->x_hi;
    dim3 grid((p.M + BM - 1) / BM, (a->g.Cin + BN - 1) / BN);
    k_conv_dgrad_simt<<<grid, NT, 0, st>>>(p);
    NN_LAUNCH_OK();
    return 0;
}

int nn_simt_conv_wgrad(const nn_conv_wgrad_args* a, int device, cudaStream_t st) {
    WgP p;
    p.g = a->g;
    nn_out_hw(a->g, p.OH, p.OW);
    p.R = a->g.B * p.OH * p.OW;
    p.K = a->g.Cin * a->g.KH * a->g.KW;
    const int splits = simt_wgrad_splits(a->g, device);
    const int64_t need = (int64_t)splits * a->g.Cout * p.K * sizeof(float);
    if (!a->workspace || a->workspace_bytes < need)
        return nn_fail("nn_noisy_conv_wgrad: workspace too small%s (need %lld bytes)", "", need);
    p.r_per_split = (((p.R + splits - 1) / splits) + BK - 1) / BK * BK;
    p.gy = a->gy; p.x = a->x; p.partial = (float*)a->workspace;
    dim3 grid((p.K + BN - 1) / BN, (a->g.Cout + BM - 1) / BM, splits);
    k_conv_wgrad_simt<<<grid, NT, 0, st>>>(p);
    NN_LAUNCH_OK();
    const int64_t n = (int64_t)a->g.Cout * p.K;
    int rb = (int)((n + 255) / 256);
    if (rb > 4 * nn_num_sms(device)) rb = 4 * nn_num_sms(device);
    k_wgrad_reduce<<<rb, 256, 0, st>>>(p.partial, splits, n, a->gw, a->w_raw, (float)a->w_lo, (float)a->w_hi);
    NN_LAUNCH_OK();
    return 0;
}
