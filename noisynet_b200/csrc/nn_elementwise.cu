// Elementwise / reduction kernels of the NoisyNet hot path (HBM-bound; float4 vectorised,
// grid sized in multiples of the SM count, Philox drawn in registers -- no separate RNG kernel).
#include "nn_common.cuh"

thread_local char g_nn_err[512] = "";
unsigned long long g_nn_launches = 0;
extern "C" uint64_t nn_launch_count(void) { return g_nn_launches; }

extern "C" const char* nn_last_error(void) { return g_nn_err; }
extern "C" int nn_abi_version(void) { return NN_ABI_VERSION; }

extern "C" int nn_device_info(int device, int* sm_count, int* cc_major, int* cc_minor) {
    int sms = 0, maj = 0, min_ = 0;
    NN_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    NN_CUDA_OK(cudaDeviceGetAttribute(&maj, cudaDevAttrComputeCapabilityMajor, device));
    NN_CUDA_OK(cudaDeviceGetAttribute(&min_, cudaDevAttrComputeCapabilityMinor, device));
    if (sm_count) *sm_count = sms;
    if (cc_major) *cc_major = maj;
    if (cc_minor) *cc_minor = min_;
    if (maj != 9 || min_ != 0) return nn_fail("noisynet_b200 is built for sm_90a only; device has compute capability %s%lld", "", (long long)(10 * maj + min_));
    return 0;
}

static inline int nn_grid_for(int64_t work_items, int threads, int device, int waves = 8) {
    int64_t blocks = (work_items + threads - 1) / threads;
    int64_t cap = (int64_t)nn_num_sms(device) * waves;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

__global__ void k_rng_advance(uint64_t* p, uint64_t inc) { *p += inc; }

extern "C" int nn_rng_advance(uint64_t* offset_dev, uint64_t inc, int device, void* stream) {
    NN_SET_DEVICE(device);
    k_rng_advance<<<1, 1, 0, (cudaStream_t)stream>>>(offset_dev, inc);
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ a1 quantize fwd
// One thread = one Philox group = 4 consecutive elements.
__device__ __forceinline__ float quant_one(float x, float neg_min, float scale, float qmax, float u,
                                           float min_v) {
    float t = __fdiv_rn(__fadd_rn(x, neg_min), scale);   // add_(-min).div_(scale)   (:154)
    t = __fadd_rn(t, u);                                  // add_(noise)              (:162)
    t = fminf(fmaxf(t, 0.0f), qmax);                      // clamp_(qmin, qmax)       (:166)
    t = rintf(t);                                         // round_() half-to-even    (:166)
    return __fadd_rn(__fmul_rn(t, scale), min_v);         // mul_(scale).add_(min)    (:170)
}

__global__ void __launch_bounds__(256)
k_quantize_fwd(const float* __restrict__ x, float* __restrict__ y, int64_t n, float neg_min, float min_v,
               float scale, float qmax, float stoch, const float* __restrict__ u_inject, nn_rng rng,
               const float* __restrict__ range_dev) {
    if (range_dev) {        // range selected on the device (nn_range_select): the host arithmetic of :148-151 in doubles
        const double mn = (double)range_dev[0], mx = (double)range_dev[1];
        double sc = (mx - mn) / (double)qmax;
        if (sc < 1e-6) sc = 1e-6;
        scale = (float)sc; neg_min = (float)(-mn); min_v = (float)mn;
    }
    const NnRng s = nn_rng_load(rng);
    const int64_t ngroups = (n + 3) >> 2;
    const bool vec = ((((uintptr_t)x | (uintptr_t)y | (uintptr_t)u_inject) & 15) == 0);
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < ngroups;
         g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i0 = g << 2;
        float xv[4], uv[4] = {0.f, 0.f, 0.f, 0.f};
        const bool full = vec && (i0 + 3 < n);
        if (full) {
            float4 t = *reinterpret_cast<const float4*>(x + i0);
            xv[0] = t.x; xv[1] = t.y; xv[2] = t.z; xv[3] = t.w;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) xv[j] = (i0 + j < n) ? x[i0 + j] : 0.f;
        }
        if (stoch > 0.f) {
            if (u_inject) {
#pragma unroll
                for (int j = 0; j < 4; ++j) uv[j] = (i0 + j < n) ? u_inject[i0 + j] : 0.f;
            } else {
                uint4 r = nn_philox(s, (uint64_t)g);
                uv[0] = nn_usym(r.x, stoch); uv[1] = nn_usym(r.y, stoch);
                uv[2] = nn_usym(r.z, stoch); uv[3] = nn_usym(r.w, stoch);
            }
        }
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = quant_one(xv[j], neg_min, scale, qmax, uv[j], min_v);
        if (full) {
            *reinterpret_cast<float4*>(y + i0) = make_float4(o[0], o[1], o[2], o[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (i0 + j < n) y[i0 + j] = o[j];
        }
    }
}

extern "C" int nn_quantize_fwd(const float* x, float* y, int64_t n, int bits, double min_value,
                               double max_value, float stochastic, const float* u_inject, nn_rng rng,
                               int device, void* stream) {
    if (n <= 0) return 0;
    if (bits < 1 || bits > 16) return nn_fail("nn_quantize_fwd: bits out of range%s (%lld)", "", bits);
    NN_SET_DEVICE(device);
    // hardware_model.py:148-151 -- scale computed in doubles, then used as an fp32 scalar
    double qmax = (double)((1u << bits) - 1u);
    double scale = (max_value - min_value) / qmax;
    if (scale < 1e-6) scale = 1e-6;
    int threads = 256;
    int grid = nn_grid_for((n + 3) / 4, threads, device);
    k_quantize_fwd<<<grid, threads, 0, (cudaStream_t)stream>>>(
        x, y, n, (float)(-min_value), (float)min_value, (float)scale, (float)qmax, stochastic, u_inject, rng, nullptr);
    NN_LAUNCH_OK();
    return 0;
}

extern "C" int nn_quantize_fwd_dev(const float* x, float* y, int64_t n, int bits, const float* range_dev, float stochastic,
                                   const float* u_inject, nn_rng rng, int device, void* stream) {
    if (n <= 0) return 0;
    if (bits < 1 || bits > 16) return nn_fail("nn_quantize_fwd_dev: bits out of range%s (%lld)", "", bits);
    if (!range_dev) return nn_fail("nn_quantize_fwd_dev: range_dev missing%s", "");
    NN_SET_DEVICE(device);
    const double qmax = (double)((1u << bits) - 1u);
    k_quantize_fwd<<<nn_grid_for((n + 3) / 4, 256, device), 256, 0, (cudaStream_t)stream>>>(
        x, y, n, 0.f, 0.f, 1.f, (float)qmax, stochastic, u_inject, rng, range_dev);
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ a2 quantize bwd (STE)
__global__ void __launch_bounds__(256)
k_quantize_bwd(const float* __restrict__ x, const float* __restrict__ gy, float* __restrict__ gx,
               int64_t n, float lo, float hi, const float* __restrict__ range_dev) {
    if (range_dev) { lo = range_dev[0]; hi = range_dev[1]; }
    const bool vec = ((((uintptr_t)x | (uintptr_t)gy | (uintptr_t)gx) & 15) == 0);
    const int64_t ngroups = (n + 3) >> 2;
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < ngroups;
         g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i0 = g << 2;
        if (vec && i0 + 3 < n) {
            float4 xv = *reinterpret_cast<const float4*>(x + i0);
            float4 gv = *reinterpret_cast<const float4*>(gy + i0);
            gv.x = (xv.x > hi || xv.x < lo) ? 0.f : gv.x;
            gv.y = (xv.y > hi || xv.y < lo) ? 0.f : gv.y;
            gv.z = (xv.z > hi || xv.z < lo) ? 0.f : gv.z;
            gv.w = (xv.w > hi || xv.w < lo) ? 0.f : gv.w;
            *reinterpret_cast<float4*>(gx + i0) = gv;
        } else {
            for (int j = 0; j < 4 && i0 + j < n; ++j) {
                float xv = x[i0 + j];
                gx[i0 + j] = (xv > hi || xv < lo) ? 0.f : gy[i0 + j];
            }
        }
    }
}

extern "C" int nn_quantize_bwd(const float* x, const float* gy, float* gx, int64_t n, double min_value,
                               double max_value, int device, void* stream) {
    if (n <= 0) return 0;
    NN_SET_DEVICE(device);
    int threads = 256;
    int grid = nn_grid_for((n + 3) / 4, threads, device);
    k_quantize_bwd<<<grid, threads, 0, (cudaStream_t)stream>>>(x, gy, gx, n, (float)min_value, (float)max_value, nullptr);
    NN_LAUNCH_OK();
    return 0;
}

extern "C" int nn_quantize_bwd_dev(const float* x, const float* gy, float* gx, int64_t n, const float* range_dev, int device,
                                   void* stream) {
    if (n <= 0) return 0;
    if (!range_dev) return nn_fail("nn_quantize_bwd_dev: range_dev missing%s", "");
    NN_SET_DEVICE(device);
    k_quantize_bwd<<<nn_grid_for((n + 3) / 4, 256, device), 256, 0, (cudaStream_t)stream>>>(x, gy, gx, n, 0.f, 0.f, range_dev);
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ a3 on the device: range selection of QuantMeasure
// hardware_model.py:232-259 picks the quantisation range with torch.kthvalue (a sort) and input.max().item() (a host
// sync per layer per batch while calibrating).  Here: an exact radix select over the order-preserving integer image of
// the floats -- 4 passes of 256-bin histograms restricted to the prefix found so far -- and an atomic max, all on the
// stream; the results stay in device memory and feed nn_quantize_fwd_dev / nn_quantize_bwd_dev directly.
//   domain 0: every element       (activations, :249)           rank k given by the host: int(n * pctl / 100)
//   domain 1: elements > 0        (signed weights, :233-235)    rank int(count * pctl / 100) computed on the device
//   domain 2: |elements < 0|
struct RangeSel {                    // device scratch of one selection
    unsigned long long hist[256];
    unsigned long long k;            // remaining rank (1-based) inside the current prefix
    unsigned int prefix;             // key bits decided so far (high bits)
    unsigned int pass;
    float max_all;                   // max over ALL elements (domain 0 only)
    float result;
};

__device__ __forceinline__ unsigned int nn_float_key(float f) {
    const unsigned int u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float nn_key_float(unsigned int k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

__global__ void k_range_init(RangeSel* sel, int nsel, long long k0) {
    for (int j = 0; j < nsel; ++j) {
        RangeSel& r = sel[j];
        if (threadIdx.x < 256) r.hist[threadIdx.x] = 0ull;
        if (threadIdx.x == 0) { r.k = (unsigned long long)k0; r.prefix = 0u; r.pass = 0u; r.max_all = __int_as_float(0xff800000); r.result = 0.f; }
    }
}

// histogram of byte (3 - pass) of the keys that match the decided prefix; pass 0 also takes max(x)
__global__ void __launch_bounds__(256)
k_range_hist(const float* __restrict__ x, int64_t n, RangeSel* sel, int first_domain, int nsel) {
    __shared__ unsigned int sh[2][256];
    for (int j = 0; j < nsel; ++j) sh[j][threadIdx.x] = 0u;
    __syncthreads();
    const unsigned int pass = sel[0].pass;
    const int shift = 24 - 8 * (int)pass;
    unsigned int pre[2], mask = pass == 0 ? 0u : (0xFFFFFFFFu << (32 - 8 * pass));
    for (int j = 0; j < nsel; ++j) pre[j] = sel[j].prefix;
    float mx = __int_as_float(0xff800000);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = __ldg(x + i);
        mx = fmaxf(mx, v);
        for (int j = 0; j < nsel; ++j) {
            const int d = first_domain + j;
            float t = v;
            bool in = true;
            if (d == 1) in = v > 0.f;
            else if (d == 2) { in = v < 0.f; t = -v; }
            if (!in) continue;
            const unsigned int key = nn_float_key(t);
            if ((key & mask) == pre[j]) atomicAdd(&sh[j][(key >> shift) & 255u], 1u);
        }
    }
    __syncthreads();
    for (int j = 0; j < nsel; ++j)
        if (sh[j][threadIdx.x]) atomicAdd(&sel[j].hist[threadIdx.x], (unsigned long long)sh[j][threadIdx.x]);
    if (pass == 0 && first_domain == 0) {
        mx = nn_warp_max(mx);
        if ((threadIdx.x & 31) == 0) nn_atomic_max_float(&sel[0].max_all, mx);
    }
}

// one warp: find the bin that holds rank k, descend into it
__global__ void k_range_pick(RangeSel* sel, int nsel, double pctl, int rank_from_count, float* out4, int mode, double min_value) {
    if (threadIdx.x == 0) {
        for (int j = 0; j < nsel; ++j) {
            RangeSel& r = sel[j];
            if (r.pass == 0 && rank_from_count) {
                unsigned long long cnt = 0;
                for (int b = 0; b < 256; ++b) cnt += r.hist[b];
                r.k = (unsigned long long)((double)cnt * pctl / 100.);          // int(numel * pctl / 100.)   (:233-234)
            }
            unsigned long long k = r.k, cum = 0;
            int bin = 255;
            for (int b = 0; b < 256; ++b) {
                if (cum + r.hist[b] >= k && k >= 1) { bin = b; break; }
                cum += r.hist[b];
            }
            r.k = k - cum;
            r.prefix |= (unsigned int)bin << (24 - 8 * r.pass);
            r.pass += 1;
            for (int b = 0; b < 256; ++b) r.hist[b] = 0ull;
            if (r.pass == 4) r.result = nn_key_float(r.prefix);
        }
        if (sel[0].pass == 4) {
            if (mode == 0) { out4[0] = sel[0].result; out4[1] = sel[0].max_all; out4[2] = (float)min_value; out4[3] = sel[0].max_all; }
            else { out4[0] = -sel[1].result; out4[1] = sel[0].result; out4[2] = -sel[1].result; out4[3] = sel[0].result; }
        }
    }
}

extern "C" int64_t nn_range_scratch_bytes(void) { return (int64_t)(2 * sizeof(RangeSel) + 64); }

extern "C" int nn_range_select(const float* x, int64_t n, int64_t k_rank, double pctl_percent, int mode, double min_value, float* out4,
                               void* scratch, int device, void* stream) {
    if (!x || !out4 || !scratch || n <= 0) return nn_fail("nn_range_select: bad arguments%s", "");
    if (mode != 0 && mode != 1) return nn_fail("nn_range_select: mode must be 0 (activations) or 1 (signed weights)%s", "");
    NN_SET_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    RangeSel* sel = (RangeSel*)(((uintptr_t)scratch + 15) & ~(uintptr_t)15);
    const int nsel = mode == 0 ? 1 : 2, first_domain = mode == 0 ? 0 : 1;
    const long long k0 = mode == 0 ? (long long)k_rank : 0;      // the caller's int(input.numel() * self.pctl / 100.)  (:249, quant.py:109)
    if (mode == 0 && (k0 < 1 || k0 > n)) return nn_fail("nn_range_select: percentile rank out of range%s (%lld)", "", k0);
    k_range_init<<<1, 256, 0, st>>>(sel, nsel, k0);
    NN_LAUNCH_OK();
    const int grid = nn_grid_for(n, 256, device, 4);
    for (int pass = 0; pass < 4; ++pass) {
        k_range_hist<<<grid, 256, 0, st>>>(x, n, sel, first_domain, nsel);
        NN_LAUNCH_OK();
        k_range_pick<<<1, 32, 0, st>>>(sel, nsel, pctl_percent, mode == 1 ? 1 : 0, out4, mode, min_value);
        NN_LAUNCH_OK();
    }
    return 0;
}

// ------------------------------------------------------------------ a4 AddNoise
__global__ void __launch_bounds__(256)
k_weight_noise(const float* __restrict__ w, float* __restrict__ out, int64_t n, float noise,
               const float* __restrict__ u_inject, nn_rng rng) {
    const NnRng s = nn_rng_load(rng);
    const int64_t ngroups = (n + 3) >> 2;
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < ngroups;
         g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i0 = g << 2;
        uint4 r = make_uint4(0, 0, 0, 0);
        if (!u_inject) r = nn_philox(s, (uint64_t)g);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (i0 + j < n) {
                float wv = w[i0 + j];
                float u = u_inject ? u_inject[i0 + j] : nn_usym(rr[j], noise);
                out[i0 + j] = __fadd_rn(wv, __fmul_rn(wv, u));      // output.add_(output * U)  (:297-298)
            }
        }
    }
}

extern "C" int nn_weight_noise_fwd(const float* w, float* out, int64_t n, float noise,
                                   const float* u_inject, nn_rng rng, int device, void* stream) {
    if (n <= 0) return 0;
    NN_SET_DEVICE(device);
    int threads = 256;
    int grid = nn_grid_for((n + 3) / 4, threads, device);
    k_weight_noise<<<grid, threads, 0, (cudaStream_t)stream>>>(w, out, n, noise, u_inject, rng);
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ tensor stats: max, max|.|, count>0
__global__ void k_stats_init(float* out3) {
    out3[0] = __int_as_float(0xff800000);   // -inf
    out3[1] = 0.f;
    out3[2] = 0.f;
}

__global__ void __launch_bounds__(256)
k_tensor_stats(const float* __restrict__ x, int64_t n, float* __restrict__ out3) {
    float mx = __int_as_float(0xff800000), amx = 0.f;
    unsigned int cnt = 0;
    const int64_t nvec = (((uintptr_t)x & 15) == 0) ? (n >> 2) : 0;
    const float4* xv = reinterpret_cast<const float4*>(x);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
        float4 v = xv[i];
        mx = fmaxf(fmaxf(mx, v.x), fmaxf(v.y, fmaxf(v.z, v.w)));
        amx = fmaxf(fmaxf(amx, fabsf(v.x)), fmaxf(fabsf(v.y), fmaxf(fabsf(v.z), fabsf(v.w))));
        cnt += (v.x > 0.f) + (v.y > 0.f) + (v.z > 0.f) + (v.w > 0.f);
    }
    for (int64_t i = (nvec << 2) + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * blockDim.x) {
        float v = x[i];
        mx = fmaxf(mx, v); amx = fmaxf(amx, fabsf(v)); cnt += (v > 0.f);
    }
    mx = nn_warp_max(mx); amx = nn_warp_max(amx);
    float c = nn_warp_sum((float)cnt);
    __shared__ float smx[8], samx[8], sc[8];
    int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { smx[w] = mx; samx[w] = amx; sc[w] = c; }
    __syncthreads();
    if (w == 0) {
        mx = (l < 8) ? smx[l] : __int_as_float(0xff800000);
        amx = (l < 8) ? samx[l] : 0.f;
        c = (l < 8) ? sc[l] : 0.f;
        mx = nn_warp_max(mx); amx = nn_warp_max(amx); c = nn_warp_sum(c);
        if (l == 0) {
            nn_atomic_max_float(out3 + 0, mx);
            nn_atomic_max_float(out3 + 1, amx);
            atomicAdd(out3 + 2, c);
        }
    }
}

extern "C" int nn_tensor_stats(const float* x, int64_t n, float* out3, int device, void* stream) {
    NN_SET_DEVICE(device);
    k_stats_init<<<1, 1, 0, (cudaStream_t)stream>>>(out3);
    if (n > 0) {
        int grid = nn_grid_for((n + 3) / 4, 256, device, 4);
        k_tensor_stats<<<grid, 256, 0, (cudaStream_t)stream>>>(x, n, out3);
        NN_LAUNCHED(1);
    }
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ a9 clamp + absmax
__global__ void k_zero1(float* p) { *p = 0.f; }

__global__ void __launch_bounds__(256)
k_clamp_absmax(float* __restrict__ w, int64_t n, float w_max, float* __restrict__ absmax_out) {
    float amx = 0.f;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float v = w[i];
        if (w_max > 0.f) {
            float c = fminf(fmaxf(v, -w_max), w_max);
            if (c != v) w[i] = c;
            v = c;
        }
        amx = fmaxf(amx, fabsf(v));
    }
    if (absmax_out) {
        amx = nn_warp_max(amx);
        __shared__ float s[8];
        int wi = threadIdx.x >> 5, l = threadIdx.x & 31;
        if (l == 0) s[wi] = amx;
        __syncthreads();
        if (wi == 0) {
            amx = (l < 8) ? s[l] : 0.f;
            amx = nn_warp_max(amx);
            if (l == 0) nn_atomic_max_float(absmax_out, amx);
        }
    }
}

extern "C" int nn_clamp_absmax(float* w, int64_t n, float w_max, float* absmax_out, int device, void* stream) {
    NN_SET_DEVICE(device);
    if (absmax_out) { k_zero1<<<1, 1, 0, (cudaStream_t)stream>>>(absmax_out); NN_LAUNCHED(1); }
    if (n > 0) {
        int grid = nn_grid_for(n, 256, device, 2);
        k_clamp_absmax<<<grid, 256, 0, (cudaStream_t)stream>>>(w, n, w_max, absmax_out);
    }
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ a7 unfused epilogue
// Philox mapping identical to the fused conv epilogue: element (m, n) -> group m*ceil(N/4) + n/4
// when (rows, cols) = (M, N) row-major; callers with NCHW tensors pass rows = numel/4.. see below.
// Here the tensor is treated as flat with groups of 4 consecutive elements: rows*cols elements.
__global__ void __launch_bounds__(256)
k_noise_epilogue(const float* __restrict__ y, const float* __restrict__ S, float* __restrict__ out, int64_t n,
                 const float* __restrict__ scale_dev, float current, const float* __restrict__ z_inject,
                 float* __restrict__ z_export, float* __restrict__ stats2, nn_rng rng) {
    const NnRng s = nn_rng_load(rng);
    const float coef = nn_noise_coef(*scale_dev, current);
    float sum_abs = 0.f, mx = __int_as_float(0xff800000);
    const int64_t ngroups = (n + 3) >> 2;
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < ngroups;
         g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i0 = g << 2;
        float z[4];
        if (z_inject) {
#pragma unroll
            for (int j = 0; j < 4; ++j) z[j] = (i0 + j < n) ? z_inject[i0 + j] : 0.f;
        } else {
            nn_normal4(s, (uint64_t)g, z);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (i0 + j < n) {
                float yv = y[i0 + j];
                float nz = __fmul_rn(z[j], nn_sigma(coef, S[i0 + j]));
                out[i0 + j] = __fadd_rn(yv, nz);
                if (z_export) z_export[i0 + j] = z[j];
                sum_abs += fabsf(nz);
                mx = fmaxf(mx, yv);
            }
        }
    }
    if (stats2) {
        sum_abs = nn_warp_sum(sum_abs);
        mx = nn_warp_max(mx);
        if ((threadIdx.x & 31) == 0) {
            atomicAdd(stats2 + 0, sum_abs);
            nn_atomic_max_float(stats2 + 1, mx);
        }
    }
}

extern "C" int nn_noise_epilogue(const float* y, const float* S, float* out, int64_t rows, int64_t cols,
                                 const float* scale_dev, float current, const float* z_inject,
                                 float* z_export, float* stats2, nn_rng rng, int device, void* stream) {
    int64_t n = rows * cols;
    if (n <= 0) return 0;
    if (!(current > 0.f)) return nn_fail("nn_noise_epilogue: current must be > 0%s", "");
    NN_SET_DEVICE(device);
    int grid = nn_grid_for((n + 3) / 4, 256, device);
    k_noise_epilogue<<<grid, 256, 0, (cudaStream_t)stream>>>(y, S, out, n, scale_dev, current, z_inject,
                                                              z_export, stats2, rng);
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ alternative noise models
__global__ void __launch_bounds__(256)
k_alt_noise(const float* __restrict__ y, float* __restrict__ out, int64_t n, int kind, float level,
            const float* __restrict__ absmax_dev, const float* __restrict__ rnd_inject, nn_rng rng) {
    const NnRng s = nn_rng_load(rng);
    const float amax = absmax_dev ? *absmax_dev : 0.f;
    const int64_t ngroups = (n + 3) >> 2;
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < ngroups;
         g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i0 = g << 2;
        float r[4];
        if (rnd_inject) {
#pragma unroll
            for (int j = 0; j < 4; ++j) r[j] = (i0 + j < n) ? rnd_inject[i0 + j] : 0.f;
        } else if (kind == 3 || kind == 4) {
            nn_normal4(s, (uint64_t)g, r);
        } else {
            uint4 q = nn_philox(s, (uint64_t)g);
            r[0] = nn_u01(q.x); r[1] = nn_u01(q.y); r[2] = nn_u01(q.z); r[3] = nn_u01(q.w);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (i0 + j >= n) continue;
            float yv = y[i0 + j], o;
            switch (kind) {
                case 1: o = yv + (r[j] * 2.f - 1.f) * (level * amax); break;               // :25-27
                case 2: o = yv * (level + r[j] * (1.f / level - level)); break;            // :29-31, :122-123
                case 3: o = yv + r[j] * (level * amax); break;                              // :33-36
                case 4: o = yv + r[j] * (level * yv); break;                                // :38-41
                default: o = yv + yv * ((r[j] * 2.f - 1.f) * level); break;                 // :17-20
            }
            out[i0 + j] = o;
        }
    }
}

extern "C" int nn_alt_noise(const float* y, float* out, int64_t n, int kind, float level,
                            const float* absmax_dev, const float* rnd_inject, nn_rng rng,
                            int device, void* stream) {
    if (n <= 0) return 0;
    if (kind < 1 || kind > 5) return nn_fail("nn_alt_noise: unknown kind%s %lld", "", kind);
    if ((kind == 1 || kind == 3) && !absmax_dev) return nn_fail("nn_alt_noise: absmax_dev required%s", "");
    NN_SET_DEVICE(device);
    int grid = nn_grid_for((n + 3) / 4, 256, device);
    k_alt_noise<<<grid, 256, 0, (cudaStream_t)stream>>>(y, out, n, kind, level, absmax_dev, rnd_inject, rng);
    NN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------ fused AdamW step + weight clamp + max|W|
// Replaces, in ONE launch for all parameter tensors, `optimizer.step()` of torch.optim.AdamW
// (noisynet.py:1163, :1520; decoupled weight decay, bias-corrected moments, no amsgrad) followed by
// `weight.data.clamp_(-w_max, w_max)` (noisynet.py:1527-1542) and the max|W| reduction the next forward's
// merged-DAC noise needs (hardware_model.py:47).  `grad_scale` folds the 1/world of the gradient mean.
struct AdamWP {
    nn_adamw_tensor t[NN_ADAMW_MAX_TENSORS];
    int count;
    float beta1, beta2, eps, grad_scale;
    int64_t* step_dev;                         // the step counter: read by every block, incremented by the last one
    int advance;                               // 0: a partial launch of the step (more tensors follow; the counter stays)
    unsigned* ctl;                             // per-device control words, see AW_*
    int first_block[NN_ADAMW_MAX_TENSORS];     // first 1024-element slab of each tensor in the flat block list
};
// control words: [0] arrival ticket (self-resetting); [4 + 4 * parity + {0,1,2}] the two bias-correction constants of a
// step and the step they belong to, double-buffered by step parity; [16 + 32 * parity + tensor] max|w| bits of the tensor
constexpr int AW_CONST = 4, AW_MAX = 16, AW_WORDS = 16 + 2 * 32;
static_assert(NN_ADAMW_MAX_TENSORS <= 32, "control block layout");

// blockIdx.x enumerates the 1024-element slabs of all tensors back to back (first_block[i] = first slab of tensor i).
// ONE launch per step, no memset nodes: the bias-correction constants of step s are prepared during step s - 1 (by its
// block 0, off the critical path: two fp64 pow); max|w| is an atomic max on the floats' bit patterns (order-independent,
// so deterministic) into the parity slot that the previous step's last block cleared; the last block to finish publishes
// the maxima, clears the other slot and advances the counter.
__global__ void __launch_bounds__(256)
k_adamw(const AdamWP p) {
    int ti = 0;
    while (ti + 1 < p.count && (int)blockIdx.x >= p.first_block[ti + 1]) ++ti;
    const nn_adamw_tensor t = p.t[ti];
    const int64_t base = (int64_t)((int)blockIdx.x - p.first_block[ti]) * blockDim.x * 4;
    __shared__ float s_red[8];
    __shared__ float s_c[2];
    __shared__ int s_par, s_last;
    if (threadIdx.x == 0) {
        const int64_t step = *p.step_dev + 1;
        const int par = (int)(step & 1);
        const float* cs = reinterpret_cast<const float*>(p.ctl + AW_CONST + 4 * par);
        const int tag = __float_as_int(p.beta1) ^ (__float_as_int(p.beta2) * 31);      // the slot is shared by every optimizer of the device
        if (__float_as_int(__ldcg(cs + 2)) == (int)step && __float_as_int(__ldcg(cs + 3)) == tag) {     // usual case: no fp64 pow
            s_c[0] = __ldcg(cs); s_c[1] = __ldcg(cs + 1);
        } else {                                                // first launch, or the counter was set from outside (checkpoint)
            s_c[0] = (float)(1.0 - pow((double)p.beta1, (double)step));
            s_c[1] = (float)sqrt(1.0 - pow((double)p.beta2, (double)step));
        }
        s_par = par;
        // constants of the NEXT step into the other slot (nobody reads it during this step): by the first launch of the step
        // that gets here -- with partial launches that is the early, large one, not the small one on the critical path
        float* nx = reinterpret_cast<float*>(p.ctl + AW_CONST + 4 * (par ^ 1));
        if (blockIdx.x == 0 && !(__float_as_int(__ldcg(nx + 2)) == (int)(step + 1) && __float_as_int(__ldcg(nx + 3)) == tag)) {
            nx[0] = (float)(1.0 - pow((double)p.beta1, (double)(step + 1)));
            nx[1] = (float)sqrt(1.0 - pow((double)p.beta2, (double)(step + 1)));
            nx[2] = __int_as_float((int)(step + 1));
            nx[3] = __int_as_float(tag);
        }
    }
    __syncthreads();
    const float step_size = (float)((double)t.lr / (double)s_c[0]), bc2s = s_c[1];
    const float decay = 1.0f - t.lr * t.weight_decay;
    const float om1 = 1.0f - p.beta1, om2 = 1.0f - p.beta2;
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int64_t i = base + (int64_t)j * blockDim.x + threadIdx.x;
        if (i < t.n) {
            const float g = t.g[i] * p.grad_scale;
            float w = t.p[i] * decay;                                  // param.mul_(1 - lr * wd)
            float m = t.m[i];
            m = m + om1 * (g - m);                                     // exp_avg.lerp_(grad, 1 - beta1)
            float v = t.v[i] * p.beta2 + om2 * g * g;                  // exp_avg_sq.mul_(b2).addcmul_(g, g, 1 - b2)
            const float denom = sqrtf(v) / bc2s + p.eps;
            w = w - step_size * (m / denom);                           // param.addcdiv_(exp_avg, denom, -step_size)
            if (t.clamp > 0.f) w = fminf(fmaxf(w, -t.clamp), t.clamp);
            t.p[i] = w; t.m[i] = m; t.v[i] = v;
            amax = fmaxf(amax, fabsf(w));
        }
    }
    const int wi = threadIdx.x >> 5, l = threadIdx.x & 31;
    amax = nn_warp_max(amax);
    if (l == 0) s_red[wi] = amax;
    __syncthreads();
    if (threadIdx.x == 0) {
        float bm = s_red[0];
#pragma unroll
        for (int w = 1; w < 8; ++w) bm = fmaxf(bm, s_red[w]);
        unsigned* mx = p.ctl + AW_MAX + 32 * s_par;
        if (t.absmax_out && bm > 0.f) atomicMax(mx + ti, __float_as_uint(bm));      // bm >= 0: bit order == value order
        __threadfence();
        s_last = atomicAdd(p.ctl, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if ((int)threadIdx.x < p.count) {
        unsigned* mx = p.ctl + AW_MAX + 32 * s_par;
        if (p.t[threadIdx.x].absmax_out) *p.t[threadIdx.x].absmax_out = __uint_as_float(__ldcg(mx + threadIdx.x));
        p.ctl[AW_MAX + 32 * (s_par ^ 1) + threadIdx.x] = 0u;         // the next step's slot
        mx[threadIdx.x] = 0u;                                        // (and this one, for a step counter set from outside)
    }
    if (threadIdx.x == 0) { p.ctl[0] = 0u; if (p.advance) *p.step_dev += 1; }
}

extern "C" int nn_adamw_step(const nn_adamw_tensor* tensors, int count, float beta1, float beta2, float eps,
                             float grad_scale, int64_t* step_dev, int device, void* stream) {
    return nn_adamw_step_part(tensors, count, beta1, beta2, eps, grad_scale, step_dev, 1, device, stream);
}

extern "C" int nn_adamw_step_part(const nn_adamw_tensor* tensors, int count, float beta1, float beta2, float eps,
                                  float grad_scale, int64_t* step_dev, int advance, int device, void* stream) {
    if (count <= 0) return 0;
    if (count > NN_ADAMW_MAX_TENSORS) return nn_fail("nn_adamw_step: too many tensors%s (%lld)", "", count);
    if (!step_dev) return nn_fail("nn_adamw_step: step_dev missing%s", "");
    NN_SET_DEVICE(device);
    AdamWP p;
    p.count = count; p.beta1 = beta1; p.beta2 = beta2; p.eps = eps; p.grad_scale = grad_scale; p.step_dev = step_dev;
    p.advance = advance ? 1 : 0;
    if (device < 0 || device >= 64) return nn_fail("nn_adamw_step: bad device%s", "");
    int blocks = 0;
    for (int i = 0; i < count; ++i) {
        p.t[i] = tensors[i];
        p.first_block[i] = blocks;
        blocks += (int)((tensors[i].n + 1023) / 1024);
    }
    if (blocks == 0) return nn_fail("nn_adamw_step: empty tensors%s", "");
    static unsigned* ctl[64] = {nullptr};        // allocated by the first (uncaptured) step of a device
    if (!ctl[device]) {
        NN_CUDA_OK(cudaMalloc(&ctl[device], AW_WORDS * sizeof(unsigned)));
        NN_CUDA_OK(cudaMemset(ctl[device], 0, AW_WORDS * sizeof(unsigned)));
    }
    p.ctl = ctl[device];
    k_adamw<<<blocks, 256, 0, (cudaStream_t)stream>>>(p);
    NN_LAUNCH_OK();
    return 0;
}
