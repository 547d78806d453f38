// Shared device/host helpers for the noisynet_b200 kernels (sm_90a).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/noisynet_b200.h"

// ---------------------------------------------------------------- error plumbing
extern thread_local char g_nn_err[512];

static inline int nn_fail(const char* fmt, const char* a = "", long long b = 0) {
    snprintf(g_nn_err, sizeof(g_nn_err), fmt, a, b);
    return 1;
}

#define NN_CUDA_OK(expr)                                                              \
    do {                                                                              \
        cudaError_t _e = (expr);                                                      \
        if (_e != cudaSuccess) {                                                      \
            snprintf(g_nn_err, sizeof(g_nn_err), "%s:%d %s -> %s", __FILE__, __LINE__, \
                     #expr, cudaGetErrorString(_e));                                  \
            return 2;                                                                 \
        }                                                                             \
    } while (0)

// Entry points take `device` per call: switch to it for the duration of the call and restore the caller's current
// device on return (a library must not leave torch's "current device" changed behind the caller's back).
struct NnDeviceGuard {
    int prev;
    cudaError_t err;
    explicit NnDeviceGuard(int dev) : prev(-1) {
        int cur = -1;
        err = cudaGetDevice(&cur);
        if (err == cudaSuccess && cur != dev) {
            err = cudaSetDevice(dev);
            if (err == cudaSuccess) prev = cur;
        }
    }
    ~NnDeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
#define NN_SET_DEVICE(dev) NnDeviceGuard _nn_dev_guard(dev); NN_CUDA_OK(_nn_dev_guard.err)

// Function attributes (opt-in dynamic shared memory) are PER DEVICE: run `body` once per device of this process.
#define NN_ONCE_PER_DEVICE(body)                                   \
    do {                                                           \
        static bool _nn_done[64] = {false};                        \
        int _nn_d = 0;                                             \
        cudaGetDevice(&_nn_d);                                     \
        if (_nn_d < 0 || _nn_d >= 64 || !_nn_done[_nn_d]) {        \
            body;                                                  \
            if (_nn_d >= 0 && _nn_d < 64) _nn_done[_nn_d] = true;  \
        }                                                          \
    } while (0)
extern unsigned long long g_nn_launches;
#define NN_LAUNCH_OK() do { ++g_nn_launches; NN_CUDA_OK(cudaGetLastError()); } while (0)
#define NN_LAUNCHED(n) (g_nn_launches += (n))

static inline int nn_num_sms(int device) {
    static int cached[64] = {0};
    if (device < 0 || device >= 64) return 148;
    if (!cached[device]) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || v <= 0) v = 148;
        cached[device] = v;
    }
    return cached[device];
}

// ---------------------------------------------------------------- Philox4x32-10
// key = seed, counter = (offset_lo, offset_hi, group_lo, group_hi).  Spec mirrored by
// oracle/noisynet_oracle.py::philox4x32_10 (tests compare bit-exactly).
struct NnRng {
    uint32_t k0, k1, c0, c1;
};

__device__ __forceinline__ NnRng nn_rng_load(const nn_rng& r) {
    uint64_t off = r.offset;
    if (r.offset_dev) off += *r.offset_dev;
    NnRng s;
    s.k0 = (uint32_t)r.seed;
    s.k1 = (uint32_t)(r.seed >> 32);
    s.c0 = (uint32_t)off;
    s.c1 = (uint32_t)(off >> 32);
    return s;
}

__device__ __forceinline__ uint4 nn_philox(const NnRng& s, uint64_t group) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    uint32_t c0 = s.c0, c1 = s.c1, c2 = (uint32_t)group, c3 = (uint32_t)(group >> 32);
    uint32_t k0 = s.k0, k1 = s.k1;
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
        uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
        uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += W0; k1 += W1;
    }
    return make_uint4(c0, c1, c2, c3);
}

// u in [0,1), 24 bits, exact in fp32
__device__ __forceinline__ float nn_u01(uint32_t r) { return (float)(r >> 8) * 5.9604644775390625e-08f; }

// U[-s, s): fl(fl(u * 2s) - s), two explicit roundings (no FMA contraction)
__device__ __forceinline__ float nn_usym(uint32_t r, float s) {
    return __fadd_rn(__fmul_rn(nn_u01(r), __fmul_rn(2.0f, s)), -s);
}

// Box-Muller on one pair, MUFU-only transcendentals (the conv epilogues are instruction-bound on the noise:
// ~32.5 M normals per NoisyNet step at batch 512).  u1 = fma(r, 2^-32, 2^-33) in (0,1];
// rad = sqrt(-2 ln u1) via lg2.approx / sqrt.approx; theta = fma(u2, 2pi, -pi), sin/cos.approx.
// Absolute error vs an exact evaluation: ~1e-6 typical, <= ~2e-3 for the rare rad < 1e-3 (P ~ 5e-7).
__device__ __forceinline__ float nn_sqrt_approx(float x) {
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float nn_lg2_approx(float x) {      // x is never subnormal here: no range fix-up code
    float r;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void nn_box_muller(uint32_t ra, uint32_t rb, float& z0, float& z1) {
    const float u1 = fmaf(__uint2float_rn(ra), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
    const float u2 = nn_u01(rb);
    const float rad = nn_sqrt_approx(-1.3862943611198906f * nn_lg2_approx(u1));
    const float th = fmaf(u2, 6.2831853071795865f, -3.14159265358979324f);
    z0 = rad * __cosf(th);
    z1 = rad * __sinf(th);
}

__device__ __forceinline__ void nn_normal4(const NnRng& s, uint64_t group, float z[4]) {
    uint4 r = nn_philox(s, group);
    nn_box_muller(r.x, r.y, z[0], z[1]);
    nn_box_muller(r.z, r.w, z[2], z[3]);
}

// ---------------------------------------------------------------- float atomics
__device__ __forceinline__ void nn_atomic_max_float(float* addr, float v) {
    // valid for any mix of signs: ordered-int trick
    if (v >= 0.0f) atomicMax((int*)addr, __float_as_int(v));
    else atomicMin((unsigned int*)addr, __float_as_uint(v));
}

__device__ __forceinline__ float nn_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float nn_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// sigma = sqrt(0.1 * (scale / I) * S) with the reference's rounding order
// (hardware_model.py:59: torch.sqrt(0.1 * (w_max / I) * sigmas)).
__device__ __forceinline__ float nn_noise_coef(float scale, float current) {
    return __fmul_rn(0.1f, __fdiv_rn(scale, current));
}
__device__ __forceinline__ float nn_sigma(float coef, float S) { return nn_sqrt_approx(__fmul_rn(coef, S)); }

static inline void nn_out_hw(const nn_conv_geom& g, int& OH, int& OW) {
    OH = (g.H + 2 * g.pad - g.KH) / g.stride + 1;
    OW = (g.W + 2 * g.pad - g.KW) / g.stride + 1;
}

// ---- BatchNorm batch statistics from fixed-order partial sums (shared by the stage kernels and the conv1 epilogue fusion)
struct BnFinP {
    double count;
    float eps, momentum;
    float *mean, *invstd, *running_mean, *running_var, *xmax_out;
    int eval_mode;
};
// partial[s * stride + {0, 1}] = (sum, sum of squares) of slice s of channel c.  mean / invstd (biased var) + running
// statistics update (momentum, unbiased var); eval_mode: noisynet.py:1560-1567
__device__ __forceinline__ void bn_finalize_channel(const double* partial, int splits, int64_t stride, int c, const BnFinP& f) {
    if (f.eval_mode) {          // model.eval(): normalise with the running statistics, update nothing
        f.mean[c] = f.running_mean[c];
        f.invstd[c] = (float)(1.0 / sqrt((double)f.running_var[c] + (double)f.eps));
        return;
    }
    double s1 = 0, s2 = 0;
    for (int s = 0; s < splits; ++s) { s1 += __ldcg(partial + (int64_t)s * stride); s2 += __ldcg(partial + (int64_t)s * stride + 1); }
    const double m = s1 / f.count;
    double var = s2 / f.count - m * m;
    if (var < 0) var = 0;
    f.mean[c] = (float)m;
    f.invstd[c] = (float)(1.0 / sqrt(var + (double)f.eps));
    if (f.running_mean) {
        const double unb = f.count > 1 ? var * f.count / (f.count - 1) : var;
        f.running_mean[c] = (float)((1.0 - f.momentum) * f.running_mean[c] + f.momentum * m);
        f.running_var[c] = (float)((1.0 - f.momentum) * f.running_var[c] + f.momentum * unb);
    }
}
