/*
 * noisynet_b200 -- C ABI of the H100 (sm_90a) NoisyNet hot path.
 *
 * The reference (michaelklachko/NoisyNet) is pure Python on PyTorch and has no FFI of its
 * own; its "operator API" for this path is the set of Python names the drivers import
 * (noisynet.py:14, models/resnet.py:9-11, models/mobilenet.py:9, main.py:37).  This header
 * is the boundary a binding for those names sits on: each entry point cites the reference
 * code it replaces (file:line in the reference tree).  Plain pointers and sizes only; all
 * pointers are DEVICE pointers unless stated; all tensors are fp32, contiguous, NCHW
 * (the reference's layout, SURVEY.md section 8a).
 *
 * Every function returns 0 on success, non-zero on error (message via nn_last_error()).
 * Kernels are enqueued on `stream` (a cudaStream_t passed as void*) of device `device`;
 * nothing synchronises the host.  All entry points are re-entrant per device.
 */
#ifndef NOISYNET_B200_H
#define NOISYNET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NN_ABI_VERSION 18

/* ---- common ---------------------------------------------------------------------- */

/* Philox4x32-10 stream: key = seed, counter = (offset + *offset_dev, group index).
 * offset_dev (device uint64, may be NULL) lets a captured CUDA graph advance the stream
 * without re-capturing (see nn_rng_advance).  Replaces the global torch generator the
 * reference draws from (hardware_model.py:59,81,161,297). */
typedef struct nn_rng {
    uint64_t seed;
    uint64_t offset;
    const uint64_t* offset_dev;
} nn_rng;

const char* nn_last_error(void);
int nn_abi_version(void);
/* number of kernels this library has launched in this process (host-side counter). */
uint64_t nn_launch_count(void);
/* sm_count / compute capability of `device`; fails unless the device is sm_90 (H100). */
int nn_device_info(int device, int* sm_count, int* cc_major, int* cc_minor);
/* *offset_dev += inc (one thread); graph-capturable. */
int nn_rng_advance(uint64_t* offset_dev, uint64_t inc, int device, void* stream);

/* ---- a1/a2: UniformQuantize  (hardware_model.py:133-183, quant.py:12-61) ------------- */

/* y = rne(clamp((x-min)/scale + U(-stochastic,stochastic), 0, 2^bits-1)) * scale + min,
 * scale = max((max-min)/(2^bits-1), 1e-6)  (:148-170).  u_inject (optional, device, n floats
 * already in [-stochastic, stochastic)) replaces the Philox draw -- parity/test hook.
 * In place allowed (y == x) -- the reference's `inplace=True` (:141-144). */
int nn_quantize_fwd(const float* x, float* y, int64_t n, int bits, double min_value,
                    double max_value, float stochastic, const float* u_inject, nn_rng rng,
                    int device, void* stream);
/* Saturated STE (:176-183): gx = gy * 1[min <= x <= max].  Does NOT modify gy. */
int nn_quantize_bwd(const float* x, const float* gy, float* gx, int64_t n, double min_value,
                    double max_value, int device, void* stream);

/* ---- a3 on the device: QuantMeasure range selection (hardware_model.py:232-259) without host syncs -----------
 * mode 0 (activations, :240-259): out4[0] = kthvalue(x, k_rank), k_rank = the caller's int(n * pctl / 100) (hardware_model.py:249)
 *        or int(n * pctl) (quant.py:109)  (what the script appends to running_list),
 *        out4[1] = max(x); the quantisation range of THIS call is out4[2..3] = {min_value, max(x)}  (:253).
 * mode 1 (signed weights, :232-239): out4[0] = running_min = -kthvalue(|x[x<0]|, int(count * pctl_percent / 100)),
 *        out4[1] = running_max = kthvalue(x[x>0], ...); range out4[2..3] = {running_min, running_max}.
 * Exact (radix select on the floats' ordered integer image), deterministic, graph-capturable; `scratch` is
 * nn_range_scratch_bytes() of device memory.  out4 + 2 is the `range_dev` of the two entry points below. */
int64_t nn_range_scratch_bytes(void);
int nn_range_select(const float* x, int64_t n, int64_t k_rank, double pctl_percent, int mode, double min_value, float* out4,
                    void* scratch, int device, void* stream);
/* nn_quantize_fwd / nn_quantize_bwd with the range {min, max} read from device memory (scale = max((max-min)/(2^b-1), 1e-6)
 * evaluated in doubles on the device, as the host does at :148-151). */
int nn_quantize_fwd_dev(const float* x, float* y, int64_t n, int bits, const float* range_dev, float stochastic,
                        const float* u_inject, nn_rng rng, int device, void* stream);
int nn_quantize_bwd_dev(const float* x, const float* gy, float* gx, int64_t n, const float* range_dev, int device, void* stream);

/* ---- a4: AddNoise  (hardware_model.py:291-307) ------------------------------------- */
/* out = w + w * U(-noise, noise). */
int nn_weight_noise_fwd(const float* w, float* out, int64_t n, float noise,
                        const float* u_inject, nn_rng rng, int device, void* stream);

/* ---- reductions used by the noise model (hardware_model.py:44-47, :88) ------------- */
/* out3[0] = max(x), out3[1] = max|x|, out3[2] = count(x > 0) (as float).  Overwrites out3. */
int nn_tensor_stats(const float* x, int64_t n, float* out3, int device, void* stream);

/* ---- a9: weight clamp  (noisynet.py:1527-1542, main.py:953-957) -------------------- */
/* w = clamp(w, -w_max, w_max) in place (skipped if w_max <= 0); absmax_out (optional device
 * scalar) receives max|w| after the clamp, which the next forward's merged-DAC noise needs
 * (hardware_model.py:47). */
int nn_clamp_absmax(float* w, int64_t n, float w_max, float* absmax_out, int device, void* stream);

/* ---- optimizer step adjacent to a9 (noisynet.py:1163 AdamW, :1520 optimizer.step(), :1527-1542 clamp) --
 * One launch for all parameter tensors: torch.optim.AdamW update (decoupled weight decay, bias-corrected,
 * no amsgrad) with grads pre-multiplied by grad_scale (the 1/world of the gradient mean), then
 * clamp(+-clamp) if clamp > 0, then absmax_out[0] = max|p| (optional).  *step_dev is incremented first and
 * used as the step count (device-resident: CUDA-graph replay safe).  `tensors` is a HOST array. */
#define NN_ADAMW_MAX_TENSORS 24
typedef struct nn_adamw_tensor {
    float* p; const float* g; float* m; float* v;
    int64_t n;
    float lr, weight_decay, clamp;
    float* absmax_out;
} nn_adamw_tensor;
int nn_adamw_step(const nn_adamw_tensor* tensors, int count, float beta1, float beta2, float eps,
                  float grad_scale, int64_t* step_dev, int device, void* stream);
/* The same update for a SUBSET of the step's tensors: launches with advance = 0 use step count *step_dev + 1 and leave
 * the counter alone, the step's last launch passes advance = 1 (nn_adamw_step == advance 1).  Lets the engine update
 * the layers whose gradients are final early (and already exchanged) under the rest of the backward pass; launches of
 * one step must not overlap each other (they share the per-device control words). */
int nn_adamw_step_part(const nn_adamw_tensor* tensors, int count, float beta1, float beta2, float eps,
                       float grad_scale, int64_t* step_dev, int advance, int device, void* stream);

/* ---- a7 (unfused form): y_noisy = y + z * sqrt(0.1 * (scale / I) * S) --------------- */
/* hardware_model.py:59 / :81-83 / :125.  scale_dev: device scalar (max|W| merged DAC,
 * max(x) external DAC).  z_inject / z_export / optional.  stats2 (optional, device[2]) is
 * ACCUMULATED: [0] += sum|noise| ; [1] = max(stats[1], max(y))  (for nsr, :87). */
int nn_noise_epilogue(const float* y, const float* S, float* out, int64_t rows, int64_t cols,
                      const float* scale_dev, float current, const float* z_inject,
                      float* z_export, float* stats2, nn_rng rng, int device, void* stream);

/* Alternative output-noise models (hardware_model.py:17-41, :122-125).
 * kind: 1 uniform_ind, 2 uniform_dep (multiplicative), 3 normal_ind, 4 normal_dep,
 *       5 distort_act.  absmax_dev: device scalar max|y| (kinds 1 and 3). */
int nn_alt_noise(const float* y, float* out, int64_t n, int kind, float level,
                 const float* absmax_dev, const float* rnd_inject, nn_rng rng,
                 int device, void* stream);

/* ---- a5/a6/a7 fused: noisy conv / linear forward ------------------------------------ */

typedef struct nn_conv_geom {
    int32_t B, Cin, H, W;        /* input  [B, Cin, H, W]   (linear: H = W = 1)            */
    int32_t Cout, KH, KW;        /* weight [Cout, Cin, KH, KW]                             */
    int32_t stride, pad;         /* dilation 1, groups 1                                   */
} nn_conv_geom;                  /* output [B, Cout, OH, OW], OH = (H + 2 pad - KH)/stride + 1 */

enum { NN_NOISE_NONE = 0, NN_NOISE_MERGED = 1, NN_NOISE_EXTERNAL = 2 };
enum { NN_PREC_FP32 = 0,      /* CUDA-core fp32 FMA (reference arithmetic, any geometry)  */
       NN_PREC_TF32 = 1,      /* reserved: rejected (not implemented)                     */
       NN_PREC_BF16 = 2 };    /* wgmma bf16 x bf16, fp32 accumulate; exact when the      
                                 operands are integer codes (a_code_scale > 0)             */

typedef struct nn_conv_fwd_args {
    nn_conv_geom g;
    const float* x;          /* layer input (after any activation quantizer)               */
    const float* w_eff;      /* weight of the main contraction (quantized / noised / raw).
                                NULL (with noise_mode > 0) = noise-only mode: `y` is an INPUT
                                (the clean output computed earlier) and only the sigma^2
                                contraction + epilogue run -- the two-call flow of
                                noisynet.py:398 + :415                                     */
    const float* w_raw;      /* raw parameter for the sigma^2 contraction (noise_mode > 0) */
    const float* bias;       /* [Cout] or NULL                                             */
    float* y;                /* clean output  F.conv2d / F.linear  (hardware_model.py:362, :421) */
    float* y_noisy;          /* y + sigma * z (hardware_model.py:125); NULL iff noise_mode == 0 */
    int32_t noise_mode;      /* NN_NOISE_*                                                 */
    float current;           /* I_max in nA (args.layer_currents[layer_num])               */
    const float* scale_dev;  /* device scalar: max|w_raw| (merged) or max(x) (external)     */
    const float* z_inject;   /* optional [B,Cout,OH,OW] N(0,1) draws replacing Philox       */
    float* z_export;         /* optional: the z actually used                              */
    float* sigma_export;     /* optional: sigma                                            */
    nn_rng rng;
    float* stats;            /* optional device[3], ACCUMULATED: [0] += sum conv(x,|W|),
                                [1] += sum|noise|, [2] = max(., max(y)) (:55-57, :77-79, :87) */
    int32_t precision;       /* NN_PREC_*                                                  */
    /* Integer-code mode (NN_PREC_BF16): x holds k_a * a_scale (k_a integer in [0, 2^bits)),
     * w_eff holds c_w * w_scale (c_w odd/any integer): the operands fed to the tensor core
     * are the integers themselves (exact in bf16) and the epilogue multiplies by
     * a_scale * w_scale.  0 disables. */
    float a_code_scale, w_code_scale;
    void* workspace;         /* device scratch for packed operands (nn_conv_workspace_bytes) */
    int64_t workspace_bytes;
    const void* x_packed;    /* optional (tensor-core precisions): the input already packed as NHWC bf16
                                [B,H,W,ceil8(Cin)] (codes if a_code_scale > 0), e.g. by nn_stage_fwd;
                                `x` is then ignored and the pack kernel is skipped.  A launch on
                                NN_PACK_SHIFT weights (w_packed_layout, or nn_conv_pack_layout when
                                the weights are not packed) takes the ROW-PLANE image instead
                                (nn_conv_shift_planes_bytes, nn_input_quant_pack_rows)                */
    const void* w_packed;    /* optional: weights already packed by nn_prepare_weights (mode 0, same
                                noise_mode / stats choice); w_eff may then be NULL, w_code_scale must be
                                the quantizer's s/2                                                   */
    int32_t w_packed_layout; /* NN_PACK_*: the layout `w_packed` was prepared in (nn_wprep_job.layout)      */
    float* pooled_out;       /* optional, with argmax_out: fused MaxPool2d(2,2) (noisynet.py:419) of the (noisy)
                                output, [B,Cout,OH/2,OW/2]; y / y_noisy are then NOT written.  Served where
                                nn_conv_pool_fusable() says so (the shift kernel on a 32-wide input grid).          */
    uint8_t* argmax_out;     /* window position 0..3 of the first maximum in row-major order (nn.MaxPool2d)      */
    /* optional, with pooled_out: the BatchNorm that follows the pool (noisynet.py:419-431) gets its batch statistics
     * from the same launch -- per-CTA partial sums of the pooled values, finalized by the last CTA (fixed order:
     * deterministic).  bn_mean != NULL selects it; the stage that follows is then called with stats_ready = 1. */
    float* bn_mean;          /* out [Cout] batch mean   (eval: the running mean)                                   */
    float* bn_invstd;        /* out [Cout] 1 / sqrt(biased var + eps)                                               */
    float* bn_running_mean;  /* [Cout] updated with momentum (unbiased var), or NULL                                */
    float* bn_running_var;
    float bn_eps, bn_momentum;
    int32_t bn_eval_mode;    /* 1: normalise with the running statistics, update nothing                            */
    void* bn_scratch;        /* nn_conv_bn_scratch_bytes(Cout) bytes, zeroed once by the caller                     */
    float* zero_out;         /* optional device float set to 0 by the launch (the max-accumulator of the next stage) */
} nn_conv_fwd_args;
int64_t nn_conv_bn_scratch_bytes(int Cout);
/* bn_mean is also served for LINEAR layers whose launch is split over K (fully connected layers at training batch sizes:
 * the split-K epilogue adds the per-channel sums; BatchNorm1d, noisynet.py:540-546): 1 if this geometry qualifies.  There
 * bn_scratch is nn_stage_scratch_bytes(Cout) bytes, zeroed once, and belongs to this launch alone: the split-K epilogue
 * lays its partial sums and counters out differently from the stage kernels, so it must not share their scratch. */
int nn_conv_linear_bn_fusable(const nn_conv_geom* g, int32_t noise_mode, int32_t precision, int device);

/* Packed-weight layouts.  NN_PACK_TILED: 128B-swizzled [n-tile][k-block] shared-memory images (every geometry).
 * NN_PACK_SHIFT: [kh][plane][row][8] image of the persistent shift-GEMM forward kernel (k = kw * Cin + c of kernel
 * row kh, 8 per plane, P = 2 ceil(KW Cin / 16) planes; nn_prepare_weights packs square kernels, KH = KW =
 * sqrt(KHW)), served for stride-1 unpadded layers with Cin <= 8 (the first layer, noisynet.py:344): ask
 * nn_conv_pack_layout which one the forward of a geometry prefers; nn_noisy_conv_fwd rejects a layout it cannot
 * serve (bias / stats / export requests need NN_PACK_TILED). */
#define NN_PACK_TILED 0
#define NN_PACK_SHIFT 1
/* NN_PACK_TMA: [n-tile][tap][stage][CTA rank] image of the persistent CTA-pair kernel whose activations arrive by
 * im2col-mode tensor-map copies (cp.async.bulk.tensor, cuTensorMapEncodeIm2col): conv layers (output larger than 1x1,
 * more than 8 input channels, square kernels) on the lean path (no bias / statistics / exports / clean-output copy). */
#define NN_PACK_TMA 2
int nn_conv_pack_layout(const nn_conv_geom* g, int32_t noise_mode, int32_t precision);
/* Bytes of the row-plane input image of an NN_PACK_SHIFT forward: P = 2 ceil(KW Cin / 16) planes [plane][B][H][W][8]
 * bf16; element j of plane q at pixel (b, h, w) is x[b, c, h, w + kw] for kw * Cin + c = 8 q + j, zero where
 * w + kw >= W or 8 q + j >= KW * Cin.  0 for Cin outside 1..8. */
int64_t nn_conv_shift_planes_bytes(const nn_conv_geom* g);
/* Layout the dgrad of a geometry prefers for its (transposed, tap-flipped) weight image: NN_PACK_TMA or NN_PACK_TILED. */
int nn_conv_dgrad_pack_layout(const nn_conv_geom* g, int32_t precision);
/* Test hook: enable = 0/1 switches the TMA-im2col path off/on (< 0: query); returns the previous setting. */
int nn_debug_tma_enable(int enable);
/* 1 if nn_noisy_conv_fwd can fuse the 2x2 max pool that follows the layer (pooled_out / argmax_out). */
int nn_conv_pool_fusable(const nn_conv_geom* g, int32_t noise_mode, int32_t precision);
/* Test hook: enable = 0/1 switches the shift-GEMM path off/on (< 0: query); returns the previous setting. */
int nn_debug_shift_enable(int enable);

int64_t nn_conv_workspace_bytes(const nn_conv_geom* g, int32_t precision);
/* 1 if (geometry, precision) is served for which = 0 forward / 1 dgrad / 2 wgrad.  NN_PREC_FP32 serves
 * everything; the tensor-core precisions serve a subset (callers pick NN_PREC_FP32 for the rest). */
int nn_conv_supported(const nn_conv_geom* g, int32_t precision, int32_t which);
/* Test/debug hook: synchronises `device` and returns the tensor-core pipeline watchdog flag (0 = ok);
 * reset != 0 clears it. */
int nn_debug_error_flag(int device, int reset);
/* Measurement hook: enable = 1/0 brackets the main tensor-core forward kernel (not the operand packs) with CUDA
 * events on its launch stream; enable < 0 synchronises on them and returns the last elapsed ms (-1: none). */
float nn_debug_main_kernel_ms(int enable);
/* Debug (env NN_UMMA_DEBUG=1): per-CTA clock64 phase stamps [cta][8] of the last tensor-core forward launch. */
int nn_debug_cta_timeline(long long* host_out, int max_ctas);
int nn_noisy_conv_fwd(const nn_conv_fwd_args* a, int device, void* stream);

/* ---- a10: backward of a5/a6 with the saturated STE fused --------------------------- */
/* dgrad: gx = conv_transpose(gy, w_eff) * 1[x_lo <= x_pre <= x_hi]   (mask optional: x_pre
 * NULL disables; it is the STE of the activation quantizer in front of the layer,
 * hardware_model.py:176-183). */
typedef struct nn_conv_dgrad_args {
    nn_conv_geom g;
    const float* gy;         /* [B,Cout,OH,OW] */
    const float* w_eff;
    float* gx;               /* [B,Cin,H,W] */
    const float* x_pre; double x_lo, x_hi;
    int32_t precision;
    float w_code_scale;      /* > 0: w_eff holds integer codes * w_code_scale (exact bf16 operand), see fwd */
    void* workspace; int64_t workspace_bytes;
    const void* gy_packed;   /* optional: grad_output already NHWC bf16 [B,OH,OW,ceil8(Cout)] (nn_stage_bwd) */
    const void* w_packed;    /* optional: weights already packed by nn_prepare_weights (mode 1)        */
    int32_t w_packed_layout; /* NN_PACK_*: the layout `w_packed` was prepared in (nn_conv_dgrad_pack_layout)  */
} nn_conv_dgrad_args;
int nn_noisy_conv_dgrad(const nn_conv_dgrad_args* a, int device, void* stream);
/* dgrad of a layer whose grad_output images fit in shared memory (k_dgrad_planes): each image is loaded once as
 * zero-padded row planes and all taps read it there, instead of one im2col tile per (pixel tile, tap).  Served when
 * nn_conv_dgrad_planes_ok(g): stride 1, square kernel, pad < K, Cout <= 128, Cin <= 120 (one n-tile), and
 * H x (OW + 2 (K - 1 - pad)) <= 256 (NoisyNet's conv2; not the ResNet 3x3 layers).  Needs precision NN_PREC_BF16,
 * gy_packed (NHWC, ceil8(Cout) channels), w_packed in NN_PACK_TMA (nn_prepare_weights mode 1) and no x_pre.  gx is
 * bit-identical to nn_noisy_conv_dgrad's on the same packed operands (the same k16 groups in the same order). */
int nn_conv_dgrad_planes_ok(const nn_conv_geom* g);
int nn_conv_dgrad_planes(const nn_conv_dgrad_args* a, int device, void* stream);

/* wgrad: gw = (gy^T * im2col(x)) * 1[w_lo <= w_raw <= w_hi]  (mask optional: the STE of the
 * weight quantizer, hardware_model.py:343 + :176-183).  Deterministic split-K. */
typedef struct nn_conv_wgrad_args {
    nn_conv_geom g;
    const float* gy;
    const float* x;          /* the layer input used in the forward */
    float* gw;               /* [Cout,Cin,KH,KW] */
    const float* w_raw; double w_lo, w_hi;
    int32_t precision;
    float a_code_scale;      /* > 0: x holds integer codes * a_code_scale (exact bf16 operand), see fwd */
    void* workspace; int64_t workspace_bytes;
    const void* x_packed;    /* optional: layer input already NHWC bf16 [B,H,W,ceil8(Cin)] (codes if a_code_scale > 0) */
    const void* gy_packed;   /* optional: grad_output already packed, in the layout named below           */
    int32_t gy_packed_layout;/* NN_PACK_TILED: NHWC bf16 [B,OH,OW,ceil8(Cout)].  NN_PACK_SHIFT: the planes
                                layout [ceil(Cout/8)][P][8] bf16 on the INPUT pixel grid -- element (b,n,oh,ow)
                                at plane n/8, pixel (b*H + oh)*W + ow, zeros at every other pixel; P = B*H*W
                                rounded up to 128 (nn_conv_gy_planes_bytes).  nn_stage_bwd writes it directly */
} nn_conv_wgrad_args;
int64_t nn_conv_wgrad_workspace_bytes(const nn_conv_geom* g, int32_t precision, int device);
/* NN_PACK_SHIFT if the weight gradient of this geometry is served by the shift-GEMM kernel (stride 1, no
 * padding, Cin <= 8, Cout <= 128: both operands are read in place through shifted descriptors, nothing is
 * gathered), else NN_PACK_TILED.  Un-packed callers (gy fp32) are routed automatically. */
int nn_conv_wgrad_pack_layout(const nn_conv_geom* g, int32_t precision, int device);
int64_t nn_conv_gy_planes_bytes(const nn_conv_geom* g);
int nn_noisy_conv_wgrad(const nn_conv_wgrad_args* a, int device, void* stream);

/* ---- weight preparation for a whole step in one launch ------------------------------------------------
 * Each job packs one layer's weights into the tensor-core operand image: mode 0 = forward rows
 * [quantized main | g(|w_raw|) | colsum |w_raw|], mode 1 = transposed, tap-flipped rows for dgrad.  With
 * q_bits > 0 the weight quantizer (hardware_model.py:323, :343: range [-q_hi, q_hi], stochastic rounding)
 * runs in registers; jobs sharing `rng` (or u_inject) quantize identically.  `jobs` is a HOST array (<= 8). */
typedef struct nn_wprep_job {
    const float* w_raw;      /* [Cout,Cin,KH,KW] fp32 parameter                                       */
    int32_t Cout, Cin, KHW;
    int32_t m_rows;          /* rows of the GEMM that will consume the pack: B*OH*OW (mode 0) / B*H*W (mode 1);
                                the n-tiling is chosen from it and must match the consumer's             */
    int32_t mode;            /* 0 forward, 1 dgrad                                                    */
    int32_t noise_mode;      /* mode 0: NN_NOISE_* (which sigma rows to add)                          */
    int32_t want_wsum;       /* mode 0, external DAC: add the colsum row (power statistic)            */
    int32_t q_bits; double q_hi; float stochastic; const float* u_inject; nn_rng rng;
    void* packed_out;        /* nn_weight_pack_bytes(job) bytes                                       */
    int32_t layout;          /* NN_PACK_* (mode 0: nn_conv_pack_layout, mode 1: nn_conv_dgrad_pack_layout) */
    void* codes;             /* optional scratch, Cout*Cin*KHW bytes: the quantizer runs ONCE per parameter into it
                                (one Philox call per 4 parameters) and every job naming the same scratch -- the
                                forward and dgrad images of a layer -- packs from the codes; jobs sharing a scratch
                                must share w_raw, q_bits, q_hi, stochastic, rng / u_inject.  q_bits <= 7.          */
} nn_wprep_job;
int64_t nn_weight_pack_bytes(const nn_wprep_job* job);
int nn_prepare_weights(const nn_wprep_job* jobs, int count, int device, void* stream);

/* ---- section 8f.1: the between-layer stages, fused ---------------------------------------------------
 * conv stage (noisynet.py:419-460, 483-520): MaxPool2d(2,2) -> BatchNorm (batch statistics, running stats
 * updated) -> ReLU -> clamp(max=act_max) -> k-bit quantize (hardware_model.py:133-173, min 0) -> NHWC bf16
 * code pack for the next tensor-core contraction.  fc stage (noisynet.py:540-569): the same with pool = 0,
 * H = W = 1.  Per-channel reductions use fixed-order partial sums (deterministic). */
typedef struct nn_stage_args {
    const float* in;          /* [B,C,H,W] fp32 NCHW: the (noisy) conv / linear output               */
    int32_t B, C, H, W, pool; /* pool = 1: MaxPool2d(2,2) first (H, W even)                           */
    float* pooled;            /* out [B,C,H/2,W/2] (pool = 1), saved for the backward                  */
    uint8_t* argmax;          /* out [B,C,H/2,W/2] window position 0..3 (pool = 1)                    */
    const float *gamma, *beta;
    float *running_mean, *running_var;   /* updated with `momentum` (may be NULL)                     */
    float momentum, eps;
    float *mean, *invstd;     /* out [C], saved for the backward                                     */
    float act_max;            /* 0 = no clamp                                                        */
    int32_t q_bits;           /* 0 = no quantisation (values stored as bf16)                          */
    double q_hi;              /* quantisation range [0, q_hi]                                         */
    float stochastic;         /* stochastic-rounding amplitude (training), 0 in eval                 */
    const float* u_inject;    /* optional uniform draws, shape of the BN input (parity hook)         */
    nn_rng rng;
    void* xp; int32_t Cp;     /* out [B,H',W',Cp] bf16 codes, Cp % 8 == 0                            */
    float* act;               /* optional out: dequantised activation, NCHW fp32                      */
    float* xmax_out;          /* optional out: max of the activation (device scalar)                  */
    void* scratch;            /* at least nn_stage_scratch_bytes(C) bytes, ZEROED once by the caller (kernels keep it
                                 consistent): per-channel records of partial sums and an arrival counter, at
                                 addresses independent of C.  One scratch sized for the widest stage may serve the
                                 forward and backward of every stage, launched in order on one stream           */
    int32_t eval_mode;        /* 1: model.eval() -- BatchNorm normalises with running_mean / running_var and updates
                                 nothing (noisynet.py:1560-1567); the caller passes stochastic = 0 (hardware_model.py:283-286) */
    int32_t stats_ready;      /* 1: mean / invstd (and the running statistics, and *xmax_out = 0) were already produced by
                                 the conv launch (nn_conv_fwd_args.bn_mean): skip the statistics pass (pool must be 0)  */
    double drop_p;            /* dropout rate in [0, 1), 0 = off: nn.Dropout(p) after ReLU + clamp and before the next
                                 quantizer (noisynet.py:375-376, :456-457, :512-513, :565-566); the quantizer and act /
                                 xmax_out see x * mask / (1 - p).  0 in eval (dropout is the identity there)             */
    uint8_t* keep;            /* out [B,C,H',W'] uint8 keep mask (1 = kept), the BN input's layout like argmax; required
                                 when drop_p > 0, read back by nn_stage_bwd                                               */
    const uint8_t* keep_inject; /* optional mask in the layout of `keep`, read instead of the Philox draw (parity hook)   */
    nn_rng drop_rng;          /* the keep decisions' own Philox stream: element (pixel, channel c) draws group
                                 2 * (pixel * Cp/8 + c/8) + (c%8)/4, word c%4, and is kept iff u01 >= (float)drop_p     */
} nn_stage_args;
int64_t nn_stage_scratch_bytes(int C);
int nn_stage_fwd(const nn_stage_args* a, int device, void* stream);

/* Backward of the stage: masks of the quantizer STE (hardware_model.py:176-183), clamp and ReLU, BatchNorm
 * backward (dgamma / dbeta are OVERWRITTEN), max-pool routing; emits the gradient w.r.t. the stage input as
 * NHWC bf16 [B,H,W,Cp] -- the operand the tensor-core wgrad / dgrad kernels read -- and optionally NCHW fp32. */
typedef struct nn_stage_bwd_args {
    const float* g;           /* grad w.r.t. the stage output, NCHW fp32 (pooled shape)               */
    const float* x;           /* the BN input saved by the forward (pooled if pool = 1, else `in`)    */
    const uint8_t* argmax;
    int32_t B, C, H, W, pool; /* H, W of the stage INPUT (pre-pool)                                   */
    const float *mean, *invstd, *gamma, *beta;
    float act_max; int32_t q_bits; double q_hi;
    float *dgamma, *dbeta;
    void* gyp; int32_t Cp;    /* out: grad w.r.t. the stage input as the bf16 pack the next wgrad / dgrad reads */
    float* gy_f32;
    void* scratch;
    int32_t gy_layout;        /* NN_PACK_TILED: NHWC [B,H,W,Cp].  NN_PACK_SHIFT: planes layout on a virt_H x virt_W
                                 pixel grid (the producing conv's INPUT grid, see nn_conv_wgrad_args); the buffer
                                 must have been zeroed once -- only output positions are ever written            */
    int32_t virt_H, virt_W;
    double drop_p;            /* dropout rate of the forward (noisynet.py:456-457, :512-513, :565-566), 0 = off:
                                 g * mask / (1 - p), and the quantizer STE tests the dropped and scaled value             */
    const uint8_t* keep;      /* the forward's keep mask (nn_stage_args.keep), required when drop_p > 0               */
} nn_stage_bwd_args;
int nn_stage_bwd(const nn_stage_bwd_args* a, int device, void* stream);

/* Input quantizer (quantize1, noisynet.py:344, :390-393) + NHWC bf16 code pack of the network input. */
int nn_input_quant_pack(const float* x, void* xp, float* act, int B, int C, int HW, int Cp, int q_bits,
                        double q_hi, float stochastic, const float* u_inject, nn_rng rng, int device, void* stream);
/* The same codes (same arithmetic and Philox counters: bit-identical) as the row-plane image `planes` of a KW-wide shift
 * forward (nn_conv_shift_planes_bytes of the geometry, C <= 8) and, if xp != NULL, the NHWC image [B,H,W,8] of
 * nn_input_quant_pack with Cp = 8, from one pass over x [B,C,H,W].  x = NULL: the planes are made from the NHWC code
 * image xp instead (e.g. written by nn_input_gather_quant_pack). */
int nn_input_quant_pack_rows(const float* x, void* xp, void* planes, int B, int C, int H, int W, int KW, int q_bits,
                             double q_hi, float stochastic, const float* u_inject, nn_rng rng, int device, void* stream);

/* Data path (section 8f.4): batch assembly of noisynet.py:1232-1269 on the device -- gather B images BY INDEX (idx [B]
 * int64 on the device, NULL = the first B) from the resident, zero-padded dataset [N,C,Hp,Wp] fp32 (utils.py:165-167), crop
 * H x W at (off_y, off_x), optional horizontal flip, then quantize1 + NHWC bf16 code pack as nn_input_quant_pack.
 * aug_dev (optional, device int32[3] = {off_y, off_x, flip}) overrides the three host values: a captured CUDA graph then
 * replays with each step's own crop / flip / indices. */
int nn_input_gather_quant_pack(const float* data, const int64_t* idx, int B, int C, int Hp, int Wp, int H, int W, int off_y,
                               int off_x, int flip, const int32_t* aug_dev, void* xp, float* act, int Cp, int q_bits, double q_hi,
                               float stochastic, const float* u_inject, nn_rng rng, int device, void* stream);

/* Head (noisynet.py:594, :1278): BatchNorm1d(C <= 16, batch statistics) -> mean cross-entropy, and the
 * gradient back through both: g [B,C] fp32 (+ optional bf16 [B,Cp] pack), dgamma / dbeta (overwritten). */
int nn_head_fwd_bwd(const float* logits, const int64_t* labels, int B, int C, const float* gamma,
                    const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                    float* loss_out, float* out, float* g, void* g_packed, int Cp, float* dgamma, float* dbeta,
                    int device, void* stream);

/* Head in eval mode: out = BatchNorm1d(x) with the running statistics (noisynet.py:594 under model.eval()). */
int nn_head_eval(const float* x, int B, int C, const float* gamma, const float* beta, const float* running_mean,
                 const float* running_var, float eps, float* out, int device, void* stream);

/* Classifier tail, fused (noisynet.py:589-594 linear2 + current noise, bn4, :1278 CrossEntropyLoss, and the way
 * back: d loss / d logits through bn4, fc2 dgrad) for a last layer with <= 16 units: ONE thread-block cluster of 8
 * CTAs with the two batch-wide reductions in distributed shared memory.  Same arithmetic as nn_noisy_conv_fwd
 * (integer-code mode) + nn_head_fwd_bwd + nn_noisy_conv_dgrad; the weight gradient still goes through
 * nn_noisy_conv_wgrad (g_packed). */
typedef struct nn_tail_args {
    const void* xp;           /* layer input [B][Kp] bf16 integer codes (Kp even, >= K), e.g. from nn_stage_fwd      */
    int32_t B, K, Kp, C;
    const int8_t* w_codes;    /* [C][K] weight quantizer codes 2k - qmax (nn_wprep_job.codes)                          */
    const float* w_raw;       /* [C][K] raw parameter (sigma^2 rows), may be NULL when noise_mode == 0               */
    float a_code_scale, w_code_scale;
    int32_t noise_mode; float current; const float* scale_dev; const float* z_inject; nn_rng rng;
    const int64_t* labels;
    const float *gamma, *beta; float *running_mean, *running_var; float momentum, eps;
    float* loss_out;          /* device scalar                                                                       */
    float* logits_out;        /* optional [B][C]: the noisy fc2 output (bn4 input)                                   */
    float* g;                 /* [B][C] d loss / d (fc2 output)                                                      */
    void* g_packed; int32_t Cp_g;   /* optional bf16 [B][Cp_g] pack of g for the weight gradient                        */
    float* gx;                /* [B][K] d loss / d (layer input), before the STE masks of the previous stage         */
    float *dgamma, *dbeta;
} nn_tail_args;
int nn_classifier_tail(const nn_tail_args* a, int device, void* stream);

/* ---- section 8e: the step's one exchange -- SUM all-reduce of the gradients (main.py:786-802) over symmetric memory ----
 * Every rank maps a buffer of identical size [nn_allreduce_ctl_bytes() control words, zeroed once | gradient data]
 * (peer_ptrs[world]: this process's mappings of all ranks' buffers, its own included; mc_ptr: the NVSwitch multicast
 * mapping of the same buffers, or NULL).  nn_allreduce_start enqueues the in-place two-shot exchange of `count` floats at
 * byte offset data_off (rank r reduces slice r with multimem.ld_reduce -- in-switch reduction -- and writes the sum into
 * every rank's buffer with multimem.st; plain peer loads / stores without multicast); nn_allreduce_wait, enqueued on the
 * stream that consumes the sums, completes it.  `bucket` (< 8) names independent exchanges that may be in flight together
 * (e.g. the fully connected layers' gradients while the conv backward still runs).  CUDA-graph capturable; every rank
 * must issue the same sequence of calls per bucket.  count * 4 must be a multiple of 16 * world. */
int64_t nn_allreduce_ctl_bytes(void);
int nn_allreduce_start(const void* const* peer_ptrs, const void* mc_ptr, int rank, int world, int bucket, int64_t data_off,
                       int64_t count, int ctas, int device, void* stream);
int nn_allreduce_wait(const void* local_ptr, int world, int bucket, int device, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NOISYNET_B200_H */
