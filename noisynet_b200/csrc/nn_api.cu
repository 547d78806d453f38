// C-ABI entry points for the fused noisy conv / linear forward and its backward.
// Validates arguments and dispatches on `precision` to the CUDA-core fp32 kernels
// (nn_conv_simt.cu) or the tensor-core kernels (nn_conv_umma.cu, nn_conv_tma.cu).  No CPU fallback exists.
#include "nn_common.cuh"

int nn_simt_conv_fwd(const nn_conv_fwd_args* a, int device, cudaStream_t st);
int nn_simt_conv_dgrad(const nn_conv_dgrad_args* a, int device, cudaStream_t st);
int nn_simt_conv_wgrad(const nn_conv_wgrad_args* a, int device, cudaStream_t st);
int64_t nn_simt_wgrad_workspace(const nn_conv_geom* g, int device);

int nn_umma_conv_fwd(const nn_conv_fwd_args* a, int device, cudaStream_t st);
int nn_umma_conv_dgrad(const nn_conv_dgrad_args* a, int device, cudaStream_t st);
int nn_umma_conv_wgrad(const nn_conv_wgrad_args* a, int device, cudaStream_t st);
int64_t nn_umma_fwd_workspace(const nn_conv_geom* g, int precision);
int64_t nn_umma_wgrad_workspace(const nn_conv_geom* g, int precision, int device);
bool nn_umma_supports(const nn_conv_geom* g, int which);

static int check_geom(const nn_conv_geom& g, const char* who) {
    if (g.B <= 0 || g.Cin <= 0 || g.H <= 0 || g.W <= 0 || g.Cout <= 0 || g.KH <= 0 || g.KW <= 0 ||
        g.stride <= 0 || g.pad < 0)
        return nn_fail("%s: bad geometry", who);
    int OH, OW;
    nn_out_hw(g, OH, OW);
    if (OH <= 0 || OW <= 0) return nn_fail("%s: empty output", who);
    const int64_t lim = (int64_t)1 << 31;
    if ((int64_t)g.B * g.Cout * OH * OW >= lim || (int64_t)g.B * g.Cin * g.H * g.W >= lim)
        return nn_fail("%s: tensor too large for 32-bit pixel indexing", who);
    return 0;
}

extern "C" int nn_conv_supported(const nn_conv_geom* g, int32_t precision, int32_t which) {
    if (!g || which < 0 || which > 2) return 0;
    if (precision == NN_PREC_FP32) return 1;
    if (precision == NN_PREC_BF16) return nn_umma_supports(g, which) ? 1 : 0;
    return 0;
}

extern "C" int64_t nn_conv_workspace_bytes(const nn_conv_geom* g, int32_t precision) {
    if (precision == NN_PREC_FP32) return 0;
    return nn_umma_fwd_workspace(g, precision);
}

extern "C" int nn_noisy_conv_fwd(const nn_conv_fwd_args* a, int device, void* stream) {
    if (!a) return nn_fail("nn_noisy_conv_fwd: null args%s", "");
    if (int e = check_geom(a->g, "nn_noisy_conv_fwd")) return e;
    if (!a->x && !(a->x_packed && a->precision != NN_PREC_FP32)) return nn_fail("nn_noisy_conv_fwd: x missing%s", "");
    if (!a->w_eff && !a->w_packed && (a->noise_mode == NN_NOISE_NONE || !a->y))
        return nn_fail("nn_noisy_conv_fwd: w_eff missing%s (noise-only mode needs noise_mode > 0 and y as input)", "");
    if (a->noise_mode < 0 || a->noise_mode > 2) return nn_fail("nn_noisy_conv_fwd: bad noise_mode%s", "");
    if (a->noise_mode != NN_NOISE_NONE) {
        if ((!a->w_raw && !a->w_packed) || (!a->y_noisy && !a->pooled_out) || !a->scale_dev)
            return nn_fail("nn_noisy_conv_fwd: noise needs w_raw, y_noisy and scale_dev%s", "");
        if (!(a->current > 0.f)) return nn_fail("nn_noisy_conv_fwd: current must be > 0%s", "");
    } else if (!a->y && !a->pooled_out) {
        return nn_fail("nn_noisy_conv_fwd: y missing%s", "");
    }
    if (a->pooled_out && a->precision == NN_PREC_FP32)
        return nn_fail("nn_noisy_conv_fwd: pooled_out is a tensor-core-path fusion%s (see nn_conv_pool_fusable)", "");
    NN_SET_DEVICE(device);
    if (a->precision == NN_PREC_FP32) return nn_simt_conv_fwd(a, device, (cudaStream_t)stream);
    if (a->precision == NN_PREC_TF32)
        return nn_fail("nn_noisy_conv_fwd: NN_PREC_TF32 is not implemented%s; unquantized operands run as NN_PREC_BF16 (bf16-rounded, "
                       "fp32 accumulate, 1.5e-2 tolerance) or NN_PREC_FP32", "");
    if (a->precision == NN_PREC_BF16) {
        if (!nn_umma_supports(&a->g, 0))
            return nn_fail("nn_noisy_conv_fwd: geometry not supported by the tensor-core path%s; use NN_PREC_FP32", "");
        return nn_umma_conv_fwd(a, device, (cudaStream_t)stream);
    }
    return nn_fail("nn_noisy_conv_fwd: unknown precision%s", "");
}

extern "C" int nn_noisy_conv_dgrad(const nn_conv_dgrad_args* a, int device, void* stream) {
    if (!a) return nn_fail("nn_noisy_conv_dgrad: null args%s", "");
    if (int e = check_geom(a->g, "nn_noisy_conv_dgrad")) return e;
    if ((!a->gy && !(a->gy_packed && a->precision != NN_PREC_FP32)) ||
        (!a->w_eff && !(a->w_packed && a->precision != NN_PREC_FP32)) || !a->gx)
        return nn_fail("nn_noisy_conv_dgrad: null tensor%s", "");
    NN_SET_DEVICE(device);
    if (a->precision == NN_PREC_FP32) return nn_simt_conv_dgrad(a, device, (cudaStream_t)stream);
    if (a->precision != NN_PREC_BF16) return nn_fail("nn_noisy_conv_dgrad: precision not implemented%s (NN_PREC_FP32 / NN_PREC_BF16)", "");
    if (!nn_umma_supports(&a->g, 1))
        return nn_fail("nn_noisy_conv_dgrad: geometry not supported by the tensor-core path%s; use NN_PREC_FP32", "");
    return nn_umma_conv_dgrad(a, device, (cudaStream_t)stream);
}

extern "C" int64_t nn_conv_wgrad_workspace_bytes(const nn_conv_geom* g, int32_t precision, int dev) {
    if (precision == NN_PREC_FP32) return nn_simt_wgrad_workspace(g, dev);
    return nn_umma_wgrad_workspace(g, precision, dev);
}

extern "C" int nn_noisy_conv_wgrad(const nn_conv_wgrad_args* a, int device, void* stream) {
    if (!a) return nn_fail("nn_noisy_conv_wgrad: null args%s", "");
    if (int e = check_geom(a->g, "nn_noisy_conv_wgrad")) return e;
    const bool packed_ok = a->precision != NN_PREC_FP32;
    if ((!a->gy && !(a->gy_packed && packed_ok)) || (!a->x && !(a->x_packed && packed_ok)) || !a->gw)
        return nn_fail("nn_noisy_conv_wgrad: null tensor%s", "");
    NN_SET_DEVICE(device);
    if (a->precision == NN_PREC_FP32) return nn_simt_conv_wgrad(a, device, (cudaStream_t)stream);
    if (a->precision != NN_PREC_BF16) return nn_fail("nn_noisy_conv_wgrad: precision not implemented%s (NN_PREC_FP32 / NN_PREC_BF16)", "");
    if (!nn_umma_supports(&a->g, 2))
        return nn_fail("nn_noisy_conv_wgrad: geometry not supported by the tensor-core path%s; use NN_PREC_FP32", "");
    return nn_umma_conv_wgrad(a, device, (cudaStream_t)stream);
}
