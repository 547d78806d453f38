"""ctypes binding of libnoisynet_b200.so (the C ABI declared in include/noisynet_b200.h).

There is no CPU or eager fallback: if the shared library is missing, or a tensor is not a
CUDA tensor, the ops raise.  Build with ``python __graft_entry__.py`` (or ``build()``).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NN_LIB_PATH") or os.path.join(_HERE, "lib", "libnoisynet_b200.so")   # NN_LIB_PATH: instrumented debug builds
ABI_VERSION = 18

NOISE_NONE, NOISE_MERGED, NOISE_EXTERNAL = 0, 1, 2
PREC_FP32, PREC_TF32, PREC_BF16 = 0, 1, 2
PACK_TILED, PACK_SHIFT, PACK_TMA = 0, 1, 2

c_f32p = C.c_void_p      # device pointers travel as void* (int addresses from tensor.data_ptr())


class Rng(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", C.c_void_p)]


class ConvGeom(C.Structure):
    _fields_ = [("B", C.c_int32), ("Cin", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("Cout", C.c_int32), ("KH", C.c_int32), ("KW", C.c_int32),
                ("stride", C.c_int32), ("pad", C.c_int32)]


class ConvFwdArgs(C.Structure):
    _fields_ = [("g", ConvGeom),
                ("x", C.c_void_p), ("w_eff", C.c_void_p), ("w_raw", C.c_void_p), ("bias", C.c_void_p),
                ("y", C.c_void_p), ("y_noisy", C.c_void_p),
                ("noise_mode", C.c_int32), ("current", C.c_float),
                ("scale_dev", C.c_void_p), ("z_inject", C.c_void_p), ("z_export", C.c_void_p),
                ("sigma_export", C.c_void_p),
                ("rng", Rng),
                ("stats", C.c_void_p),
                ("precision", C.c_int32),
                ("a_code_scale", C.c_float), ("w_code_scale", C.c_float),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64), ("x_packed", C.c_void_p),
                ("w_packed", C.c_void_p), ("w_packed_layout", C.c_int32),
                ("pooled_out", C.c_void_p), ("argmax_out", C.c_void_p),
                ("bn_mean", C.c_void_p), ("bn_invstd", C.c_void_p), ("bn_running_mean", C.c_void_p), ("bn_running_var", C.c_void_p),
                ("bn_eps", C.c_float), ("bn_momentum", C.c_float), ("bn_eval_mode", C.c_int32), ("bn_scratch", C.c_void_p),
                ("zero_out", C.c_void_p)]


class ConvDgradArgs(C.Structure):
    _fields_ = [("g", ConvGeom),
                ("gy", C.c_void_p), ("w_eff", C.c_void_p), ("gx", C.c_void_p),
                ("x_pre", C.c_void_p), ("x_lo", C.c_double), ("x_hi", C.c_double),
                ("precision", C.c_int32), ("w_code_scale", C.c_float),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64), ("gy_packed", C.c_void_p),
                ("w_packed", C.c_void_p), ("w_packed_layout", C.c_int32)]


class ConvWgradArgs(C.Structure):
    _fields_ = [("g", ConvGeom),
                ("gy", C.c_void_p), ("x", C.c_void_p), ("gw", C.c_void_p),
                ("w_raw", C.c_void_p), ("w_lo", C.c_double), ("w_hi", C.c_double),
                ("precision", C.c_int32), ("a_code_scale", C.c_float),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64), ("x_packed", C.c_void_p),
                ("gy_packed", C.c_void_p), ("gy_packed_layout", C.c_int32)]


class AdamWTensor(C.Structure):
    _fields_ = [("p", C.c_void_p), ("g", C.c_void_p), ("m", C.c_void_p), ("v", C.c_void_p),
                ("n", C.c_int64), ("lr", C.c_float), ("weight_decay", C.c_float), ("clamp", C.c_float),
                ("absmax_out", C.c_void_p)]


class WPrepJob(C.Structure):
    _fields_ = [("w_raw", C.c_void_p), ("Cout", C.c_int32), ("Cin", C.c_int32), ("KHW", C.c_int32),
                ("m_rows", C.c_int32), ("mode", C.c_int32), ("noise_mode", C.c_int32), ("want_wsum", C.c_int32),
                ("q_bits", C.c_int32), ("q_hi", C.c_double), ("stochastic", C.c_float), ("u_inject", C.c_void_p),
                ("rng", Rng), ("packed_out", C.c_void_p), ("layout", C.c_int32), ("codes", C.c_void_p)]


class StageArgs(C.Structure):
    _fields_ = [("in_", C.c_void_p), ("B", C.c_int32), ("C", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("pool", C.c_int32), ("pooled", C.c_void_p), ("argmax", C.c_void_p),
                ("gamma", C.c_void_p), ("beta", C.c_void_p), ("running_mean", C.c_void_p), ("running_var", C.c_void_p),
                ("momentum", C.c_float), ("eps", C.c_float), ("mean", C.c_void_p), ("invstd", C.c_void_p),
                ("act_max", C.c_float), ("q_bits", C.c_int32), ("q_hi", C.c_double), ("stochastic", C.c_float),
                ("u_inject", C.c_void_p), ("rng", Rng), ("xp", C.c_void_p), ("Cp", C.c_int32),
                ("act", C.c_void_p), ("xmax_out", C.c_void_p), ("scratch", C.c_void_p), ("eval_mode", C.c_int32),
                ("stats_ready", C.c_int32), ("drop_p", C.c_double), ("keep", C.c_void_p), ("keep_inject", C.c_void_p),
                ("drop_rng", Rng)]


class StageBwdArgs(C.Structure):
    _fields_ = [("g", C.c_void_p), ("x", C.c_void_p), ("argmax", C.c_void_p),
                ("B", C.c_int32), ("C", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("pool", C.c_int32),
                ("mean", C.c_void_p), ("invstd", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
                ("act_max", C.c_float), ("q_bits", C.c_int32), ("q_hi", C.c_double),
                ("dgamma", C.c_void_p), ("dbeta", C.c_void_p), ("gyp", C.c_void_p), ("Cp", C.c_int32),
                ("gy_f32", C.c_void_p), ("scratch", C.c_void_p),
                ("gy_layout", C.c_int32), ("virt_H", C.c_int32), ("virt_W", C.c_int32),
                ("drop_p", C.c_double), ("keep", C.c_void_p)]


class TailArgs(C.Structure):
    _fields_ = [("xp", C.c_void_p), ("B", C.c_int32), ("K", C.c_int32), ("Kp", C.c_int32), ("C", C.c_int32),
                ("w_codes", C.c_void_p), ("w_raw", C.c_void_p), ("a_code_scale", C.c_float), ("w_code_scale", C.c_float),
                ("noise_mode", C.c_int32), ("current", C.c_float), ("scale_dev", C.c_void_p), ("z_inject", C.c_void_p),
                ("rng", Rng), ("labels", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
                ("running_mean", C.c_void_p), ("running_var", C.c_void_p), ("momentum", C.c_float), ("eps", C.c_float),
                ("loss_out", C.c_void_p), ("logits_out", C.c_void_p), ("g", C.c_void_p), ("g_packed", C.c_void_p),
                ("Cp_g", C.c_int32), ("gx", C.c_void_p), ("dgamma", C.c_void_p), ("dbeta", C.c_void_p)]


# name -> (restype, argtypes); mirrors include/noisynet_b200.h one to one
SIGNATURES = {
    "nn_last_error": (C.c_char_p, []),
    "nn_abi_version": (C.c_int, []),
    "nn_launch_count": (C.c_uint64, []),
    "nn_device_info": (C.c_int, [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "nn_rng_advance": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]),
    "nn_quantize_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_double, C.c_double,
                                  C.c_float, C.c_void_p, Rng, C.c_int, C.c_void_p]),
    "nn_quantize_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_double,
                                  C.c_int, C.c_void_p]),
    "nn_range_scratch_bytes": (C.c_int64, []),
    "nn_range_select": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_double, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int,
                                  C.c_void_p]),
    "nn_quantize_fwd_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_float, C.c_void_p, Rng,
                                      C.c_int, C.c_void_p]),
    "nn_quantize_bwd_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]),
    "nn_weight_noise_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p, Rng,
                                      C.c_int, C.c_void_p]),
    "nn_adamw_step_part": (C.c_int, [C.POINTER(AdamWTensor), C.c_int, C.c_float, C.c_float, C.c_float, C.c_float,
                                    C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "nn_adamw_step": (C.c_int, [C.POINTER(AdamWTensor), C.c_int, C.c_float, C.c_float, C.c_float, C.c_float,
                                C.c_void_p, C.c_int, C.c_void_p]),
    "nn_weight_pack_bytes": (C.c_int64, [C.POINTER(WPrepJob)]),
    "nn_prepare_weights": (C.c_int, [C.POINTER(WPrepJob), C.c_int, C.c_int, C.c_void_p]),
    "nn_stage_scratch_bytes": (C.c_int64, [C.c_int]),
    "nn_conv_bn_scratch_bytes": (C.c_int64, [C.c_int]),
    "nn_conv_linear_bn_fusable": (C.c_int, [C.POINTER(ConvGeom), C.c_int32, C.c_int32, C.c_int]),
    "nn_stage_fwd": (C.c_int, [C.POINTER(StageArgs), C.c_int, C.c_void_p]),
    "nn_stage_bwd": (C.c_int, [C.POINTER(StageBwdArgs), C.c_int, C.c_void_p]),
    "nn_input_quant_pack": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_double, C.c_float, C.c_void_p, Rng, C.c_int, C.c_void_p]),
    "nn_input_quant_pack_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_double, C.c_float, C.c_void_p, Rng, C.c_int, C.c_void_p]),
    "nn_input_gather_quant_pack": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double,
                                             C.c_float, C.c_void_p, Rng, C.c_int, C.c_void_p]),
    "nn_head_fwd_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "nn_allreduce_ctl_bytes": (C.c_int64, []),
    "nn_allreduce_start": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int,
                                     C.c_int, C.c_void_p]),
    "nn_allreduce_wait": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "nn_head_eval": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p,
                               C.c_int, C.c_void_p]),
    "nn_tensor_stats": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]),
    "nn_clamp_absmax": (C.c_int, [C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_int, C.c_void_p]),
    "nn_noise_epilogue": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                                    C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, Rng, C.c_int, C.c_void_p]),
    "nn_alt_noise": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_void_p,
                               C.c_void_p, Rng, C.c_int, C.c_void_p]),
    "nn_conv_workspace_bytes": (C.c_int64, [C.POINTER(ConvGeom), C.c_int32]),
    "nn_conv_supported": (C.c_int, [C.POINTER(ConvGeom), C.c_int32, C.c_int32]),
    "nn_debug_error_flag": (C.c_int, [C.c_int, C.c_int]),
    "nn_debug_main_kernel_ms": (C.c_float, [C.c_int]),
    "nn_debug_cta_timeline": (C.c_int, [C.c_void_p, C.c_int]),
    "nn_conv_pack_layout": (C.c_int, [C.POINTER(ConvGeom), C.c_int32, C.c_int32]),
    "nn_debug_shift_enable": (C.c_int, [C.c_int]),
    "nn_debug_tma_enable": (C.c_int, [C.c_int]),
    "nn_conv_dgrad_pack_layout": (C.c_int, [C.POINTER(ConvGeom), C.c_int32]),
    "nn_conv_pool_fusable": (C.c_int, [C.POINTER(ConvGeom), C.c_int32, C.c_int32]),
    "nn_classifier_tail": (C.c_int, [C.POINTER(TailArgs), C.c_int, C.c_void_p]),
    "nn_conv_wgrad_pack_layout": (C.c_int, [C.POINTER(ConvGeom), C.c_int32, C.c_int]),
    "nn_conv_gy_planes_bytes": (C.c_int64, [C.POINTER(ConvGeom)]),
    "nn_conv_shift_planes_bytes": (C.c_int64, [C.POINTER(ConvGeom)]),
    "nn_noisy_conv_fwd": (C.c_int, [C.POINTER(ConvFwdArgs), C.c_int, C.c_void_p]),
    "nn_noisy_conv_dgrad": (C.c_int, [C.POINTER(ConvDgradArgs), C.c_int, C.c_void_p]),
    "nn_conv_dgrad_planes_ok": (C.c_int, [C.POINTER(ConvGeom)]),
    "nn_conv_dgrad_planes": (C.c_int, [C.POINTER(ConvDgradArgs), C.c_int, C.c_void_p]),
    "nn_conv_wgrad_workspace_bytes": (C.c_int64, [C.POINTER(ConvGeom), C.c_int32, C.c_int]),
    "nn_noisy_conv_wgrad": (C.c_int, [C.POINTER(ConvWgradArgs), C.c_int, C.c_void_p]),
}

_lib = None


class NoisyNetLibraryError(RuntimeError):
    pass


def load():
    """Loads the shared library (once).  Raises loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise NoisyNetLibraryError(
            "noisynet_b200: CUDA extension %s not found; build it with "
            "`python -c 'import __graft_entry__ as g; g.build()'`. There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)         # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    v = lib.nn_abi_version()
    if v != ABI_VERSION:
        raise NoisyNetLibraryError("noisynet_b200: ABI mismatch: library %d, binding %d (rebuild)" % (v, ABI_VERSION))
    _lib = lib
    return lib


def check(rc, who=""):
    if rc != 0:
        msg = load().nn_last_error()
        raise NoisyNetLibraryError("%s failed (%d): %s" % (who, rc, msg.decode() if msg else "?"))
