"""Torch-facing wrappers over the C ABI: raw ops on CUDA tensors + autograd Functions.

PyTorch is plumbing here (device memory, streams, autograd graph); every arithmetic op of the
hot path runs in libnoisynet_b200.so.  All tensors must be CUDA fp32; anything else raises.
"""
import contextlib
import ctypes as C
import math

import torch
from torch.autograd.function import Function, InplaceFunction, once_differentiable

from . import _lib
from ._lib import (NOISE_EXTERNAL, NOISE_MERGED, NOISE_NONE, PREC_BF16, PREC_FP32, PREC_TF32,
                   ConvDgradArgs, ConvFwdArgs, ConvGeom, ConvWgradArgs, Rng)

# Default arithmetic of the contraction kernels.  PREC_FP32 = CUDA-core fp32 (reference arithmetic);
# PREC_BF16 = tensor cores (exact for integer codes, bf16-rounded operands otherwise).  Overridable per call or globally.
# "tf32" is declared in the C ABI but not implemented: asking for it raises instead of silently running something else.
_default_precision = PREC_FP32
_PREC_NAMES = {"fp32": PREC_FP32, "bf16": PREC_BF16}


def _prec_by_name(p):
    if p == "tf32" or p == PREC_TF32:
        raise ValueError("noisynet_b200: precision 'tf32' is not implemented; use 'bf16' (tensor cores, bf16-rounded operands, "
                         "fp32 accumulate, 1.5e-2 tolerance) or 'fp32' (CUDA cores)")
    return _PREC_NAMES[p]


def set_default_precision(p):
    global _default_precision
    _default_precision = _prec_by_name(p) if isinstance(p, str) else int(p)


def get_default_precision():
    return _default_precision


def _prec(p):
    if p is None:
        return _default_precision
    if isinstance(p, str):
        return _prec_by_name(p)
    if int(p) == PREC_TF32:
        _prec_by_name("tf32")
    return int(p)


# ----------------------------------------------------------------------------- plumbing

def _req(t, name="tensor"):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise _lib.NoisyNetLibraryError(
            "noisynet_b200: %s must be a CUDA tensor (got %s); there is no CPU fallback"
            % (name, "cpu tensor" if isinstance(t, torch.Tensor) else type(t).__name__))
    if t.dtype != torch.float32:
        raise TypeError("noisynet_b200: %s must be float32 (got %s)" % (name, t.dtype))
    return t if t.is_contiguous() else t.contiguous()


def _p(t):
    return None if t is None else t.data_ptr()


def _dev(t):
    return t.device.index if t.device.index is not None else torch.cuda.current_device()


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


_graph_rng = None   # (seed, offset_dev tensor, [next call slot])


@contextlib.contextmanager
def graph_rng(step_counter, seed=None):
    """While active (e.g. during CUDA-graph capture) every op draws from
    (seed, slot << 32 + *step_counter): a replay with an advanced counter draws fresh numbers.
    ``step_counter`` is a 1-element int64 CUDA tensor advanced by ``rng_advance``."""
    global _graph_rng
    if seed is None:
        seed = torch.cuda.default_generators[_dev(step_counter)].initial_seed()
    prev = _graph_rng
    _graph_rng = (int(seed) & 0xFFFFFFFFFFFFFFFF, step_counter, [1])
    try:
        yield
    finally:
        _graph_rng = prev


def rng_advance(step_counter, inc=1):
    dev = _dev(step_counter)
    _lib.check(_lib.load().nn_rng_advance(step_counter.data_ptr(), inc, dev, _stream(dev)), "nn_rng_advance")


def next_rng(dev):
    """(seed, offset) for one kernel call.  Eager: taken from torch's CUDA generator (so
    torch.manual_seed(args.seed), noisynet.py:314-317, stays the reproducibility knob)."""
    if _graph_rng is not None:
        seed, ctr, slot = _graph_rng
        s = slot[0]
        slot[0] += 1
        return Rng(seed, s << 32, ctr.data_ptr())
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("noisynet_b200: RNG used under CUDA-graph capture; wrap the capture in ops.graph_rng()")
    gen = torch.cuda.default_generators[dev]
    off = gen.get_offset()
    gen.set_offset(off + 4)
    return Rng(gen.initial_seed() & 0xFFFFFFFFFFFFFFFF, off, None)


def _fixed_rng(seed, offset):
    return Rng(int(seed) & 0xFFFFFFFFFFFFFFFF, int(offset), None)


_inject = None   # test hook: dict(u=deque, z=deque) consumed in call order by the stochastic ops


@contextlib.contextmanager
def inject_random(u_list=(), z_list=()):
    """Parity hook: the next stochastic ops take their uniform / normal draws from these tensors (in
    call order) instead of Philox -- lets a whole forward be replayed against the CPU oracle."""
    global _inject
    from collections import deque
    prev = _inject
    _inject = dict(u=deque(u_list), z=deque(z_list))
    try:
        yield _inject
    finally:
        _inject = prev


def _pop_inject(kind, like_shape=None):
    if _inject is None or not _inject[kind]:
        return None
    t = _inject[kind].popleft()
    if like_shape is not None and tuple(t.shape) != tuple(like_shape):
        t = t.reshape(like_shape)
    return t


_workspaces = {}


def _workspace(dev, nbytes, tag="fwd"):
    if nbytes <= 0:
        return None
    key = (dev, tag)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(int(nbytes * 1.25) + 1024, dtype=torch.uint8, device=torch.device("cuda", dev))
        _workspaces[key] = ws
    return ws


# ----------------------------------------------------------------------------- raw ops

def quantize_fwd(x, num_bits, min_value, max_value, stochastic=0.0, u=None, out=None, rng=None):
    x = _req(x, "input")
    dev = _dev(x)
    y = torch.empty_like(x) if out is None else out
    if u is None and stochastic > 0 and rng is None:
        u = _pop_inject("u", x.shape)
    if u is not None:
        u = _req(u, "u")
    r = rng if rng is not None else (next_rng(dev) if (stochastic > 0 and u is None) else Rng(0, 0, None))
    _lib.check(_lib.load().nn_quantize_fwd(_p(x), _p(y), x.numel(), int(num_bits), float(min_value),
                                           float(max_value), float(stochastic), _p(u), r, dev, _stream(dev)),
               "nn_quantize_fwd")
    return y


def quantize_bwd(x, gy, min_value, max_value):
    x, gy = _req(x, "input"), _req(gy, "grad_output")
    dev = _dev(x)
    gx = torch.empty_like(gy)
    _lib.check(_lib.load().nn_quantize_bwd(_p(x), _p(gy), _p(gx), x.numel(), float(min_value), float(max_value),
                                           dev, _stream(dev)), "nn_quantize_bwd")
    return gx


_range_scratch = {}


def range_select(x, pctl_percent=0.0, mode=0, min_value=0.0, k_rank=0):
    """QuantMeasure's range selection on the device (hardware_model.py:232-259): returns a float32[4] DEVICE tensor
    [percentile, max(x), range_min, range_max] (mode 0) / [running_min, running_max, running_min, running_max]
    (mode 1, signed weights) -- exact kthvalue by radix select, no host sync.  mode 0 takes the rank ``k_rank`` the caller
    computed from numel (hardware_model.py:249 / quant.py:109); mode 1 derives its ranks from the on-device counts."""
    x = _req(x, "input")
    dev = _dev(x)
    lib = _lib.load()
    sc = _range_scratch.get(dev)
    if sc is None:
        sc = _range_scratch[dev] = torch.empty(int(lib.nn_range_scratch_bytes()), dtype=torch.uint8, device=x.device)
    out4 = torch.empty(4, dtype=torch.float32, device=x.device)
    _lib.check(lib.nn_range_select(_p(x), x.numel(), int(k_rank), float(pctl_percent), int(mode), float(min_value), _p(out4), _p(sc),
                                   dev, _stream(dev)), "nn_range_select")
    return out4


def quantize_fwd_dev(x, num_bits, range_dev, stochastic=0.0, u=None, out=None, rng=None):
    """quantize_fwd with the range {min, max} in device memory (float32[2], e.g. range_select(...)[2:4])."""
    x = _req(x, "input")
    dev = _dev(x)
    y = torch.empty_like(x) if out is None else out
    if u is None and stochastic > 0 and rng is None:
        u = _pop_inject("u", x.shape)
    if u is not None:
        u = _req(u, "u")
    r = rng if rng is not None else (next_rng(dev) if (stochastic > 0 and u is None) else Rng(0, 0, None))
    _lib.check(_lib.load().nn_quantize_fwd_dev(_p(x), _p(y), x.numel(), int(num_bits), _p(_req(range_dev, "range_dev")),
                                               float(stochastic), _p(u), r, dev, _stream(dev)), "nn_quantize_fwd_dev")
    return y


def quantize_bwd_dev(x, gy, range_dev):
    x, gy = _req(x, "input"), _req(gy, "grad_output")
    dev = _dev(x)
    gx = torch.empty_like(gy)
    _lib.check(_lib.load().nn_quantize_bwd_dev(_p(x), _p(gy), _p(gx), x.numel(), _p(_req(range_dev, "range_dev")), dev, _stream(dev)),
               "nn_quantize_bwd_dev")
    return gx


def weight_noise(w, noise, u=None, rng=None):
    w = _req(w, "weight")
    dev = _dev(w)
    out = torch.empty_like(w)
    if u is None and rng is None:
        u = _pop_inject("u", w.shape)
    if u is not None:
        u = _req(u, "u")
    r = rng if rng is not None else (next_rng(dev) if u is None else Rng(0, 0, None))
    _lib.check(_lib.load().nn_weight_noise_fwd(_p(w), _p(out), w.numel(), float(noise), _p(u), r, dev, _stream(dev)),
               "nn_weight_noise_fwd")
    return out


def tensor_stats(x):
    """Device tensor [max(x), max|x|, count(x>0)] -- no host sync."""
    x = _req(x, "tensor")
    dev = _dev(x)
    out = torch.empty(3, dtype=torch.float32, device=x.device)
    _lib.check(_lib.load().nn_tensor_stats(_p(x), x.numel(), _p(out), dev, _stream(dev)), "nn_tensor_stats")
    return out


def clamp_absmax_(w, w_max, want_absmax=True, out=None):
    w = w if isinstance(w, torch.Tensor) else w.data
    if not w.is_contiguous():
        raise ValueError("clamp_absmax_: weight must be contiguous")
    _req(w, "weight")
    dev = _dev(w)
    if out is None:
        out = torch.empty(1, dtype=torch.float32, device=w.device) if want_absmax else None
    _lib.check(_lib.load().nn_clamp_absmax(_p(w), w.numel(), float(w_max), _p(out), dev, _stream(dev)),
               "nn_clamp_absmax")
    return out


def noise_epilogue(y, S, scale_dev, current, z=None, z_export=None, stats2=None, rng=None):
    y, S = _req(y, "y"), _req(S, "S")
    dev = _dev(y)
    out = torch.empty_like(y)
    r = rng if rng is not None else (next_rng(dev) if z is None else Rng(0, 0, None))
    _lib.check(_lib.load().nn_noise_epilogue(_p(y), _p(S), _p(out), y.numel(), 1, _p(scale_dev), float(current),
                                             _p(None if z is None else _req(z, "z")), _p(z_export), _p(stats2), r,
                                             dev, _stream(dev)), "nn_noise_epilogue")
    return out


ALT_KINDS = {"uniform_ind": 1, "uniform_dep": 2, "normal_ind": 3, "normal_dep": 4, "distort_act": 5}


def alt_noise(y, kind, level, rnd=None, rng=None):
    y = _req(y, "output")
    dev = _dev(y)
    k = ALT_KINDS[kind]
    absmax = tensor_stats(y)[1:2] if k in (1, 3) else None
    out = torch.empty_like(y)
    r = rng if rng is not None else (next_rng(dev) if rnd is None else Rng(0, 0, None))
    _lib.check(_lib.load().nn_alt_noise(_p(y), _p(out), y.numel(), k, float(level), _p(absmax),
                                        _p(None if rnd is None else _req(rnd, "rnd")), r, dev, _stream(dev)),
               "nn_alt_noise")
    return out


def _pick_prec(prec, g, which):
    """tensor-core precisions serve a subset of geometries; the rest run on the fp32 CUDA-core kernels."""
    if prec != PREC_FP32 and not _lib.load().nn_conv_supported(C.byref(g), int(prec), which):
        return PREC_FP32
    return prec


def error_flag(dev=0, reset=True):
    """Synchronises and returns the tensor-core pipeline watchdog flag (0 = ok)."""
    return _lib.load().nn_debug_error_flag(int(dev), 1 if reset else 0)


def _geom(x_shape, w_shape, stride, pad):
    B, Cin, H, W = x_shape
    Cout, Cin2, KH, KW = w_shape
    if Cin != Cin2:
        raise ValueError("noisynet_b200: channel mismatch: input %s weight %s (groups != 1 is not supported)"
                         % (tuple(x_shape), tuple(w_shape)))
    g = ConvGeom(B, Cin, H, W, Cout, KH, KW, int(stride), int(pad))
    OH = (H + 2 * pad - KH) // stride + 1
    OW = (W + 2 * pad - KW) // stride + 1
    return g, OH, OW


def noisy_conv_fwd(x, w_eff, w_raw=None, bias=None, stride=1, pad=0, noise_mode=NOISE_NONE, current=0.0,
                   scale_dev=None, z=None, want_z=False, want_sigma=False, stats=None, precision=None,
                   a_code_scale=0.0, w_code_scale=0.0, y_in=None, want_y=True, rng=None):
    """One launch: y = conv(x, w_eff) [+ bias]; y_noisy = y + z * sqrt(0.1 * scale / I * conv(x, g(|w_raw|))).

    ``w_eff=None`` with ``y_in`` given = noise-only mode (the two-call flow of noisynet.py:398+415:
    the clean output already exists, only the sigma^2 contraction and the epilogue run).
    Returns dict(y=, y_noisy=, z=, sigma=)."""
    x = _req(x, "input")
    dev = _dev(x)
    prec = _prec(precision)
    wshape = (w_eff if w_eff is not None else w_raw).shape
    g, OH, OW = _geom(x.shape, wshape, stride, pad)
    prec = _pick_prec(prec, g, 0)
    oshape = (g.B, g.Cout, OH, OW)
    a = ConvFwdArgs()
    a.g = g
    a.x = _p(x)
    keep = [x]
    if w_eff is not None:
        w_eff = _req(w_eff, "weight")
        a.w_eff = _p(w_eff)
        y = x.new_empty(oshape) if (want_y or noise_mode == NOISE_NONE) else None
    else:
        if y_in is None or noise_mode == NOISE_NONE:
            raise ValueError("noise-only mode needs y_in and a noise_mode")
        y = _req(y_in, "output")
        a.w_eff = None
    keep.append(w_eff)
    a.y = _p(y)
    if bias is not None:
        bias = _req(bias, "bias")
    a.bias = _p(bias)
    out = dict(y=y, y_noisy=None, z=None, sigma=None)
    a.noise_mode = int(noise_mode)
    if noise_mode != NOISE_NONE:
        w_raw = _req(w_raw, "raw weight")
        a.w_raw = _p(w_raw)
        a.current = float(current)
        a.scale_dev = _p(_req(scale_dev, "scale_dev"))
        out["y_noisy"] = x.new_empty(oshape)
        a.y_noisy = _p(out["y_noisy"])
        if z is None and rng is None:
            z = _pop_inject("z", oshape)
        if z is not None:
            z = _req(z, "z")
            a.z_inject = _p(z)
        if want_z:
            out["z"] = x.new_empty(oshape)
            a.z_export = _p(out["z"])
        if want_sigma:
            out["sigma"] = x.new_empty(oshape)
            a.sigma_export = _p(out["sigma"])
        a.rng = rng if rng is not None else (next_rng(dev) if z is None else Rng(0, 0, None))
        a.stats = _p(stats)
    a.precision = int(prec)
    a.a_code_scale = float(a_code_scale)
    a.w_code_scale = float(w_code_scale)
    lib = _lib.load()
    nbytes = lib.nn_conv_workspace_bytes(C.byref(g), int(prec))
    ws = _workspace(dev, nbytes, "fwd")
    a.workspace = _p(ws)
    a.workspace_bytes = 0 if ws is None else ws.numel()
    _lib.check(lib.nn_noisy_conv_fwd(C.byref(a), dev, _stream(dev)), "nn_noisy_conv_fwd")
    return out


def conv_dgrad(gy, w_eff, x_shape, stride=1, pad=0, x_pre=None, x_lo=0.0, x_hi=0.0, precision=None, w_code_scale=0.0):
    gy, w_eff = _req(gy, "grad_output"), _req(w_eff, "weight")
    dev = _dev(gy)
    prec = _prec(precision)
    g, OH, OW = _geom(x_shape, w_eff.shape, stride, pad)
    prec = _pick_prec(prec, g, 1)
    gx = gy.new_empty(tuple(x_shape))
    a = ConvDgradArgs()
    a.g = g
    a.gy, a.w_eff, a.gx = _p(gy), _p(w_eff), _p(gx)
    if x_pre is not None:
        x_pre = _req(x_pre, "x_pre")
        a.x_pre, a.x_lo, a.x_hi = _p(x_pre), float(x_lo), float(x_hi)
    a.precision = int(prec)
    a.w_code_scale = float(w_code_scale)
    lib = _lib.load()
    ws = _workspace(dev, lib.nn_conv_workspace_bytes(C.byref(g), int(prec)), "fwd")
    a.workspace = _p(ws)
    a.workspace_bytes = 0 if ws is None else ws.numel()
    _lib.check(lib.nn_noisy_conv_dgrad(C.byref(a), dev, _stream(dev)), "nn_noisy_conv_dgrad")
    return gx


def conv_wgrad(gy, x, w_shape, stride=1, pad=0, w_raw=None, w_lo=0.0, w_hi=0.0, precision=None, a_code_scale=0.0):
    gy, x = _req(gy, "grad_output"), _req(x, "input")
    dev = _dev(gy)
    prec = _prec(precision)
    g, OH, OW = _geom(x.shape, w_shape, stride, pad)
    prec = _pick_prec(prec, g, 2)
    gw = gy.new_empty(tuple(w_shape))
    a = ConvWgradArgs()
    a.g = g
    a.gy, a.x, a.gw = _p(gy), _p(x), _p(gw)
    if w_raw is not None:
        w_raw = _req(w_raw, "raw weight")
        a.w_raw, a.w_lo, a.w_hi = _p(w_raw), float(w_lo), float(w_hi)
    a.precision = int(prec)
    a.a_code_scale = float(a_code_scale)
    lib = _lib.load()
    nbytes = lib.nn_conv_wgrad_workspace_bytes(C.byref(g), int(prec), dev)
    ws = _workspace(dev, nbytes, "wgrad")
    a.workspace = _p(ws)
    a.workspace_bytes = 0 if ws is None else ws.numel()
    _lib.check(lib.nn_noisy_conv_wgrad(C.byref(a), dev, _stream(dev)), "nn_noisy_conv_wgrad")
    return gw


# ----------------------------------------------------------------------------- autograd

class UniformQuantize(InplaceFunction):
    """Same call form as the reference: ``UniformQuantize().apply(input, num_bits, min_value,
    max_value, stochastic, inplace, debug)`` (hardware_model.py:130-183, quant.py:10-61)."""

    @staticmethod
    def forward(ctx, input, num_bits=8, min_value=None, max_value=None, stochastic=0.5, inplace=False,
                debug=False, u=None, range_dev=None):
        """``range_dev`` (float32[2] device tensor {min, max}, from ops.range_select) replaces min_value / max_value: the
        range never visits the host (the reference's ``input.max().item()`` / ``running_max.item()`` syncs)."""
        ctx.range_dev = range_dev
        if range_dev is None:
            ctx.min_value = float(min_value)
            ctx.max_value = float(max_value)
        ctx.bits = int(num_bits)
        if inplace and not input.is_contiguous():
            raise ValueError("noisynet_b200: UniformQuantize(inplace=True) needs a contiguous input (the kernel writes "
                             "numel contiguous floats)")
        x = _req(input, "input")
        fwd = (lambda out=None: quantize_fwd_dev(x, num_bits, range_dev, stochastic, u, out=out)) if range_dev is not None else \
            (lambda out=None: quantize_fwd(x, num_bits, min_value, max_value, stochastic, u, out=out))
        if inplace:
            # the backward needs the pre-quantisation values -> keep a copy, write in place
            ctx.save_for_backward(x.clone())
            ctx.mark_dirty(input)
            fwd(out=input)
            return input
        ctx.save_for_backward(x)
        return fwd()

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        (x,) = ctx.saved_tensors
        if ctx.range_dev is not None:
            return quantize_bwd_dev(x, grad_output, ctx.range_dev), None, None, None, None, None, None, None, None
        return quantize_bwd(x, grad_output, ctx.min_value, ctx.max_value), None, None, None, None, None, None, None, None


class AddNoise(InplaceFunction):
    """hardware_model.py:291-307: w + w*U(-n, n), straight-through gradient."""

    @staticmethod
    def forward(ctx, input, noise=0, debug=False, u=None):
        return weight_noise(input, noise, u)

    @staticmethod
    def backward(ctx, grad_output):
        return grad_output, None, None, None


class StraightThrough(Function):
    """forward: returns ``value`` (computed outside autograd from ``y``); backward: identity to ``y``."""

    @staticmethod
    def forward(ctx, y, value):
        return value

    @staticmethod
    def backward(ctx, g):
        return g, None


class ConvFn(Function):
    """F.conv2d(x, w, bias, stride, padding) (hardware_model.py:362) on the C-ABI kernels, with the
    optional saturated-STE masks of the quantizers in front of it fused into dgrad / wgrad:
    ``w_ste=(w_raw, lo, hi)`` makes ``w`` the *quantized* weight and routes the weight gradient,
    masked, to ``w_raw`` (hardware_model.py:343 + :176-183)."""

    @staticmethod
    def forward(ctx, x, w, bias, stride, pad, precision, w_raw=None, w_lo=0.0, w_hi=0.0,
                a_code_scale=0.0, w_code_scale=0.0):
        x = _req(x, "input")
        w = _req(w, "weight")
        ctx.save_for_backward(x, w, w_raw)
        ctx.cfg = (stride, pad, precision, w_lo, w_hi, bias is not None)
        ctx.codes = (a_code_scale, w_code_scale)
        return noisy_conv_fwd(x, w, None, bias, stride, pad, precision=precision,
                              a_code_scale=a_code_scale, w_code_scale=w_code_scale)["y"]

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x, w, w_raw = ctx.saved_tensors
        stride, pad, precision, w_lo, w_hi, has_bias = ctx.cfg
        gy = gy.contiguous()
        a_cs, w_cs = ctx.codes
        gx = gw = gb = gwr = None
        if ctx.needs_input_grad[0]:
            gx = conv_dgrad(gy, w, x.shape, stride, pad, precision=precision, w_code_scale=w_cs)
        if w_raw is not None and ctx.needs_input_grad[6]:
            gwr = conv_wgrad(gy, x, w.shape, stride, pad, w_raw, w_lo, w_hi, precision=precision, a_code_scale=a_cs)
        elif ctx.needs_input_grad[1]:
            gw = conv_wgrad(gy, x, w.shape, stride, pad, precision=precision, a_code_scale=a_cs)
        if has_bias and ctx.needs_input_grad[2]:
            gb = gy.sum((0, 2, 3))
        return gx, gw, gb, None, None, None, gwr, None, None, None, None


class CurrentNoiseFn(Function):
    """y_noisy = y + z * sigma(x, w_raw) -- additive constant in autograd (the reference computes the
    noise under no_grad, hardware_model.py:23, :125): gradient is identity w.r.t. y."""

    @staticmethod
    def forward(ctx, y, x, w_raw, stride, pad, mode, current, scale_dev, stats, z, precision):
        r = noisy_conv_fwd(x, None, w_raw, None, stride, pad, noise_mode=mode, current=current,
                           scale_dev=scale_dev, z=z, stats=stats, precision=precision, y_in=y.detach())
        return r["y_noisy"]

    @staticmethod
    def backward(ctx, g):
        return (g,) + (None,) * 10


class FusedNoisyConvFn(Function):
    """Single launch: (y, y_noisy) = fused noisy conv.  Gradients of both outputs flow to x / w."""

    @staticmethod
    def forward(ctx, x, w, bias, w_raw_noise, stride, pad, mode, current, scale_dev, stats, z, precision,
                w_ste_raw=None, w_lo=0.0, w_hi=0.0, a_code_scale=0.0, w_code_scale=0.0):
        x = _req(x, "input")
        w = _req(w, "weight")
        ctx.save_for_backward(x, w, w_ste_raw)
        ctx.cfg = (stride, pad, precision, w_lo, w_hi, bias is not None)
        ctx.codes = (a_code_scale, w_code_scale)
        r = noisy_conv_fwd(x, w, w_raw_noise, bias, stride, pad, noise_mode=mode, current=current,
                           scale_dev=scale_dev, z=z, stats=stats, precision=precision,
                           a_code_scale=a_code_scale, w_code_scale=w_code_scale)
        return r["y"], r["y_noisy"]

    @staticmethod
    @once_differentiable
    def backward(ctx, gy, gyn):
        x, w, w_raw = ctx.saved_tensors
        stride, pad, precision, w_lo, w_hi, has_bias = ctx.cfg
        if gy is None:
            g = gyn
        elif gyn is None:
            g = gy
        else:
            g = gy + gyn
        g = g.contiguous()
        a_cs, w_cs = ctx.codes
        gx = gw = gb = gwr = None
        if ctx.needs_input_grad[0]:
            gx = conv_dgrad(g, w, x.shape, stride, pad, precision=precision, w_code_scale=w_cs)
        if w_raw is not None and ctx.needs_input_grad[12]:
            gwr = conv_wgrad(g, x, w.shape, stride, pad, w_raw, w_lo, w_hi, precision=precision, a_code_scale=a_cs)
        elif ctx.needs_input_grad[1]:
            gw = conv_wgrad(g, x, w.shape, stride, pad, precision=precision, a_code_scale=a_cs)
        if has_bias and ctx.needs_input_grad[2]:
            gb = g.sum((0, 2, 3))
        return (gx, gw, gb) + (None,) * 9 + (gwr,) + (None,) * 4
