"""The fully connected layers' split-K GEMM (k_conv_umma + k_splitk_epilogue) and conv1's weight gradient
(k_wgrad_shift<NROW> + its reduce), csrc/nn_conv_umma.cu, bit for bit against float64.

The operands are those of test_gpu_tma_sweep.py, whose exact oracle and operand helpers this file imports: activation
codes 0..15, odd weight codes, integer gradients and power-of-two code scales, so every partial sum is an integer below
2^24, the fp32 accumulation is exact in any order and a correct kernel stores exactly _scaled(_exact(float64 result)).
That holds for every split of the k-blocks too, so a split launch must equal the float64 result bit for bit, and a
Philox launch on the lean epilogue (split or not) must equal the generic epilogue's launch with the same rng bit for bit:
the sigma^2 sums are exact, and the square root and the Philox group mapping m * ceil(N / 4) + n / 4 are the same
instructions in all three epilogues.

Every GPU case runs under torch.profiler and asserts which kernels ran.  The profiler does not show the split count or the
weight-gradient plan, so those come from restatements of the host plans (tiled_plan, split_count, wg_shift_plan below),
which the CPU tests pin against the library.
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch

from test_gpu_tma_sweep import (_KERNEL, CURRENT, EXTERNAL, MERGED, NONE, S_A, S_W, SMS_H100, _act_codes, _assert_within,
                                _cdiv, _coef, _exact, _grads, _noisy_ref, _nhwc_bf16, _pad, _scaled, _sigma_sum, _w_codes,
                                _w_raw, dev, lib)  # noqa: F401  (dev, lib: module fixtures)

SMS_NO_DEVICE = 148             # what the library's nn_num_sms answers without a device


# ---------------------------------------------------------------------------------------------- plan restatements

def tiled_plan(cin_k, khw, n_out, sigma, wsum, m_rows, main=True):
    """make_plan (csrc/nn_conv_umma.cu) for a GEMM over khw taps of cin_k channels producing n_out columns (+ the sigma^2
    columns when noisy, + the colsum column with wsum) on m_rows output rows (0: no narrowing, as for weight jobs without
    m_rows).  The forward passes (Cin, KH * KW, Cout), the dgrad (Cout, KH * KW, Cin)."""
    cp = _pad(cin_k, 8)
    num_kb = _cdiv(khw * cp, 64)
    max_nt = (120 if main else 248) if sigma else 256
    n_tiles = _cdiv(n_out, max_nt)
    m_tiles = _cdiv(m_rows, 128)
    if m_tiles > 0:
        while m_tiles * n_tiles < 96 and _cdiv(n_out, n_tiles) > 48:
            n_tiles *= 2
    n_t = _pad(_cdiv(n_out, n_tiles), 8)
    n_tiles = _cdiv(n_out, n_t)
    cols = (n_t if main else 0) + (n_t if sigma else 0) + (1 if wsum else 0)
    n_mma = max(16, _pad(cols, 16))
    stages = max(2, min(4, 192 * 1024 // (128 * 128 + n_mma * 128)))
    stages = min(stages, max(num_kb, 1))
    return dict(cp=cp, n_t=n_t, n_tiles=n_tiles, n_mma=n_mma, num_kb=num_kb, stages=stages,
                wp_bytes=n_tiles * num_kb * n_mma * 64 * 2)


def split_count(pl, m_rows, epi, sms, ohw=1, ws_bytes=None):
    """launch_umma's split-K share count: only the lean epilogues <1> / <2> of linear layers (OH * OW == 1), only when
    2 * CTAs <= SMs and num_kb >= 8; 4 shares, fewer while a share would get fewer than 4 k-blocks; 1 when the split-K
    workspace (ws_bytes; None: room enough) cannot hold the partial sums"""
    m_tiles = _cdiv(m_rows, 128)
    if epi not in (1, 2) or ohw != 1 or 2 * m_tiles * pl["n_tiles"] > sms or pl["num_kb"] < 8:
        return 1
    s = 4
    while s > 1 and pl["num_kb"] // s < 4:
        s -= 1
    if ws_bytes is not None and s * pl["n_tiles"] * pl["n_mma"] * m_tiles * 128 * 4 > ws_bytes:
        return 1
    return s


def shares(num_kb, splits):
    """k-blocks of each split share: ceil(num_kb / splits) each, the rest to the last"""
    per = _cdiv(num_kb, splits)
    return [min(num_kb, (z + 1) * per) - z * per for z in range(splits)]


def linear_bn_fusable(B, cin, khw, cout, noisy, sms):
    """nn_conv_linear_bn_fusable for a linear layer (B samples): the launch splits and M % 256 == 0, M <= 4096"""
    if B % 256 or B > 4096:
        return False
    return split_count(tiled_plan(cin, khw, cout, noisy, False, B), B, 1 if noisy else 2, sms) > 1


def wg_shift_plan(B, cin, H, W, cout, kh, kw, sms, stride=1, pad=0):
    """make_wg_shift_plan and the reduce launch of shift_conv_wgrad (csrc/nn_conv_umma.cu); None where the shift path
    refuses the geometry"""
    if cin > 8 or stride != 1 or pad != 0 or kh > H or kw > W or W >= 2048 or cout > 128:
        return None
    n_planes, n_row = _cdiv(cout, 8), _pad(kw * 8, 16)
    if n_row > 64:
        return None
    total = B * H * W
    plane_stride = _pad(total, 128)
    n_chunks = plane_stride // 128
    b_pixels = _pad(128 + (kh - 1) * W + n_row // 8, 8)
    a_stage, b_stage = n_planes * 128 * 16, _pad(b_pixels * 16, 128)
    fixed = 128 + 16 * 128 * 16 + 16 * 6 + 64
    stages = min(6, (190 * 1024 - fixed) // (a_stage + b_stage))
    if stages < 2:
        return None
    grid = min(sms, n_chunks)
    OH = H - kh + 1
    hw = H * W

    def live(t):
        v0, v1 = t * 128, min(t * 128 + 127, total - 1)
        return v0 // hw != v1 // hw or (v0 % hw) // W < OH

    alive = [live(t) for t in range(n_chunks)]
    khb = 256 // n_row
    kc = kh * kw * 8
    g = 0
    if kc <= 256:
        g = 1
        while g < 32 and cout * 64 * g < 131072 and grid >= 8 * g:
            g *= 2
    return dict(n_row=n_row, khb=khb, passes=_cdiv(kh, khb), stages=stages, grid=grid, n_chunks=n_chunks,
                dead_chunks=alive.count(False),
                dead_ctas=sum(not any(alive[t] for t in range(c, n_chunks, grid)) for c in range(grid)),
                reduce="k_wgrad_tma_reduce" if kc <= 256 else "k_wgrad_umma_reduce2", G=g,
                gy_planes_bytes=n_planes * plane_stride * 16, n_planes=n_planes, plane_stride=plane_stride)


def fwd_names(epi, splits):
    return {"k_conv_umma<%d>" % epi} | ({"k_splitk_epilogue"} if splits > 1 else set())


def wg_names(wp):
    return {"k_wgrad_shift<%d>" % wp["n_row"], wp["reduce"]}


# ---------------------------------------------------------------------------------------------- GPU cases
# linear forward: (B, Cin, k, Cout, noise mode, all generic-epilogue options); the input is B x Cin x k x k, the filter
# k x k (one output position per sample).  Shares by num_kb: 7 -> 1, 8-11 -> 2, 12-15 -> 3, >= 16 -> 4.
FWD = [
    (37, 400, 1, 100, EXTERNAL, True),      # num_kb 7: not split
    (128, 556, 1, 16, MERGED, False),       # num_kb 9 -> 5 / 4, Cin % 8 = 4, ragged last k-block
    (129, 600, 1, 390, EXTERNAL, True),     # 2 m-tiles, num_kb 10 -> 5 / 5
    (129, 500, 1, 100, MERGED, False),      # num_kb 8 -> 4 / 4
    (1, 802, 1, 10, MERGED, True),          # num_kb 13 -> 5 / 5 / 3, Cin % 8 = 2, one row
    (512, 768, 1, 512, EXTERNAL, False),    # num_kb 12 -> 4 / 4 / 4, 16 n-tiles
    (512, 1024, 1, 392, MERGED, False),     # num_kb 16 -> 4 x 4, float4 stores
    (1, 3000, 1, 390, MERGED, False),       # fc1 as a 1 x 1: num_kb 47 -> 12 / 12 / 12 / 11
    (512, 120, 5, 390, EXTERNAL, True),     # fc1 as the step runs it: 120 x 5 x 5, a k-block straddles taps
    (512, 390, 1, 10, EXTERNAL, True),      # fc2: num_kb 7, per-element stores
    (2048, 120, 5, 390, EXTERNAL, False),   # 16 m-tiles: 2 x CTAs > SMs, not split
]

# linear dgrad: (B, n_out, Cout of the layer): gx [B, n_out] = gy [B, Cout] x W
DGRAD = [(512, 3000, 390), (512, 390, 10), (37, 3000, 390), (1, 390, 10), (129, 10, 390), (2048, 10, 100)]

# bn3 statistics from the split-K epilogue: groups of (M, K) that share one scratch per Cout.  390 columns split only up
# to M = 512 on an H100: at M = 1024 they narrow to 13 n-tiles of 32 (8 x 13 CTAs), and 2 x CTAs > SMs
BN = {390: [(256, 1000), (512, 600)], 90: [(256, 520), (512, 1000), (1024, 800), (4096, 520)]}

# conv1 weight gradient: (B, Cin, H, W, Cout, KH, KW, grad_output range)
WGRAD = [
    (2, 3, 9, 9, 8, 1, 1, 8),               # NROW 16: 1 x 1, 2 chunks (G = 1)
    (3, 1, 30, 33, 9, 2, 2, 8),             # 2 x 2, 2970 pixels (G = 4)
    (1, 3, 17, 128, 64, 17, 1, 8),          # 17 x 1: two passes, OH = 1 -> 16 CTAs without a live chunk, 3 stages
    (5, 8, 9, 11, 120, 1, 2, 8),            # 1 x 2, 495 pixels, 8 channels
    (4, 8, 40, 40, 120, 3, 3, 8),           # NROW 32: 3 x 3, 8 channels, 50 chunks (G = 8)
    (8, 3, 32, 32, 128, 4, 4, 8),           # 4 x 4, Cout = 128 (both warpgroups full), 64 chunks (G = 16)
    (2, 1, 11, 60, 65, 9, 3, 8),            # 9 x 3: two passes, 5 stages, 7 CTAs without a live chunk (G = 2)
    (512, 3, 32, 32, 65, 5, 5, 2),          # NROW 48: conv1 at batch 512, 4096 chunks over the SMs (G = 32), 6 stages
    (3, 3, 14, 14, 1, 6, 6, 8),             # 6 x 6: two passes, one output channel, reduce2
    (2, 3, 12, 20, 9, 3, 7, 8),             # NROW 64: 3 x 7, one pass
    (2, 1, 16, 16, 33, 7, 7, 8),            # 7 x 7: two passes, reduce2
    (1, 3, 8, 200, 128, 8, 8, 8),           # 8 x 8: two passes, Cout = 128, 2 stages, 11 CTAs without a live chunk
]


def _fwd_id(c):
    return "B%d-K%dx%d-N%d" % (c[0], c[1], c[2] * c[2], c[3])


# ---------------------------------------------------------------------------------------------- CPU tests

def _lib_sms():
    """the SM count the library plans with: the device's, or the library's answer without one"""
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else SMS_NO_DEVICE


def test_tiled_plan_matches_pack_bytes(lib):
    """tiled_plan's weight image size equals the library's for NN_PACK_TILED forward (every noise mode, with and without
    the colsum row) and dgrad jobs over a range of m_rows"""
    from noisynet_b200._lib import PACK_TILED, WPrepJob
    n = 0
    for cin in (3, 10, 65, 120, 390, 556, 3000):
        for khw in (1, 9, 25):
            for cout in (1, 10, 16, 100, 390, 392, 512, 3000):
                for m_rows in (0, 1, 129, 512, 1024, 2048):
                    for mode, noise, wsum in ((0, NONE, 0), (0, MERGED, 0), (0, EXTERNAL, 0), (0, EXTERNAL, 1), (1, NONE, 0)):
                        jb = WPrepJob()
                        jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.m_rows = cout, cin, khw, mode, m_rows
                        jb.noise_mode, jb.want_wsum, jb.layout = noise, wsum, PACK_TILED
                        if mode == 0:
                            p = tiled_plan(cin, khw, cout, noise != NONE, noise == EXTERNAL and wsum, m_rows)
                        else:
                            p = tiled_plan(cout, khw, cin, False, False, m_rows)
                        assert lib.nn_weight_pack_bytes(C.byref(jb)) == _pad(p["wp_bytes"], 1024), (cin, khw, cout, m_rows, mode, noise)
                        n += 1
    assert n > 1000


def test_engine_linear_plans():
    """the fully connected GEMMs of the benchmarked step (batch 512) on an H100"""
    p = tiled_plan(120, 25, 390, True, False, 512)                 # fc1 forward: 120 x 5 x 5 -> 390, noisy
    assert (_cdiv(512, 128), p["n_tiles"], p["n_t"], 390 - (p["n_tiles"] - 1) * p["n_t"]) == (4, 13, 32, 6)
    assert p["num_kb"] == 47 and split_count(p, 512, 1, SMS_H100) == 4 and shares(47, 4) == [12, 12, 12, 11]
    p = tiled_plan(390, 1, 10, True, False, 512)                   # fc2 forward
    assert p["num_kb"] == 7 and split_count(p, 512, 1, SMS_H100) == 1
    p = tiled_plan(390, 1, 3000, False, False, 512)                # fc1 dgrad as a 390 -> 3000 linear layer
    assert (p["n_tiles"], p["n_t"], 3000 - (p["n_tiles"] - 1) * p["n_t"]) == (24, 128, 56)
    p = tiled_plan(10, 1, 390, False, False, 512)                  # fc2 dgrad
    assert (p["n_tiles"], p["n_t"], 390 - (p["n_tiles"] - 1) * p["n_t"]) == (13, 32, 6)
    assert shares(13, 3) == [5, 5, 3] and split_count(tiled_plan(802, 1, 10, True, False, 1), 1, 1, SMS_H100) == 3


def test_linear_bn_fusable_restated(lib):
    """nn_conv_linear_bn_fusable against the restated split decision (the library's SM count)"""
    from noisynet_b200._lib import PREC_BF16, ConvGeom
    sms, n = _lib_sms(), 0
    for B in (1, 128, 256, 500, 512, 768, 1024, 2048, 4096, 4352):
        for cin, k in ((120, 5), (390, 1), (520, 1), (1000, 1), (3000, 1), (64, 1)):
            for cout in (10, 90, 100, 382, 390, 512):
                for noise in (NONE, MERGED, EXTERNAL):
                    g = ConvGeom(B, cin, k, k, cout, k, k, 1, 0)
                    want = linear_bn_fusable(B, cin, k * k, cout, noise != NONE, sms)
                    assert bool(lib.nn_conv_linear_bn_fusable(C.byref(g), noise, PREC_BF16, 0)) == want, (B, cin, k, cout, noise)
                    n += want
    assert n > 20
    for B, K, cout in [(M, K, cout) for cout, ms in BN.items() for M, K in ms]:
        assert linear_bn_fusable(B, K, 1, cout, False, sms) and linear_bn_fusable(B, K, 1, cout, True, sms)
    assert not linear_bn_fusable(1024, 1000, 1, 390, True, min(sms, SMS_H100))
    # conv layers are never served
    assert lib.nn_conv_linear_bn_fusable(C.byref(ConvGeom(512, 120, 7, 7, 390, 5, 5, 1, 0)), MERGED, PREC_BF16, 0) == 0


def test_wg_shift_plan_restated(lib):
    """nn_conv_wgrad_pack_layout (the shift path serves the geometry) and nn_conv_gy_planes_bytes against wg_shift_plan"""
    from noisynet_b200._lib import PACK_SHIFT, PACK_TILED, PREC_BF16, ConvGeom
    n = 0
    for B, H, W in ((1, 8, 8), (2, 9, 11), (3, 17, 128), (512, 32, 32), (1, 8, 200), (1, 6, 700), (2, 40, 2047), (1, 9, 2048)):
        for cin in (1, 3, 8, 9):
            for cout in (1, 9, 64, 65, 120, 128, 129):
                for kh, kw in ((1, 1), (2, 2), (3, 3), (5, 5), (6, 6), (8, 8), (9, 3), (17, 1), (1, 9), (5, 2)):
                    g = ConvGeom(B, cin, H, W, cout, kh, kw, 1, 0)
                    wp = wg_shift_plan(B, cin, H, W, cout, kh, kw, SMS_NO_DEVICE)
                    assert lib.nn_conv_wgrad_pack_layout(C.byref(g), PREC_BF16, 0) == (PACK_SHIFT if wp else PACK_TILED), \
                        (B, cin, H, W, cout, kh, kw)
                    assert lib.nn_conv_gy_planes_bytes(C.byref(g)) == _cdiv(cout, 8) * _pad(B * H * W, 128) * 16
                    n += wp is not None
    assert n > 500
    for s in (2, 0):        # stride and padding go to the other kernels
        g = ConvGeom(2, 3, 12, 12, 8, 3, 3, 1 + (s == 2), 1 if s == 0 else 0)
        assert lib.nn_conv_wgrad_pack_layout(C.byref(g), PREC_BF16, 0) == PACK_TILED


def test_default_workspace_holds_the_split(lib):
    """nn_conv_workspace_bytes leaves room for the partial sums of every split forward case (so the ops.noisy_conv_fwd
    launches below split as split_count says), including its 1024-byte alignment"""
    from noisynet_b200._lib import PREC_BF16, ConvGeom
    for B, cin, k, cout, mode, full in FWD:
        ws = lib.nn_conv_workspace_bytes(C.byref(ConvGeom(B, cin, k, k, cout, k, k, 1, 0)), PREC_BF16)
        for sigma in (False, True):
            p = tiled_plan(cin, k * k, cout, sigma, False, B)
            rest = ws - 1023 - _pad(B * k * k * p["cp"] * 2, 1024) - _pad(p["wp_bytes"], 1024)
            s = split_count(p, B, 1 if sigma else 2, SMS_H100)
            assert split_count(p, B, 1 if sigma else 2, SMS_H100, ws_bytes=rest) == s, (B, cin, k, cout, sigma)


def test_sweep_covers_every_cell():
    """the GPU cases reach every epilogue x split count, both generic-epilogue option sets, every NROW with one and two
    passes, both reduces, every reduce group count and every ring depth (on an H100)"""
    lean = set()
    for B, cin, k, cout, mode, full in FWD:
        for sigma, epi in ((False, 2), (True, 1)):
            lean.add((epi, split_count(tiled_plan(cin, k * k, cout, sigma, False, B), B, epi, SMS_H100)))
    assert lean == {(e, s) for e in (1, 2) for s in (1, 2, 3, 4)}
    assert {c[4] for c in FWD if c[5]} == {MERGED, EXTERNAL}
    assert {_pad(c[1], 8) % 64 != 0 for c in FWD} == {True, False} and any(c[1] % 8 for c in FWD)
    assert {_cdiv(c[0], 128) for c in FWD} >= {1, 2, 4, 16} and {c[3] for c in FWD} >= {10, 16, 100, 390, 392, 512}
    uneven = set()
    for B, cin, k, cout, mode, full in FWD:
        p = tiled_plan(cin, k * k, cout, True, False, B)
        s = split_count(p, B, 1, SMS_H100)
        uneven.add(tuple(shares(p["num_kb"], s)))
    assert {(5, 5, 3), (12, 12, 12, 11), (5, 4)} <= uneven
    assert {tiled_plan(c, 1, n, False, False, B)["n_tiles"] for B, n, c in DGRAD} >= {24, 13}
    wps = [wg_shift_plan(B, cin, H, W, cout, kh, kw, SMS_H100) for B, cin, H, W, cout, kh, kw, r in WGRAD]
    assert all(wps)
    assert {(w["n_row"], w["passes"]) for w in wps} == {(n, p) for n in (16, 32, 48, 64) for p in (1, 2)}
    assert {w["reduce"] for w in wps} == {"k_wgrad_tma_reduce", "k_wgrad_umma_reduce2"}
    assert {w["G"] for w in wps if w["G"]} == {1, 2, 4, 8, 16, 32}
    assert {w["stages"] for w in wps} == set(range(2, 7))
    assert any(w["dead_ctas"] for w in wps) and any(w["grid"] < SMS_H100 for w in wps)
    assert any((B * H * W) % 128 for B, cin, H, W, cout, kh, kw, r in WGRAD)
    assert {c[4] for c in WGRAD} >= {1, 8, 9, 64, 65, 120, 128} and {c[1] for c in WGRAD} == {1, 3, 8}
    assert {cout for cout in BN} == {390, 90} and {M for ms in BN.values() for M, K in ms} == {256, 512, 1024, 4096}


# ---------------------------------------------------------------------------------------------- GPU helpers

def _profiled(fn):
    """fn() under torch.profiler -> (its result, the conv / wgrad kernels recorded).  The session first runs one marker
    kernel and waits 10 ms: late in the whole GPU suite the profiler was seen to start recording only after the first
    kernels of a session (and to report them in a later one)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.cuda._sleep(1000)
        torch.cuda.synchronize()
        time.sleep(0.01)
        out = fn()
        torch.cuda.synchronize()
    seen = set()
    for e in prof.events():
        m = _KERNEL.search(e.name) if e.device_type == torch.autograd.DeviceType.CUDA else None
        if m:
            seen.add(m.group(1) + (m.group(2) or ""))
    return out, seen


def _launch(expect, fn):
    """runs fn under torch.profiler: the conv / wgrad kernels it launched must be exactly `expect`, and the pipeline
    watchdog flag clear.  The routing is deterministic, so a session whose kernel set differs is profiled again, up to three
    times in all (every fn here recomputes the same outputs from the same inputs): a wrong routing fails every time."""
    from noisynet_b200 import ops
    for _ in range(3):
        out, seen = _profiled(fn)
        assert ops.error_flag() == 0
        if seen == set(expect):
            break
    assert seen == set(expect), (sorted(seen), sorted(expect))
    return out


def _tma_a(lib_, on):
    """A by the tensor-map row copy (on, the default) or by the cp.async gather; returns the previous setting"""
    return lib_.nn_debug_tma_enable(1 if on else 0)


def _scale_dev(dev):
    return torch.tensor([0.75], device=dev)


class Linear:
    """one linear-layer problem on the device: codes, the float64 results and the launches through ops"""

    def __init__(self, dev, B, cin, k, cout, mode, seed):
        self.dev, self.B, self.cin, self.k, self.cout, self.mode = dev, B, cin, k, cout, mode
        gen = torch.Generator().manual_seed(seed)
        self.ka = _act_codes((B, cin, k, k), gen).to(dev)
        self.cw = _w_codes((cout, cin, k, k), gen).to(dev)
        self.wr = _w_raw((cout, cin, k, k), gen).to(dev)
        self.x, self.w = self.ka * S_A, self.cw * S_W
        self.y_int = _exact(self.ka.reshape(B, -1).double() @ self.cw.reshape(cout, -1).double().t()).reshape(B, cout, 1, 1)
        self.y = _scaled(self.y_int, S_A * S_W)
        self.s = _sigma_sum(self.ka, self.wr, mode, 1, 0)
        self.scale = _scale_dev(dev)
        self.z = torch.randn(B, cout, 1, 1, generator=gen).to(dev)

    def plan(self, sigma, wsum=False, main=True):
        return tiled_plan(self.cin, self.k * self.k, self.cout, sigma, wsum, self.B, main)

    def fwd(self, expect, noisy=True, **kw):
        from noisynet_b200 import ops
        if noisy:
            kw.update(w_raw=self.wr, noise_mode=self.mode, current=CURRENT, scale_dev=self.scale)
        w = kw.pop("w_eff", self.w)
        return _launch(expect, lambda: ops.noisy_conv_fwd(self.x, w, precision="bf16", a_code_scale=S_A, w_code_scale=S_W, **kw))


# ---------------------------------------------------------------------------------------------- GPU tests: linear forward

@pytest.mark.gpu
@pytest.mark.parametrize("case", FWD, ids=_fwd_id)
def test_linear_forward(dev, case):
    """plain <2> exact, Philox <1> (with and without the clean copy) bit-identical to the generic <0> launch with the same
    rng, whose exported draws satisfy the oracle bound -- split as split_count says, with A by the tensor map and by the
    gather; repeated launches bit-equal"""
    from noisynet_b200 import _lib, ops
    B, cin, k, cout, mode, full = case
    L = Linear(dev, B, cin, k, cout, mode, 1000 + B + cin + cout)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n2 = split_count(L.plan(False), B, 2, sms)
    n1 = split_count(L.plan(True), B, 1, sms)
    lib_ = _lib.load()
    rng = ops._fixed_rng(77 + cout, 3)
    ref = L.fwd({"k_conv_umma<0>"}, rng=rng, want_z=True)
    assert torch.equal(ref["y"], L.y)
    _assert_within(ref["y_noisy"], *_noisy_ref(L.y, L.s, ref["z"], _coef()))
    for tma in (True, False):
        prev = _tma_a(lib_, tma)
        try:
            y = L.fwd(fwd_names(2, n2), noisy=False)["y"]
            assert torch.equal(y, L.y), tma
            o1 = L.fwd(fwd_names(1, n1), rng=rng, want_y=False)["y_noisy"]
            assert torch.equal(o1, ref["y_noisy"]), tma
            r1 = L.fwd(fwd_names(1, n1), rng=rng)
            assert torch.equal(r1["y_noisy"], ref["y_noisy"]) and torch.equal(r1["y"], L.y), tma
            if tma:
                assert torch.equal(L.fwd(fwd_names(2, n2), noisy=False)["y"], y)
                assert torch.equal(L.fwd(fwd_names(1, n1), rng=rng, want_y=False)["y_noisy"], o1)
        finally:
            _tma_a(lib_, prev)
    # injected draws on the generic epilogue
    yn = L.fwd({"k_conv_umma<0>"}, z=L.z, want_y=False)["y_noisy"]
    _assert_within(yn, *_noisy_ref(L.y, L.s, L.z, _coef()))
    if full:
        _generic_options(L)


def _generic_options(L):
    """<0> with bias, with z and sigma exported, with the power statistics (both noise modes), and the noise-only launch"""
    dev, B, cout = L.dev, L.B, L.cout
    from noisynet_b200 import ops
    gen = torch.Generator().manual_seed(cout)
    bias = (torch.randint(-64, 65, (cout,), generator=gen).float() / 8.0).to(dev)
    yb = L.fwd({"k_conv_umma<0>"}, noisy=False, bias=bias)["y"]
    assert torch.equal(yb, L.y + bias.view(1, -1, 1, 1))
    r = L.fwd({"k_conv_umma<0>"}, rng=ops._fixed_rng(5, cout), want_z=True, want_sigma=True)
    sig_ref = torch.sqrt(_coef() * (L.s * S_A))
    _assert_within(r["sigma"], sig_ref, 2.0 ** -21 * sig_ref + 1e-30)
    assert torch.equal(r["y_noisy"], r["y"] + r["z"] * r["sigma"]) and torch.equal(r["y"], L.y)
    # noise-only: the clean output is an input, the plan has no main columns (248-column n-tiles)
    r2 = L.fwd({"k_conv_umma<0>"}, w_eff=None, z=L.z, y_in=L.y)
    _assert_within(r2["y_noisy"], *_noisy_ref(L.y, L.s, L.z, _coef()))
    # power statistics: [sum of S (MERGED) or of x (*) colsum|w| (EXTERNAL), sum |z sigma|, max y]
    for mode in (MERGED, EXTERNAL):
        L.mode, L.s = mode, _sigma_sum(L.ka, L.wr, mode, 1, 0)
        stats = torch.tensor([0.0, 0.0, float("-inf")], device=dev)
        yn = L.fwd({"k_conv_umma<0>"}, z=L.z, stats=stats)["y_noisy"]
        ref, tol = _noisy_ref(L.y, L.s, L.z, _coef())
        _assert_within(yn, ref, tol)
        if mode == MERGED:
            plain = (L.s * S_A).sum()
        else:       # one colsum row per n-tile: bf16(sum over the tile's rows of |w_raw|), k by k
            nt = L.plan(True, wsum=True)["n_t"]
            a = L.wr.abs().reshape(cout, -1).double()
            cs = torch.stack([a[t:t + nt].sum(0) for t in range(0, cout, nt)]).float().bfloat16().double()
            plain = (L.ka.reshape(B, -1).double() @ cs.t()).sum() * S_A
        got = stats.tolist()
        assert got[0] == pytest.approx(plain.item(), rel=1e-4), mode
        assert got[1] == pytest.approx((ref - L.y.double()).abs().sum().item(), rel=1e-4), mode
        assert got[2] == L.y.max().item(), mode


def _fwd_abi(L, noisy, rng, ws_bytes=None, bn=None, out=None, check=True):
    """the forward through the C ABI with an explicit workspace (None: nn_conv_workspace_bytes); returns rc, output,
    workspace (check: raise with the library's message unless rc == 0)"""
    from noisynet_b200 import _lib
    from noisynet_b200._lib import PREC_BF16, ConvFwdArgs, ConvGeom
    lib_ = _lib.load()
    g = ConvGeom(L.B, L.cin, L.k, L.k, L.cout, L.k, L.k, 1, 0)
    y = torch.empty(L.B, L.cout, 1, 1, device=L.dev) if out is None else out
    a = ConvFwdArgs()
    a.g, a.x, a.w_eff = g, L.x.data_ptr(), L.w.data_ptr()
    if noisy:
        a.w_raw, a.y_noisy, a.noise_mode, a.current, a.scale_dev, a.rng = \
            L.wr.data_ptr(), y.data_ptr(), L.mode, CURRENT, L.scale.data_ptr(), rng
    else:
        a.y = y.data_ptr()
    a.precision, a.a_code_scale, a.w_code_scale = PREC_BF16, S_A, S_W
    if ws_bytes is None:
        ws_bytes = int(lib_.nn_conv_workspace_bytes(C.byref(g), PREC_BF16))
    ws = torch.full((ws_bytes,), 0x5A, dtype=torch.uint8, device=L.dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    if bn is not None:
        a.bn_mean, a.bn_invstd, a.bn_running_mean, a.bn_running_var = (t.data_ptr() for t in bn[:4])
        a.bn_eps, a.bn_momentum, a.bn_eval_mode, a.bn_scratch, a.zero_out = 1e-5, 0.1, bn[4], bn[5].data_ptr(), bn[6].data_ptr()
    rc = lib_.nn_noisy_conv_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream)
    if check:
        _lib.check(rc, "nn_noisy_conv_fwd (B %d, K %d, N %d, workspace %d bytes)" % (L.B, L.cin * L.k * L.k, L.cout, ws_bytes))
    return rc, y, ws


def _packs_only(L, sigma):
    """a workspace that holds the operand packs and nothing else: no room for split-K partial sums"""
    p = L.plan(sigma)
    return _pad(L.B * L.k * L.k * p["cp"] * 2, 1024) + _pad(p["wp_bytes"], 1024) + 1024


@pytest.mark.gpu
@pytest.mark.parametrize("case", [FWD[4], FWD[8]], ids=_fwd_id)
def test_workspace_fallback_unsplit(dev, case):
    """without room for the partial sums the launch is not split, and its output is bit-identical to the split launch's"""
    from noisynet_b200 import _lib, ops
    B, cin, k, cout, mode, full = case
    L = Linear(dev, B, cin, k, cout, mode, 2000 + cout)
    rng = ops._fixed_rng(31, 1)
    for noisy, epi in ((False, 2), (True, 1)):
        assert split_count(L.plan(noisy), B, epi, _lib_sms()) > 1
        assert split_count(L.plan(noisy), B, epi, _lib_sms(), ws_bytes=1024) == 1
        rc, ys, _ = _launch(fwd_names(epi, split_count(L.plan(noisy), B, epi, _lib_sms())), lambda: _fwd_abi(L, noisy, rng))
        assert rc == 0
        rc, y1, _ = _launch(fwd_names(epi, 1), lambda: _fwd_abi(L, noisy, rng, ws_bytes=_packs_only(L, noisy)))
        assert rc == 0
        assert torch.equal(ys, y1)
        if not noisy:
            assert torch.equal(ys, L.y)


# ---------------------------------------------------------------------------------------------- GPU tests: bn3 statistics

def _bn_ref(y):
    """E[y] and E[y^2] - E[y]^2 over the rows, in float64 (the kernel's formula)"""
    y = y.reshape(y.shape[0], -1).double()
    m = y.sum(0) / y.shape[0]
    return m, ((y * y).sum(0) / y.shape[0] - m * m).clamp_min(0.0)


def _check_bn(y, mean, invstd):
    m, var = _bn_ref(y)
    rms = (y.reshape(y.shape[0], -1).double() ** 2).mean(0).sqrt()
    assert ((mean.double() - m).abs() <= 2.0 ** -22 * m.abs() + 1e-13 * rms).all()
    inv = 1.0 / torch.sqrt(var + float(np.float32(1e-5)))
    assert ((invstd.double() - inv).abs() <= 2.0 ** -21 * inv).all()
    return m, var


@pytest.mark.gpu
@pytest.mark.parametrize("cout", sorted(BN))
def test_linear_bn_statistics_exact(dev, cout):
    """mean / invstd from the split-K epilogue against float64 statistics of the exact outputs, M = 256 .. 4096 (1 .. 16
    slices) on ONE scratch (the arrival counters reset themselves), the running statistics after two launches, eval mode,
    zero_out, and the noisy launch's statistics of its own output"""
    from noisynet_b200 import _lib, ops
    lib_ = _lib.load()
    scratch = torch.zeros(int(lib_.nn_stage_scratch_bytes(cout)) + 64, dtype=torch.uint8, device=dev)
    mean, invstd = torch.empty(cout, device=dev), torch.empty(cout, device=dev)
    zero = torch.empty(1, device=dev)
    mom = float(np.float32(0.1))
    for M, K in BN[cout]:
        L = Linear(dev, M, K, 1, cout, MERGED, 3000 + M + K)
        n = split_count(L.plan(False), M, 2, _lib_sms())
        assert n > 1
        rm, rv = torch.zeros(cout, device=dev), torch.ones(cout, device=dev)
        bn = [mean, invstd, rm, rv, 0, scratch, zero]
        rm_ref, rv_ref = np.zeros(cout), np.ones(cout)
        for rep in range(2):
            zero.fill_(3.0)
            before = rm.clone(), rv.clone()     # (a launch profiled again must update from the same state)
            rc, y, _ = _launch(fwd_names(2, n), lambda: (rm.copy_(before[0]), rv.copy_(before[1]),
                                                         _fwd_abi(L, False, None, bn=bn))[-1])
            assert rc == 0 and torch.equal(y, L.y) and zero.item() == 0.0
            m, var = _check_bn(y, mean, invstd)
            m, unb = m.cpu().numpy(), (var * M / (M - 1)).cpu().numpy()
            rm_ref = ((1.0 - mom) * rm_ref.astype(np.float32) + mom * m).astype(np.float32)
            rv_ref = ((1.0 - mom) * rv_ref.astype(np.float32) + mom * unb).astype(np.float32)
            assert np.allclose(rm.cpu().numpy(), rm_ref, rtol=2.0 ** -21, atol=1e-12)
            assert np.allclose(rv.cpu().numpy(), rv_ref, rtol=2.0 ** -21, atol=1e-12)
        # eval mode: the running statistics normalise, nothing updates
        rm0, rv0 = rm.clone(), rv.clone()
        bn[4] = 1
        zero.fill_(3.0)
        rc, y, _ = _launch(fwd_names(2, n), lambda: _fwd_abi(L, False, None, bn=bn))
        assert rc == 0 and torch.equal(y, L.y) and zero.item() == 0.0
        assert torch.equal(mean, rm0) and torch.equal(rm, rm0) and torch.equal(rv, rv0)
        inv = (1.0 / np.sqrt(rv0.cpu().numpy().astype(np.float64) + float(np.float32(1e-5)))).astype(np.float32)
        assert np.allclose(invstd.cpu().numpy(), inv, rtol=2.0 ** -23, atol=0)
        # noisy (Philox <1>): statistics of the output it wrote, which equals the generic launch's
        bn[4] = 0
        n1 = split_count(L.plan(True), M, 1, _lib_sms())
        rng = ops._fixed_rng(M, K)
        rc, yn, _ = _launch(fwd_names(1, n1), lambda: _fwd_abi(L, True, rng, bn=bn))
        assert rc == 0
        _check_bn(yn, mean, invstd)
        assert torch.equal(yn, L.fwd({"k_conv_umma<0>"}, rng=rng, want_z=True)["y_noisy"])


@pytest.mark.gpu
def test_linear_bn_refusals_write_nothing(dev):
    """bn_mean calls the split-K epilogue cannot serve return an error before any launch: outputs, statistics and the
    workspace keep their sentinel values (M % 256 != 0, M > 4096, a workspace without room for the split)"""
    from noisynet_b200 import _lib
    lib_ = _lib.load()
    cout = 90
    scratch = torch.zeros(int(lib_.nn_stage_scratch_bytes(cout)) + 64, dtype=torch.uint8, device=dev)
    for M, K, ws_for in ((500, 520, None), (4352, 520, None), (512, 1000, "packs")):
        L = Linear(dev, M, K, 1, cout, MERGED, 4000 + M)
        for noisy in (False, True):
            stats = [torch.full((cout,), 7.0, device=dev) for _ in range(4)]
            zero = torch.full((1,), 3.0, device=dev)
            out = torch.full((M, cout, 1, 1), 5.0, device=dev)
            from noisynet_b200 import ops
            rc, y, ws = _launch(set(), lambda: _fwd_abi(L, noisy, ops._fixed_rng(1, 1), out=out, check=False,
                                                        ws_bytes=_packs_only(L, noisy) if ws_for else None,
                                                        bn=stats + [0, scratch, zero]))
            torch.cuda.synchronize()
            assert rc != 0, (M, noisy)
            assert bool((out == 5.0).all()) and all(bool((t == 7.0).all()) for t in stats) and zero.item() == 3.0
            assert bool((ws == 0x5A).all()), (M, noisy)
            assert lib_.nn_last_error()


# ---------------------------------------------------------------------------------------------- GPU tests: linear dgrad

@pytest.mark.gpu
@pytest.mark.parametrize("case", DGRAD, ids=lambda c: "B%d-%dx%d" % c)
def test_linear_dgrad(dev, case):
    """<2> without a mask equals the float64 product; with x_pre, <0> equals it with the masked entries zeroed; both A
    paths"""
    from noisynet_b200 import _lib, ops
    B, n_out, cout = case
    gen = torch.Generator().manual_seed(5000 + B + n_out)
    cw = _w_codes((cout, n_out, 1, 1), gen).to(dev)
    gy = _grads((B, cout, 1, 1), gen).to(dev)
    x_pre = (torch.randn(B, n_out, 1, 1, generator=gen) * 0.6).to(dev)
    r = _exact(gy.reshape(B, cout).double() @ cw.reshape(cout, n_out).double()).reshape(B, n_out, 1, 1)
    want = _scaled(r, S_W)
    keep = (x_pre >= -0.5) & (x_pre <= 0.5)
    lib_ = _lib.load()
    w = cw * S_W
    for tma in (True, False):
        prev = _tma_a(lib_, tma)
        try:
            gx = _launch({"k_conv_umma<2>"}, lambda: ops.conv_dgrad(gy, w, (B, n_out, 1, 1), precision="bf16", w_code_scale=S_W))
            assert torch.equal(gx, want), tma
            gxm = _launch({"k_conv_umma<0>"}, lambda: ops.conv_dgrad(gy, w, (B, n_out, 1, 1), x_pre=x_pre, x_lo=-0.5, x_hi=0.5,
                                                                     precision="bf16", w_code_scale=S_W))
            assert torch.equal(gxm, torch.where(keep, want, torch.zeros_like(want))), tma
        finally:
            _tma_a(lib_, prev)
    assert torch.equal(gx, _launch({"k_conv_umma<2>"}, lambda: ops.conv_dgrad(gy, w, (B, n_out, 1, 1), precision="bf16",
                                                                               w_code_scale=S_W)))


# ---------------------------------------------------------------------------------------------- GPU tests: packed operands

@pytest.mark.gpu
def test_packed_operands_fc(dev):
    """the engine's fc operands through the C ABI at batch 512: NN_PACK_TILED images from nn_prepare_weights (4-bit,
    round to nearest) for fc1 (120 x 5 x 5 -> 390) and fc2 forward, and for the dgrads of fc2 and of fc1 as a 390 -> 3000
    linear layer; NHWC bf16 code images.  fc1 runs split 4 ways with bn_mean, as in the training step."""
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import (PACK_TILED, PREC_BF16, ConvDgradArgs, ConvFwdArgs, ConvGeom, Rng, WPrepJob)
    from oracle import noisynet_oracle as O
    lib_ = _lib.load()
    B = 512
    st = torch.cuda.current_stream().cuda_stream
    gen = torch.Generator().manual_seed(512)
    w_cs = float(np.float32(2.0 / 15.0)) / 2.0
    wr1, wr2 = _w_raw((390, 120, 5, 5), gen).to(dev), _w_raw((10, 390, 1, 1), gen).to(dev)
    codes = []
    for wr in (wr1, wr2):
        c = torch.round(O.uniform_quantize_fwd(wr.cpu(), 4, -1.0, 1.0).double() / w_cs)
        assert bool((c.remainder(2) == 1).all())
        codes.append(c.to(dev))
    g1, g2 = ConvGeom(B, 120, 5, 5, 390, 5, 5, 1, 0), ConvGeom(B, 390, 1, 1, 10, 1, 1, 1, 0)
    g1_lin = ConvGeom(B, 3000, 1, 1, 390, 1, 1, 1, 0)
    assert lib_.nn_conv_pack_layout(C.byref(g1), EXTERNAL, PREC_BF16) == PACK_TILED
    assert lib_.nn_conv_pack_layout(C.byref(g2), EXTERNAL, PREC_BF16) == PACK_TILED
    specs = [(wr1, (390, 120, 25), 0, EXTERNAL, 0), (wr2, (10, 390, 1), 0, EXTERNAL, 1),
             (wr2, (10, 390, 1), 1, NONE, 1), (wr1, (390, 3000, 1), 1, NONE, 0)]
    jobs = (WPrepJob * 4)()
    scratch = [torch.zeros(wr.numel() + 16, dtype=torch.int8, device=dev) for wr in (wr1, wr2)]
    bufs = []
    for j, (wr, (co, ci, khw), mode, noise, layer) in enumerate(specs):
        jb = jobs[j]
        jb.w_raw, jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.m_rows = wr.data_ptr(), co, ci, khw, mode, B
        jb.noise_mode, jb.want_wsum, jb.layout = noise, 0, PACK_TILED
        jb.q_bits, jb.q_hi, jb.stochastic, jb.u_inject, jb.rng = 4, 1.0, 0.0, None, Rng(0, 0, None)
        jb.codes = scratch[layer].data_ptr()
        buf = torch.zeros(int(lib_.nn_weight_pack_bytes(C.byref(jb))) + 1024, dtype=torch.uint8, device=dev)
        jb.packed_out = (buf.data_ptr() + 1023) // 1024 * 1024
        bufs.append(buf)
    _lib.check(lib_.nn_prepare_weights(jobs, 4, 0, st), "nn_prepare_weights")
    ws = torch.empty(max(int(lib_.nn_conv_workspace_bytes(C.byref(g), PREC_BF16)) for g in (g1, g2, g1_lin)) + 4096,
                     dtype=torch.uint8, device=dev)
    scale = _scale_dev(dev)

    ka3, ka4 = _act_codes((B, 120, 5, 5), gen).to(dev), _act_codes((B, 390, 1, 1), gen).to(dev)
    for layer, (g, ka, c, wr, job) in enumerate(((g1, ka3, codes[0], wr1, 0), (g2, ka4, codes[1], wr2, 1))):
        p = tiled_plan(g.Cin, g.KH * g.KW, g.Cout, True, False, B)
        n1 = split_count(p, B, 1, _lib_sms())
        assert n1 == (4 if layer == 0 else 1)
        yn = torch.empty(B, g.Cout, 1, 1, device=dev)
        a = ConvFwdArgs()
        a.g, a.y_noisy, a.noise_mode, a.current, a.scale_dev = g, yn.data_ptr(), EXTERNAL, CURRENT, scale.data_ptr()
        a.rng, a.precision, a.a_code_scale, a.w_code_scale = ops._fixed_rng(9, layer), PREC_BF16, S_A, w_cs
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        xp = _nhwc_bf16(ka, _pad(g.Cin, 8))
        a.x_packed, a.w_packed, a.w_packed_layout = xp.data_ptr(), jobs[job].packed_out, PACK_TILED
        if layer == 0:
            bn = [torch.empty(390, device=dev), torch.empty(390, device=dev), torch.zeros(390, device=dev), torch.ones(390, device=dev)]
            bn_scratch = torch.zeros(int(lib_.nn_stage_scratch_bytes(390)) + 64, dtype=torch.uint8, device=dev)
            a.bn_mean, a.bn_invstd, a.bn_running_mean, a.bn_running_var = (t.data_ptr() for t in bn)
            a.bn_eps, a.bn_momentum, a.bn_scratch = 1e-5, 0.1, bn_scratch.data_ptr()
        _launch(fwd_names(1, n1), lambda: _lib.check(lib_.nn_noisy_conv_fwd(C.byref(a), 0, st), "nn_noisy_conv_fwd"))
        # the same draws on the generic epilogue with unpacked operands, and its exported z against the oracle
        r0 = _launch({"k_conv_umma<0>"}, lambda: ops.noisy_conv_fwd(
            ka * S_A, (c * w_cs).float(), wr, None, 1, 0, noise_mode=EXTERNAL, current=CURRENT, scale_dev=scale,
            precision="bf16", a_code_scale=S_A, w_code_scale=w_cs, rng=ops._fixed_rng(9, layer), want_z=True))
        y = _scaled(_exact(ka.reshape(B, -1).double() @ c.reshape(g.Cout, -1).t()), np.float32(S_A) * np.float32(w_cs))
        assert torch.equal(r0["y"], y.reshape(B, g.Cout, 1, 1))
        assert torch.equal(yn, r0["y_noisy"]), layer
        _assert_within(yn, *_noisy_ref(r0["y"], _sigma_sum(ka, wr, EXTERNAL, 1, 0), r0["z"], _coef()))
        if layer == 0:
            _check_bn(yn, bn[0], bn[1])

    # dgrads: fc2 (10 -> 390) and fc1 as a linear layer (390 -> 3000), packed grad_output [B][Coutp] bf16
    for g, c, job in ((g2, codes[1], 2), (g1_lin, codes[0], 3)):
        n_out, cout = g.Cin, g.Cout
        gy = _grads((B, cout), gen).to(dev)
        gyp = _nhwc_bf16(gy.reshape(B, cout, 1, 1), _pad(cout, 8))
        gx = torch.empty(B, n_out, 1, 1, device=dev)
        d = ConvDgradArgs()
        d.g, d.gx, d.precision, d.w_code_scale = g, gx.data_ptr(), PREC_BF16, w_cs
        d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
        d.gy_packed, d.w_packed, d.w_packed_layout = gyp.data_ptr(), jobs[job].packed_out, PACK_TILED
        _launch({"k_conv_umma<2>"}, lambda: _lib.check(lib_.nn_noisy_conv_dgrad(C.byref(d), 0, st), "nn_noisy_conv_dgrad"))
        r = _exact(gy.double() @ c.reshape(cout, n_out))
        assert torch.equal(gx.reshape(B, n_out), _scaled(r, w_cs)), n_out
    assert ops.error_flag() == 0


# ---------------------------------------------------------------------------------------------- GPU tests: conv1 wgrad

def _gy_planes(gy, H, W, wp):
    """grad_output in the NN_PACK_SHIFT planes layout: [channel chunk][pixel of the input grid, padded][8] bf16, zeros at
    positions that are not outputs"""
    B, cout, OH, OW = gy.shape
    n = wp["n_planes"]
    full = torch.zeros(B, n * 8, H, W, device=gy.device)
    full[:, :cout, :OH, :OW] = gy
    planes = torch.zeros(n, wp["plane_stride"], 8, dtype=torch.bfloat16, device=gy.device)
    planes[:, :B * H * W] = full.reshape(B, n, 8, H, W).permute(1, 0, 3, 4, 2).reshape(n, B * H * W, 8).to(torch.bfloat16)
    return planes


@pytest.mark.gpu
@pytest.mark.parametrize("case", WGRAD, ids=lambda c: "B%d-C%d-%dx%d-N%d-%dx%d" % c[:7])
def test_conv1_wgrad(dev, case):
    """k_wgrad_shift<NROW> + its reduce exactly: grad_output as fp32 (packed to planes by the library) and as the engine's
    NN_PACK_SHIFT planes with the NHWC code image; the STE-masked variant; a repeat bit-equal"""
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import PACK_SHIFT, PREC_BF16, ConvGeom, ConvWgradArgs
    B, cin, H, W, cout, kh, kw, r = case
    wp = wg_shift_plan(B, cin, H, W, cout, kh, kw, torch.cuda.get_device_properties(0).multi_processor_count)
    lib_ = _lib.load()
    g = ConvGeom(B, cin, H, W, cout, kh, kw, 1, 0)
    assert lib_.nn_conv_wgrad_pack_layout(C.byref(g), PREC_BF16, 0) == PACK_SHIFT
    gen = torch.Generator().manual_seed(6000 + sum(case))
    OH, OW = H - kh + 1, W - kw + 1
    ka = _act_codes((B, cin, H, W), gen).to(dev)
    gy = torch.randint(-r, r + 1, (B, cout, OH, OW), generator=gen).float().to(dev)
    w_shape = (cout, cin, kh, kw)
    bound = torch.nn.grad.conv2d_weight(ka.abs().double(), w_shape, gy.abs().double())
    assert bound.max().item() < 2 ** 24
    want = _scaled(_exact(torch.nn.grad.conv2d_weight(ka.double(), w_shape, gy.double())), S_A)
    names = wg_names(wp)
    gw = _launch(names, lambda: ops.conv_wgrad(gy, ka * S_A, w_shape, precision="bf16", a_code_scale=S_A))
    assert torch.equal(gw, want)
    w_raw = (torch.randn(w_shape, generator=gen) * 0.8).to(dev)
    gwm = _launch(names, lambda: ops.conv_wgrad(gy, ka * S_A, w_shape, w_raw=w_raw, w_lo=-1.0, w_hi=1.0, precision="bf16",
                                                a_code_scale=S_A))
    assert torch.equal(gwm, torch.where((w_raw >= -1.0) & (w_raw <= 1.0), want, torch.zeros_like(want)))
    # the engine's operands: planes + NHWC codes (Cp = 8)
    planes, xp = _gy_planes(gy, H, W, wp), _nhwc_bf16(ka, 8)
    assert planes.numel() * 2 == lib_.nn_conv_gy_planes_bytes(C.byref(g))
    ws = torch.empty(int(lib_.nn_conv_wgrad_workspace_bytes(C.byref(g), PREC_BF16, 0)) + 4096, dtype=torch.uint8, device=dev)
    gwp = torch.empty(w_shape, device=dev)
    a = ConvWgradArgs()
    a.g, a.gw, a.precision, a.a_code_scale = g, gwp.data_ptr(), PREC_BF16, S_A
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    a.x_packed, a.gy_packed, a.gy_packed_layout = xp.data_ptr(), planes.data_ptr(), PACK_SHIFT
    st = torch.cuda.current_stream().cuda_stream
    for rep in range(2):
        gwp.fill_(float("nan"))
        _launch(names, lambda: _lib.check(lib_.nn_noisy_conv_wgrad(C.byref(a), 0, st), "nn_noisy_conv_wgrad"))
        assert torch.equal(gwp, want), rep
    assert torch.equal(gw, _launch(names, lambda: ops.conv_wgrad(gy, ka * S_A, w_shape, precision="bf16", a_code_scale=S_A)))
