"""Every accumulator width, tap-pair chain shape and tile schedule of the shift-GEMM forward k_conv_shift, in all three
modes (plain, Philox noise, injected z), pooled and not.

Operands are integer codes (activation codes 0..15, odd weight codes -15..15, each times one fp32 scale), so every
partial sum of the main contraction is an integer below 2^24: the float64 reference, multiplied once by the fp32 scales,
is what a correct kernel stores (rtol 1e-6 covers the one final multiply).  The plain output must also be bit-identical to the tiled
tensor-core kernel's (nn_debug_shift_enable(0)) and to a repeated launch.  sigma comes from the same bf16 operands with an
fp32 sum, so the noisy output agrees with the tiled kernel's to the sigma tolerance of test_gpu_shift.py.  Pooled launches
are checked against a MaxPool of the same mode's unfused output (values and first-maximum window position, exactly) and the
BatchNorm statistics against float64.  Each launch runs under torch.profiler and asserts the k_conv_shift instantiation,
because the layer would otherwise be served by another kernel without a word.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__ as entry
    entry.build()
    return torch.device("cuda:0")


def _pad(v, m):
    return (v + m - 1) // m * m


def n_mma(cout, noisy):
    """the shift plan's accumulator width (make_shift_plan)"""
    n_t = _pad(cout, 8)
    return _pad(2 * n_t if noisy else n_t, 16)


def _names(fn):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, [e.key for e in prof.key_averages()]


def _ran(names, mode, pool):
    want = "k_conv_shift<%d, 16, %s>" % (mode, "true" if pool else "false")
    assert any(want in n for n in names), (want, names)


def _mk(B, Cin, H, W, Cout, KH, KW, seed):
    gen = torch.Generator().manual_seed(seed)
    s_a = 5.0 / 15.0
    ka = torch.randint(0, 16, (B, Cin, H, W), generator=gen).float()
    cw = (torch.randint(0, 16, (Cout, Cin, KH, KW), generator=gen) * 2 - 15).float()
    wq = cw / 15.0
    w_raw = torch.randn(Cout, Cin, KH, KW, generator=gen) * 0.3
    z = torch.randn(B, Cout, H - KH + 1, W - KW + 1, generator=gen)
    return s_a, ka, cw, wq, w_raw, z


def _check_unpooled(dev, B, Cin, H, W, Cout, KH, KW, modes=(0, 1, 2)):
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_NONE, PACK_SHIFT, PREC_BF16, ConvGeom
    lib = _lib.load()
    g = ConvGeom(B, Cin, H, W, Cout, KH, KW, 1, 0)
    s_a, ka, cw, wq, w_raw, z = _mk(B, Cin, H, W, Cout, KH, KW, B * 1000 + Cout * 10 + KH * 3 + KW)
    x = (ka * s_a).to(dev)
    wqd, wrd, zd = wq.to(dev), w_raw.to(dev), z.to(dev)
    exact = F.conv2d(ka.double(), cw.double()) * (float(np.float32(s_a)) * float(np.float32(1.0 / 15.0)))
    kw = dict(precision="bf16", a_code_scale=s_a, w_code_scale=1.0 / 15.0)
    try:
        if 0 in modes:
            assert lib.nn_conv_pack_layout(C.byref(g), NOISE_NONE, PREC_BF16) == PACK_SHIFT
            lib.nn_debug_shift_enable(1)
            a, names = _names(lambda: ops.noisy_conv_fwd(x, wqd, None, None, 1, 0, noise_mode=NOISE_NONE, **kw)["y"])
            _ran(names, 0, False)
            assert ops.error_flag() == 0
            assert torch.allclose(a.cpu().double(), exact, rtol=1e-6, atol=1e-9)
            a2 = ops.noisy_conv_fwd(x, wqd, None, None, 1, 0, noise_mode=NOISE_NONE, **kw)["y"]
            assert torch.equal(a, a2)
            lib.nn_debug_shift_enable(0)
            b = ops.noisy_conv_fwd(x, wqd, None, None, 1, 0, noise_mode=NOISE_NONE, **kw)["y"]
            assert torch.equal(a, b)
        noisy = [m for m in modes if m]
        if noisy:
            lib.nn_debug_shift_enable(1)
            assert lib.nn_conv_pack_layout(C.byref(g), NOISE_EXTERNAL, PREC_BF16) == PACK_SHIFT
            scale = ops.tensor_stats(x)[0:1]
            common = dict(noise_mode=NOISE_EXTERNAL, current=1.0, scale_dev=scale, **kw)
            lib.nn_debug_shift_enable(0)
            ref = ops.noisy_conv_fwd(x, wqd, wrd, None, 1, 0, rng=ops._fixed_rng(7, 3), want_z=True, want_sigma=True, **common)
            tol = 1e-5 * float(ref["sigma"].abs().max()) * float(ref["z"].abs().max()) + 1e-6
            lib.nn_debug_shift_enable(1)
            for mode in noisy:
                extra = dict(rng=ops._fixed_rng(7, 3)) if mode == 1 else dict(z=ref["z"])
                a, names = _names(lambda: ops.noisy_conv_fwd(x, wqd, wrd, None, 1, 0, **extra, **common))
                _ran(names, mode, False)
                assert ops.error_flag() == 0
                assert torch.allclose(a["y"].cpu().double(), exact, rtol=1e-6, atol=1e-9)
                assert torch.equal(a["y"], ref["y"])
                assert (a["y_noisy"] - ref["y_noisy"]).abs().max().item() <= tol
                a2 = ops.noisy_conv_fwd(x, wqd, wrd, None, 1, 0, **extra, **common)
                assert torch.equal(a["y_noisy"], a2["y_noisy"]) and torch.equal(a["y"], a2["y"])
    finally:
        lib.nn_debug_shift_enable(1)


# every accumulator width the shift plan can produce: noisy 16 .. 256 (Cout 8 k: n_t = 8 k, 2 n_t = 16 k), plain 16 .. 128
# from the same channel counts, plain 144 .. 256 from wider layers (a ragged Cout where the width allows)
NOISY_COUTS = [8 * k - (k % 3) for k in range(1, 17)]
PLAIN_COUTS = [16 * k - (k % 5) for k in range(9, 17)]


def test_sweep_covers_every_width():
    widths_noisy = {n_mma(c, True) for c in NOISY_COUTS}
    widths_plain = {n_mma(c, False) for c in NOISY_COUTS + PLAIN_COUTS}
    every = set(range(16, 257, 16))
    assert widths_noisy == every and widths_plain == every


@pytest.mark.parametrize("cout", NOISY_COUTS)
def test_every_width_all_modes(dev, cout):
    # 3 x 3 taps: 5 pairs = chain blocks of 4 and 1, a padding tap; 2 x 14 x 14 positions = 4 tiles
    _check_unpooled(dev, 2, 3, 14, 14, cout, 3, 3)


@pytest.mark.parametrize("cout", PLAIN_COUTS)
def test_wide_plain_widths(dev, cout):
    _check_unpooled(dev, 2, 3, 14, 14, cout, 3, 3, modes=(0,))


# (KH, KW): tap pairs -> chain blocks of up to 4
TAPS = [
    (1, 1),      # 1 tap: one pair with a padding tap, one block of 1
    (2, 2),      # 4 taps: a block of 2
    (3, 2),      # 6 taps: a block of 3
    (2, 4),      # 8 taps: a block of 4
    (3, 3),      # 9 taps: 4 + 1, padding tap
    (4, 3),      # 12 taps: 4 + 2
    (7, 2),      # 14 taps: 4 + 3
    (5, 5),      # 25 taps (conv1): 4 + 4 + 4 + 1, padding tap
    (7, 7),      # 49 taps: 6 blocks of 4 + 1
]


@pytest.mark.parametrize("kh,kw", TAPS)
def test_tap_pair_blocks(dev, kh, kw):
    _check_unpooled(dev, 3, 2, 16, 18, 33, kh, kw)


def test_many_tiles_partial_last_round(dev):
    # 40 x 32 x 32 positions = 320 tiles: two full rounds of tiles over the SMs and a partly empty third
    _check_unpooled(dev, 40, 3, 32, 32, 65, 5, 5)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("B,Cout,k", [(40, 65, 5), (3, 4, 3), (5, 64, 5), (2, 33, 1)])
def test_pooled(dev, mode, B, Cout, k):
    """pooled_out / argmax_out == MaxPool2d(2,2) of the same mode's unfused output, and the BatchNorm statistics of the
    pooled values against float64."""
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_NONE, PREC_BF16, ConvFwdArgs, ConvGeom
    lib = _lib.load()
    H = 32
    OH = H - k + 1
    g = ConvGeom(B, 3, H, H, Cout, k, k, 1, 0)
    nm = NOISE_NONE if mode == 0 else NOISE_EXTERNAL
    assert lib.nn_conv_pool_fusable(C.byref(g), nm, PREC_BF16) == 1
    s_a, ka, cw, wq, w_raw, z = _mk(B, 3, H, H, Cout, k, k, 77 + B + Cout + k + mode)
    x, wqd, wrd, zd = (ka * s_a).to(dev), wq.to(dev), w_raw.to(dev), z.to(dev)
    scale = ops.tensor_stats(x)[0:1]
    kw = dict(precision="bf16", a_code_scale=s_a, w_code_scale=1.0 / 15.0, noise_mode=nm)
    if mode:
        kw.update(current=1.0, scale_dev=scale, want_y=False)
        kw.update(rng=ops._fixed_rng(5, 2)) if mode == 1 else kw.update(z=zd)
    ref = ops.noisy_conv_fwd(x, wqd, wrd if mode else None, None, 1, 0, **kw)
    full = ref["y_noisy"] if mode else ref["y"]
    if mode == 0:
        exact = F.conv2d(ka.double(), cw.double()) * (float(np.float32(s_a)) * float(np.float32(1.0 / 15.0)))
        assert torch.allclose(full.cpu().double(), exact, rtol=1e-6, atol=1e-9)
    pv, pi = F.max_pool2d(full, 2, 2, return_indices=True)
    ih, iw = pi // OH, pi % OH
    pos = ((ih % 2) * 2 + (iw % 2)).to(torch.uint8)
    a = ConvFwdArgs()
    a.g = g
    a.x, a.w_eff, a.w_raw = x.data_ptr(), wqd.data_ptr(), wrd.data_ptr() if mode else None
    pooled = torch.empty(B, Cout, OH // 2, OH // 2, device=dev)
    arg = torch.empty(B, Cout, OH // 2, OH // 2, dtype=torch.uint8, device=dev)
    a.pooled_out, a.argmax_out, a.noise_mode = pooled.data_ptr(), arg.data_ptr(), nm
    if mode:
        a.current, a.scale_dev = 1.0, scale.data_ptr()
        if mode == 1:
            a.rng = ops._fixed_rng(5, 2)
        else:
            a.z_inject = zd.data_ptr()
    a.precision, a.a_code_scale, a.w_code_scale = PREC_BF16, s_a, 1.0 / 15.0
    ws = torch.empty(int(lib.nn_conv_workspace_bytes(C.byref(g), PREC_BF16)) + 4096, dtype=torch.uint8, device=dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    mean, invstd = torch.empty(Cout, device=dev), torch.empty(Cout, device=dev)
    rm, rv = torch.zeros(Cout, device=dev), torch.ones(Cout, device=dev)
    scratch = torch.zeros(int(lib.nn_conv_bn_scratch_bytes(Cout)), dtype=torch.uint8, device=dev)
    a.bn_mean, a.bn_invstd, a.bn_running_mean, a.bn_running_var = mean.data_ptr(), invstd.data_ptr(), rm.data_ptr(), rv.data_ptr()
    a.bn_eps, a.bn_momentum, a.bn_eval_mode, a.bn_scratch = 1e-5, 0.1, 0, scratch.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    _, names = _names(lambda: _lib.check(lib.nn_noisy_conv_fwd(C.byref(a), 0, st), "nn_noisy_conv_fwd"))
    _ran(names, mode, True)
    assert ops.error_flag() == 0
    assert torch.equal(pooled, pv)
    assert torch.equal(arg, pos)
    m_ref = pv.double().mean(dim=(0, 2, 3))
    v_ref = pv.double().var(dim=(0, 2, 3), unbiased=False)
    assert torch.allclose(mean.double(), m_ref, rtol=1e-5, atol=1e-6)
    assert torch.allclose(invstd.double(), 1.0 / torch.sqrt(v_ref + 1e-5), rtol=1e-5)
    first = (pooled.clone(), arg.clone(), mean.clone(), invstd.clone())
    _lib.check(lib.nn_noisy_conv_fwd(C.byref(a), 0, st), "nn_noisy_conv_fwd")
    torch.cuda.synchronize()
    for u, v in zip(first, (pooled, arg, mean, invstd)):
        assert torch.equal(u, v)
