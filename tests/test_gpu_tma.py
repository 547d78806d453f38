"""The persistent CTA-pair kernel with TMA-im2col operands (csrc/nn_conv_tma.cu) against float64 evaluations of the same
operands, the fp32 CUDA-core kernels and the gathered-im2col tensor-core kernel it replaces on the lean path.

Stated tolerances (as in test_gpu_umma.py):
  * integer-code mode: the tensor-core sum is exact -> rtol 1e-6 against float64;
  * noisy output: same Philox stream and (m, n) mapping as every other kernel of the library; sigma from bf16-rounded
    g(|w_raw|) -> y_noisy within atol 3e-3 * max|noise| + 1e-5 of the fp32 kernel's with the same seeds;
  * plain operands / dgrad: both operands rounded to bf16 -> |err| <= 1.5e-2 * max|ref|.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__ as entry
    entry.build()
    return torch.device("cuda:0")


def _codes(shape, gen, s_a, zero_frac=0.3):
    k = torch.randint(0, 16, shape, generator=gen).float()
    k = k * (torch.rand(shape, generator=gen) > zero_frac).float()
    return k, (k * s_a).float()


def _wcodes(shape, gen):
    c = (torch.randint(0, 16, shape, generator=gen) * 2 - 15).float()
    return c, (c * (2.0 / 15.0) / 2.0).float()


SHAPES = [  # B, Cin, H, W, Cout, k, stride, pad
    (5, 65, 14, 14, 120, 5, 1, 0),      # NoisyNet conv2: 64 + 16-channel tail (SWIZZLE_32B), ragged last tile, odd tile count
    (3, 64, 12, 12, 64, 3, 1, 1),       # ResNet 3x3: one 64-channel chunk per tap, padding taps
    (2, 64, 16, 16, 128, 3, 2, 1),      # ResNet 3x3 stride 2
    (2, 128, 9, 9, 96, 3, 1, 1),        # two 64-channel chunks per stage
    (2, 256, 8, 8, 72, 3, 1, 1),        # four chunks per tap = two stages per tap
    (2, 16, 15, 15, 24, 3, 1, 1),       # tail chunk only (16 channels)
    (2, 40, 10, 10, 56, 3, 1, 0),       # tail chunk only, zero-padded to 64 channels
    (2, 96, 10, 10, 136, 1, 2, 0),      # 1x1 stride 2 downsample, 64 + 32-channel tail (SWIZZLE_64B), two n-tiles when noisy
    (1, 24, 33, 33, 16, 7, 2, 3),       # 7x7 stride 2 pad 3
]


def _layout(dev, shape, noise_mode):
    from noisynet_b200 import _lib
    B, Cin, H, W, Cout, k, s, p = shape
    g = _lib.ConvGeom(B, Cin, H, W, Cout, k, k, s, p)
    return _lib.load().nn_conv_pack_layout(C.byref(g), noise_mode, _lib.PREC_BF16)


@pytest.mark.parametrize("shape", SHAPES)
def test_tma_forward_code_mode(dev, shape):
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_MERGED, PACK_TMA
    B, Cin, H, W, Cout, k, s, p = shape
    assert _layout(dev, shape, NOISE_EXTERNAL) == PACK_TMA
    gen = torch.Generator().manual_seed(hash(shape) % 1000)
    s_a = 5.0 / 15.0
    ka, x = _codes((B, Cin, H, W), gen, s_a)
    cw, wq = _wcodes((Cout, Cin, k, k), gen)
    w_raw = torch.randn(Cout, Cin, k, k, generator=gen) * 0.3
    xd, wqd, wrd = x.to(dev), wq.to(dev), w_raw.to(dev)
    exact = F.conv2d(ka.double(), cw.double(), None, s, p) * (float(np.float32(s_a)) * float(np.float32(1.0 / 15.0)))
    # plain launch (no noise): exact
    y = ops.noisy_conv_fwd(xd, wqd, None, None, s, p, precision="bf16", a_code_scale=s_a, w_code_scale=1.0 / 15.0)["y"]
    assert ops.error_flag() == 0
    assert torch.allclose(y.cpu().double(), exact, rtol=1e-6, atol=1e-9), (y.cpu().double() - exact).abs().max()
    lib = _lib.load()
    for mode in (NOISE_MERGED, NOISE_EXTERNAL):
        scale = ops.tensor_stats(wrd)[1:2] if mode == NOISE_MERGED else ops.tensor_stats(xd)[0:1]
        kw = dict(noise_mode=mode, current=1.0, scale_dev=scale, a_code_scale=s_a, w_code_scale=1.0 / 15.0, want_y=False)
        r = ops.noisy_conv_fwd(xd, wqd, wrd, None, s, p, precision="bf16", rng=ops._fixed_rng(11, 5), **kw)      # TMA kernel
        assert ops.error_flag() == 0
        prev = lib.nn_debug_tma_enable(0)
        try:
            r_old = ops.noisy_conv_fwd(xd, wqd, wrd, None, s, p, precision="bf16", rng=ops._fixed_rng(11, 5), **kw)   # gathered im2col
        finally:
            lib.nn_debug_tma_enable(prev)
        r32 = ops.noisy_conv_fwd(xd, wqd, wrd, None, s, p, precision="fp32", rng=ops._fixed_rng(11, 5), want_z=True,
                                 want_sigma=True, noise_mode=mode, current=1.0, scale_dev=scale)
        noise_max = (r32["z"] * r32["sigma"]).abs().max().item()
        # same operands (bf16 g(|w|), integer codes), different K order of the fp32 accumulation of sigma^2 only
        assert (r["y_noisy"] - r_old["y_noisy"]).abs().max().item() <= 1e-4 * noise_max + 1e-5
        assert (r["y_noisy"] - r32["y_noisy"]).abs().max().item() <= 3e-3 * noise_max + 1e-5
        # injected draws (the parity hook the engine tests use): same kernel family, z read from memory
        rz = ops.noisy_conv_fwd(xd, wqd, wrd, None, s, p, precision="bf16", z=r32["z"], **kw)
        assert (rz["y_noisy"] - r32["y_noisy"]).abs().max().item() <= 3e-3 * noise_max + 1e-5
        assert ops.error_flag() == 0


@pytest.mark.parametrize("shape", SHAPES)
def test_tma_plain_and_dgrad(dev, shape):
    from noisynet_b200 import ops
    B, Cin, H, W, Cout, k, s, p = shape
    gen = torch.Generator().manual_seed(5 + hash(shape) % 1000)
    x = torch.randn(B, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5
    y = F.conv2d(x, w, None, s, p)
    r = ops.noisy_conv_fwd(x.to(dev), w.to(dev), None, None, s, p, precision="bf16")
    assert ops.error_flag() == 0
    assert (r["y"].cpu() - y).abs().max().item() <= 1.5e-2 * y.abs().max().item()
    if s == 1:
        gy = torch.randn(y.shape, generator=gen)
        ref = torch.nn.grad.conv2d_input(x.shape, w, gy, s, p)
        gx = ops.conv_dgrad(gy.to(dev), w.to(dev), x.shape, s, p, precision="bf16").cpu()
        assert ops.error_flag() == 0
        assert (gx - ref).abs().max().item() <= 1.5e-2 * ref.abs().max().item() + 1e-6
        # integer weight codes: exact weight operand
        cw, wq = _wcodes((Cout, Cin, k, k), gen)
        gyb = gy.bfloat16().float()
        ref2 = torch.nn.grad.conv2d_input(x.shape, cw.double(), gyb.double(), s, p) * float(np.float32(1.0 / 15.0))
        gx2 = ops.conv_dgrad(gyb.to(dev), wq.to(dev), x.shape, s, p, precision="bf16", w_code_scale=1.0 / 15.0).cpu()
        assert torch.allclose(gx2.double(), ref2, rtol=2e-5, atol=1e-5 * ref2.abs().max().item())


def test_tma_full_size_conv2(dev):
    """BASELINE config 2 size (batch 512): exactness on a slice, per-sample independence, sign linearity, and the noisy
    launch against the gathered-im2col kernel with the same seeds."""
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import NOISE_EXTERNAL
    B = 512
    gen = torch.Generator().manual_seed(9)
    s_a = 5.0 / 15.0
    ka, x = _codes((B, 65, 14, 14), gen, s_a)
    cw, wq = _wcodes((120, 65, 5, 5), gen)
    w_raw = torch.randn(120, 65, 5, 5, generator=gen) * 0.1
    xd, wqd, wrd = x.to(dev), wq.to(dev), w_raw.to(dev)
    y = ops.noisy_conv_fwd(xd, wqd, precision="bf16", a_code_scale=s_a, w_code_scale=1 / 15.0)["y"]
    assert ops.error_flag() == 0
    for sl in (slice(0, 2), slice(255, 258), slice(510, 512)):
        exact = F.conv2d(ka[sl].double(), cw.double()) * (float(np.float32(s_a)) * float(np.float32(1 / 15.0)))
        assert torch.allclose(y[sl].cpu().double(), exact, rtol=1e-6, atol=1e-9)
    ys = ops.noisy_conv_fwd(xd[200:203].contiguous(), wqd, precision="bf16", a_code_scale=s_a, w_code_scale=1 / 15.0)["y"]
    assert torch.equal(ys, y[200:203])
    y2 = ops.noisy_conv_fwd(xd, -wqd, precision="bf16", a_code_scale=s_a, w_code_scale=1 / 15.0)["y"]
    assert torch.equal(y2, -y)
    scale = ops.tensor_stats(xd)[0:1]
    kw = dict(noise_mode=NOISE_EXTERNAL, current=1.0, scale_dev=scale, a_code_scale=s_a, w_code_scale=1 / 15.0, want_y=False)
    r = ops.noisy_conv_fwd(xd, wqd, wrd, None, 1, 0, precision="bf16", rng=ops._fixed_rng(3, 1), **kw)
    lib = _lib.load()
    prev = lib.nn_debug_tma_enable(0)
    try:
        r_old = ops.noisy_conv_fwd(xd, wqd, wrd, None, 1, 0, precision="bf16", rng=ops._fixed_rng(3, 1), **kw)
    finally:
        lib.nn_debug_tma_enable(prev)
    assert ops.error_flag() == 0
    d = (r["y_noisy"] - r_old["y_noisy"]).abs().max().item()
    assert d <= 1e-4 * (r_old["y_noisy"] - y).abs().max().item() + 1e-5, d
    # dgrad at full size: exact weight codes, bf16 gradients
    gy = torch.randn(B, 120, 10, 10, generator=gen).bfloat16().float()
    gx = ops.conv_dgrad(gy.to(dev), wqd, x.shape, 1, 0, precision="bf16", w_code_scale=1 / 15.0)
    assert ops.error_flag() == 0
    sl = slice(300, 302)
    ref = torch.nn.grad.conv2d_input((2, 65, 14, 14), cw.double(), gy[sl].double(), 1, 0) * float(np.float32(1 / 15.0))
    assert torch.allclose(gx[sl].cpu().double(), ref, rtol=2e-5, atol=1e-5 * ref.abs().max().item())
