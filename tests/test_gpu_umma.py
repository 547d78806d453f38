"""Tensor-core (NN_PREC_BF16) kernels against the fp32 CUDA-core kernels / the CPU oracle.

Stated tolerances:
  * integer-code mode (4-bit activation codes x odd-integer weight codes): the tensor-core sum is EXACT
    (integers in bf16, fp32 accumulate, |sum| < 2^24); the only rounding is the final scale multiply
    -> rtol 1e-6 against a float64 evaluation of the same quantised operands.
  * sigma^2 contraction: g(|w_raw|) is rounded to bf16 (2^-9 per weight, all terms positive)
    -> sigma within rtol 3e-3 of the fp32 value.
  * plain (non-code) operands and dgrad: both operands rounded to bf16 -> |err| <= 1.5e-2 * max|ref|.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import noisynet_oracle as O

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
    return c, (c * (2.0 / 15.0) / 2.0).float()          # c/15 computed as the quantizer does: k*scale + min


SHAPES = [  # B, Cin, H, W, Cout, k, stride, pad
    (4, 3, 32, 32, 65, 5, 1, 0),        # NoisyNet conv1
    (5, 65, 14, 14, 120, 5, 1, 0),      # NoisyNet conv2 (M = 500: ragged last tile)
    (9, 3000, 1, 1, 390, 1, 1, 0),      # NoisyNet fc1 (4 n-tiles)
    (33, 390, 1, 1, 10, 1, 1, 0),       # NoisyNet fc2
    (2, 16, 15, 15, 24, 3, 1, 1),       # padded 3x3
    (2, 16, 14, 14, 32, 1, 2, 0),       # 1x1 stride 2 (ResNet downsample)
    (1, 3, 33, 33, 16, 7, 2, 3),        # 7x7 stride 2 pad 3 (ResNet stem)
    (1, 1, 5, 5, 1, 5, 1, 0),           # degenerate
]


@pytest.mark.parametrize("shape", SHAPES)
def test_code_mode_exact_and_noise(dev, shape):
    from noisynet_b200 import ops
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_MERGED
    B, Cin, H, W, Cout, k, s, p = shape
    gen = torch.Generator().manual_seed(hash(shape) % 1000)
    s_a = 5.0 / 15.0
    ka, x = _codes((B, Cin, H, W), gen, s_a)
    cw, wq = _wcodes((Cout, Cin, k, k), gen)
    w_raw = torch.randn(Cout, Cin, k, k, generator=gen) * 0.3
    xd, wqd, wrd = x.to(dev), wq.to(dev), w_raw.to(dev)
    exact = (F.conv2d(ka.double(), cw.double(), None, s, p) * (float(np.float32(s_a)) * float(np.float32(1.0 / 15.0))))
    for mode in (NOISE_MERGED, NOISE_EXTERNAL):
        scale = ops.tensor_stats(wrd)[1:2] if mode == NOISE_MERGED else ops.tensor_stats(xd)[0:1]
        stats = torch.tensor([0.0, 0.0, float("-inf")], device=dev)
        r = ops.noisy_conv_fwd(xd, wqd, wrd, None, s, p, noise_mode=mode, current=1.0, scale_dev=scale,
                               want_z=True, want_sigma=True, stats=stats, precision="bf16",
                               a_code_scale=s_a, w_code_scale=1.0 / 15.0, rng=ops._fixed_rng(7, 3))
        assert ops.error_flag() == 0
        y = r["y"].cpu().double()
        assert torch.allclose(y, exact, rtol=1e-6, atol=1e-9), (y - exact).abs().max()
        # fp32 reference of the same launch
        stats0 = torch.tensor([0.0, 0.0, float("-inf")], device=dev)
        r0 = ops.noisy_conv_fwd(xd, wqd, wrd, None, s, p, noise_mode=mode, current=1.0, scale_dev=scale,
                                want_z=True, want_sigma=True, stats=stats0, precision="fp32", rng=ops._fixed_rng(7, 3))
        assert torch.allclose(r["sigma"], r0["sigma"], rtol=3e-3, atol=1e-6)
        assert torch.equal(r["z"], r0["z"])                       # same Philox stream, same (m, n) mapping
        assert torch.allclose(r["y_noisy"], r["y"] + r["z"] * r["sigma"], rtol=0, atol=1e-5)
        a, b = stats.tolist(), stats0.tolist()
        assert a[0] == pytest.approx(b[0], rel=3e-3) and a[1] == pytest.approx(b[1], rel=5e-3)
        assert a[2] == pytest.approx(b[2], rel=1e-5, abs=1e-6)
        # noise-only launch (two-call flow): clean output is an input
        r2 = ops.noisy_conv_fwd(xd, None, wrd, None, s, p, noise_mode=mode, current=1.0, scale_dev=scale,
                                z=r["z"], precision="bf16", a_code_scale=s_a, y_in=r["y"])
        assert torch.allclose(r2["y_noisy"], r["y_noisy"], rtol=0, atol=1e-6)
        assert ops.error_flag() == 0


@pytest.mark.parametrize("shape", SHAPES)
def test_plain_operands_and_dgrad(dev, shape):
    from noisynet_b200 import ops
    B, Cin, H, W, Cout, k, s, p = shape
    gen = torch.Generator().manual_seed(5 + hash(shape) % 1000)
    x = torch.randn(B, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=gen)
    y = F.conv2d(x, w, b, s, p)
    r = ops.noisy_conv_fwd(x.to(dev), w.to(dev), None, b.to(dev), s, p, precision="bf16")
    assert ops.error_flag() == 0
    assert (r["y"].cpu() - y).abs().max().item() <= 1.5e-2 * y.abs().max().item()
    gy = torch.randn(y.shape, generator=gen)
    ref = torch.nn.grad.conv2d_input(x.shape, w, gy, s, p)
    gx = ops.conv_dgrad(gy.to(dev), w.to(dev), x.shape, s, p, precision="bf16").cpu()   # stride 2 -> fp32 kernels
    assert ops.error_flag() == 0
    assert (gx - ref).abs().max().item() <= 1.5e-2 * ref.abs().max().item() + 1e-6
    # STE mask fused into the dgrad store
    gxm = ops.conv_dgrad(gy.to(dev), w.to(dev), x.shape, s, p, x_pre=x.to(dev), x_lo=-0.5, x_hi=0.5,
                         precision="bf16").cpu()
    keep = ((x >= -0.5) & (x <= 0.5)).float()
    # (the unmasked call may run on the TMA-im2col kernel, the masked one on the gathered-im2col kernel: same bf16 operands,
    #  different order of the fp32 accumulation)
    assert torch.allclose(gxm, gx * keep, rtol=1e-4, atol=1e-5 * ref.abs().max().item())
    assert (gxm[keep == 0] == 0).all()


def test_full_size_conv2_properties(dev):
    """Batch 512 (BASELINE config 2): per-sample independence, linearity in the weights and exactness of
    integer codes at full size (float64 reference on a slice)."""
    from noisynet_b200 import ops
    B = 512
    gen = torch.Generator().manual_seed(9)
    s_a = 5.0 / 15.0
    ka, x = _codes((B, 65, 14, 14), gen, s_a)
    cw, wq = _wcodes((120, 65, 5, 5), gen)
    xd, wqd = x.to(dev), wq.to(dev)
    y = ops.noisy_conv_fwd(xd, wqd, precision="bf16", a_code_scale=s_a, w_code_scale=1 / 15.0)["y"]
    assert ops.error_flag() == 0
    sl = slice(200, 203)
    exact = F.conv2d(ka[sl].double(), cw.double()) * (float(np.float32(s_a)) * float(np.float32(1 / 15.0)))
    assert torch.allclose(y[sl].cpu().double(), exact, rtol=1e-6, atol=1e-9)
    ys = ops.noisy_conv_fwd(xd[sl].contiguous(), wqd, precision="bf16", a_code_scale=s_a, w_code_scale=1 / 15.0)["y"]
    assert torch.equal(ys, y[sl])
    y2 = ops.noisy_conv_fwd(xd, -wqd, precision="bf16", a_code_scale=s_a, w_code_scale=1 / 15.0)["y"]
    assert torch.equal(y2, -y)


def test_linear_bn_statistics_from_splitk_epilogue(dev):
    """bn_mean on a fully connected layer (nn_conv_linear_bn_fusable): the split-K epilogue adds the per-channel sums of its
    output, the last slice finalizes -- mean / invstd / running statistics against torch on the output the same launch
    wrote, twice in a row (self-resetting counters), and the zero_out side effect."""
    import ctypes as C
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import NOISE_MERGED, PREC_BF16, ConvFwdArgs, ConvGeom
    lib = _lib.load()
    B, K, N = 512, 3000, 390
    g = ConvGeom(B, K, 1, 1, N, 1, 1, 1, 0)
    assert lib.nn_conv_linear_bn_fusable(C.byref(g), NOISE_MERGED, PREC_BF16, 0) == 1
    assert lib.nn_conv_linear_bn_fusable(C.byref(ConvGeom(500, K, 1, 1, N, 1, 1, 1, 0)), NOISE_MERGED, PREC_BF16, 0) == 0
    gen = torch.Generator().manual_seed(3)
    s_a = 5.0 / 15.0
    ka, x = _codes((B, K, 1, 1), gen, s_a)
    cw, wq = _wcodes((N, K, 1, 1), gen)
    w_raw = torch.randn(N, K, 1, 1, generator=gen) * 0.05
    xd, wqd, wrd = x.to(dev), wq.to(dev), w_raw.to(dev)
    scale = ops.tensor_stats(wrd)[1:2]
    y = torch.empty(B, N, 1, 1, device=dev)
    mean, invstd = torch.empty(N, device=dev), torch.empty(N, device=dev)
    rm, rv = torch.zeros(N, device=dev), torch.ones(N, device=dev)
    scratch = torch.zeros(int(lib.nn_stage_scratch_bytes(N)) + 64, dtype=torch.uint8, device=dev)
    zero = torch.full((1,), 3.0, device=dev)
    ws = torch.empty(int(lib.nn_conv_workspace_bytes(C.byref(g), PREC_BF16)) + 4096, dtype=torch.uint8, device=dev)
    a = ConvFwdArgs()
    a.g = g
    a.x, a.w_eff, a.w_raw, a.y_noisy = xd.data_ptr(), wqd.data_ptr(), wrd.data_ptr(), y.data_ptr()
    a.noise_mode, a.current, a.scale_dev, a.rng = NOISE_MERGED, 1.0, scale.data_ptr(), ops._fixed_rng(4, 4)
    a.precision, a.a_code_scale, a.w_code_scale = PREC_BF16, s_a, 1.0 / 15.0
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    a.bn_mean, a.bn_invstd, a.bn_running_mean, a.bn_running_var = mean.data_ptr(), invstd.data_ptr(), rm.data_ptr(), rv.data_ptr()
    a.bn_eps, a.bn_momentum, a.bn_eval_mode, a.bn_scratch, a.zero_out = 1e-5, 0.1, 0, scratch.data_ptr(), zero.data_ptr()
    for rep in range(2):
        zero.fill_(3.0)
        _lib.check(lib.nn_noisy_conv_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream), "nn_noisy_conv_fwd")
        assert ops.error_flag() == 0
        yy = y.view(B, N).double()
        m_ref, v_ref = yy.mean(0), yy.var(0, unbiased=False)
        assert torch.allclose(mean.double(), m_ref, rtol=1e-5, atol=1e-6)
        assert torch.allclose(invstd.double(), 1.0 / torch.sqrt(v_ref + 1e-5), rtol=1e-5)
        assert zero.item() == 0.0
    assert torch.allclose(rm.double(), (0.9 * 0.1 + 0.1) * m_ref, rtol=1e-4, atol=1e-6)       # two updates from 0 with the same batch
    # the same call without bn_mean writes the same output (same Philox stream)
    y2 = torch.empty_like(y)
    a.y_noisy, a.bn_mean = y2.data_ptr(), None
    _lib.check(lib.nn_noisy_conv_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream), "nn_noisy_conv_fwd")
    assert torch.equal(y, y2)
