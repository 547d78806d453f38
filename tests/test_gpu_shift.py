"""The persistent shift-GEMM forward (k_conv_shift: narrow-input layers, weights resident in shared memory, the
im2col rows read through shifted SWIZZLE_NONE descriptors) against the tiled tensor-core kernel, the fp32 CUDA-core
kernel and a float64 evaluation.

Stated tolerances (same as test_gpu_umma.py): integer-code main contraction exact up to the final scale multiply
(rtol 1e-6); sigma within rtol 3e-3 of fp32; the Philox draws are the same stream with the same (m, n) -> group
mapping as every other path, so with equal sigma the noisy outputs agree to the sigma tolerance.
"""
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


SHAPES = [  # B, Cin, H, W, Cout, k
    (4, 3, 32, 32, 65, 5),        # NoisyNet conv1 (25 taps: odd -> one padding tap)
    (3, 3, 32, 32, 9, 5),         # the narrow golden net
    (2, 1, 28, 28, 16, 4),        # MNIST-like, even tap count, 784 pixels/image: tiles straddle images
    (5, 8, 9, 11, 120, 3),        # Cin = 8 exactly, W not a divisor of 128, widest accumulator (2 x 120 -> 240 cols)
    (1, 3, 5, 5, 4, 5),           # single output pixel, fewer pixels than one tile
    (300, 2, 12, 12, 33, 3),      # more tiles than SMs: several tiles per CTA, both accumulator buffers reused
]


def _mk(shape, gen):
    B, Cin, H, W, Cout, k = shape
    s_a = 5.0 / 15.0
    ka = torch.randint(0, 16, (B, Cin, H, W), generator=gen).float()
    ka = ka * (torch.rand(ka.shape, generator=gen) > 0.3).float()
    cw = (torch.randint(0, 16, (Cout, Cin, k, k), generator=gen) * 2 - 15).float()
    wq = (cw * (2.0 / 15.0) / 2.0).float()
    w_raw = torch.randn(Cout, Cin, k, k, generator=gen) * 0.3
    return s_a, ka, (ka * s_a).float(), cw, wq, w_raw


@pytest.mark.parametrize("shape", SHAPES)
def test_shift_matches_tiled_and_exact(dev, shape):
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_MERGED, NOISE_NONE, PACK_SHIFT, PREC_BF16, ConvGeom
    import ctypes as C
    lib = _lib.load()
    B, Cin, H, W, Cout, k = shape
    g = ConvGeom(B, Cin, H, W, Cout, k, k, 1, 0)
    assert lib.nn_conv_pack_layout(C.byref(g), NOISE_MERGED, PREC_BF16) == PACK_SHIFT
    gen = torch.Generator().manual_seed(sum(shape))
    s_a, ka, x, cw, wq, w_raw = _mk(shape, gen)
    xd, wqd, wrd = x.to(dev), wq.to(dev), w_raw.to(dev)
    exact = F.conv2d(ka.double(), cw.double()) * (float(np.float32(s_a)) * float(np.float32(1.0 / 15.0)))
    kw = dict(precision="bf16", a_code_scale=s_a, w_code_scale=1.0 / 15.0)
    try:
        # plain (no noise)
        r = ops.noisy_conv_fwd(xd, wqd, None, None, 1, 0, noise_mode=NOISE_NONE, **kw)
        assert ops.error_flag() == 0
        assert torch.allclose(r["y"].cpu().double(), exact, rtol=1e-6, atol=1e-9)
        for mode in (NOISE_MERGED, NOISE_EXTERNAL):
            scale = ops.tensor_stats(wrd)[1:2] if mode == NOISE_MERGED else ops.tensor_stats(xd)[0:1]
            common = dict(noise_mode=mode, current=1.0, scale_dev=scale)
            lib.nn_debug_shift_enable(1)
            a = ops.noisy_conv_fwd(xd, wqd, wrd, None, 1, 0, rng=ops._fixed_rng(11, 5), **common, **kw)
            assert ops.error_flag() == 0
            lib.nn_debug_shift_enable(0)
            b = ops.noisy_conv_fwd(xd, wqd, wrd, None, 1, 0, rng=ops._fixed_rng(11, 5), want_z=True, want_sigma=True,
                                   **common, **kw)
            assert ops.error_flag() == 0
            assert torch.allclose(a["y"].cpu().double(), exact, rtol=1e-6, atol=1e-9)
            assert torch.equal(a["y"], b["y"])
            # same z; sigma from the same bf16 operands, only the fp32 summation order may differ
            tol = 1e-5 * float(b["sigma"].abs().max()) * float(b["z"].abs().max()) + 1e-6
            assert (a["y_noisy"] - b["y_noisy"]).abs().max().item() <= tol
            # injected z (parity hook variant of the kernel)
            lib.nn_debug_shift_enable(1)
            c = ops.noisy_conv_fwd(xd, wqd, wrd, None, 1, 0, z=b["z"], **common, **kw)
            assert ops.error_flag() == 0
            assert (c["y_noisy"] - a["y_noisy"]).abs().max().item() <= tol
            # fp32 CUDA-core kernel: sigma tolerance
            f = ops.noisy_conv_fwd(xd, wqd, wrd, None, 1, 0, z=b["z"], want_sigma=True, precision="fp32", **common)
            assert torch.allclose(b["sigma"], f["sigma"], rtol=3e-3, atol=1e-6)
            lim = 3e-3 * (f["sigma"] * b["z"].abs()) + 2e-5 * f["y"].abs().max()
            assert ((a["y_noisy"] - f["y_noisy"]).abs() <= lim).all()
    finally:
        lib.nn_debug_shift_enable(1)


def test_shift_layout_rejected_when_not_served(dev):
    from noisynet_b200 import _lib
    from noisynet_b200._lib import NOISE_MERGED, PACK_SHIFT, PACK_TILED, PREC_BF16, ConvGeom
    import ctypes as C
    lib = _lib.load()
    for g in (ConvGeom(4, 65, 14, 14, 120, 5, 5, 1, 0), ConvGeom(4, 3, 32, 32, 65, 5, 5, 1, 2),
              ConvGeom(4, 3, 32, 32, 65, 5, 5, 2, 0), ConvGeom(4, 3, 32, 32, 200, 5, 5, 1, 0)):
        assert lib.nn_conv_pack_layout(C.byref(g), NOISE_MERGED, PREC_BF16) != PACK_SHIFT
    # wider inputs go to the TMA-im2col kernel, narrow ones that the shift kernel cannot serve to the tiled one
    assert lib.nn_conv_pack_layout(C.byref(ConvGeom(4, 65, 14, 14, 120, 5, 5, 1, 0)), NOISE_MERGED, PREC_BF16) == _lib.PACK_TMA
    assert lib.nn_conv_pack_layout(C.byref(ConvGeom(4, 3, 32, 32, 65, 5, 5, 2, 0)), NOISE_MERGED, PREC_BF16) == PACK_TILED
    g = ConvGeom(4, 3, 32, 32, 200, 5, 5, 1, 0)
    assert lib.nn_conv_pack_layout(C.byref(g), 0, PREC_BF16) == PACK_SHIFT      # 200 plain columns fit, 400 do not


WG_SHAPES = [  # B, Cin, H, W, Cout, k
    (4, 3, 32, 32, 65, 5),        # NoisyNet conv1
    (3, 1, 28, 28, 16, 4),        # even kernel, 784 pixels per image (chunks straddle images)
    (5, 8, 9, 11, 120, 3),        # 495 pixels: the last reduction chunk is padding; 15 channel planes
    (2, 3, 12, 12, 7, 1),         # 1x1
    (40, 2, 16, 16, 33, 7),       # 7x7 (KH * 64 = 448 accumulator columns), more chunks than one per CTA
]


@pytest.mark.parametrize("shape", WG_SHAPES)
def test_shift_wgrad_matches_tiled_and_fp64(dev, shape):
    """Weight gradient through the in-place (shift) kernel: integer activation codes x bf16 grad_output, fp32
    accumulation.  Against float64 on the SAME bf16-rounded grad_output the only error is the fp32 summation
    (rtol 2e-5 of the largest entry); against the tiled tensor-core kernel (same operands, different summation order)
    likewise."""
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import PACK_SHIFT, PREC_BF16, ConvGeom
    import ctypes as C
    lib = _lib.load()
    B, Cin, H, W, Cout, k = shape
    g = ConvGeom(B, Cin, H, W, Cout, k, k, 1, 0)
    assert lib.nn_conv_wgrad_pack_layout(C.byref(g), PREC_BF16, 0) == PACK_SHIFT
    gen = torch.Generator().manual_seed(sum(shape) + 1)
    s_a = 5.0 / 15.0
    ka = torch.randint(0, 16, (B, Cin, H, W), generator=gen).float()
    x = (ka * s_a).float()
    OH, OW = H - k + 1, W - k + 1
    gy = torch.randn(B, Cout, OH, OW, generator=gen) * 0.01
    w_raw = torch.randn(Cout, Cin, k, k, generator=gen) * 0.6          # some |w| > 1: STE mask zeros those entries
    gyb = gy.bfloat16().double()
    ref = torch.nn.grad.conv2d_weight(ka.double(), (Cout, Cin, k, k), gyb) * float(np.float32(s_a))
    ref = ref * ((w_raw >= -1) & (w_raw <= 1)).double()
    xd, gyd, wrd = x.to(dev), gy.to(dev), w_raw.to(dev)
    try:
        lib.nn_debug_shift_enable(1)
        a = ops.conv_wgrad(gyd, xd, w_raw.shape, 1, 0, w_raw=wrd, w_lo=-1.0, w_hi=1.0, precision="bf16", a_code_scale=s_a)
        assert ops.error_flag() == 0
        lib.nn_debug_shift_enable(0)
        b = ops.conv_wgrad(gyd, xd, w_raw.shape, 1, 0, w_raw=wrd, w_lo=-1.0, w_hi=1.0, precision="bf16", a_code_scale=s_a)
        assert ops.error_flag() == 0
    finally:
        lib.nn_debug_shift_enable(1)
    tol = 2e-5 * float(ref.abs().max())
    assert (a.cpu().double() - ref).abs().max().item() <= tol
    assert (a - b).abs().max().item() <= tol


def test_stage_bwd_planes_layout(dev):
    """nn_stage_bwd with gy_layout = NN_PACK_SHIFT writes the same values as the NHWC pack, at the planes-layout
    addresses of the (larger) virtual grid, and nothing else."""
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import PACK_SHIFT, StageArgs, StageBwdArgs
    import ctypes as C
    lib = _lib.load()
    B, Cc, H, W, vH, vW = 3, 13, 8, 8, 12, 12
    gen = torch.Generator().manual_seed(5)
    x_in = torch.randn(B, Cc, H, W, generator=gen).to(dev)
    gamma, beta = (torch.rand(Cc, generator=gen) + 0.5).to(dev), (torch.randn(Cc, generator=gen) * 0.1).to(dev)
    PH, PW = H // 2, W // 2
    f32 = lambda *s: torch.empty(*s, device=dev)
    pooled, amax = f32(B, Cc, PH, PW), torch.empty(B, Cc, PH, PW, dtype=torch.uint8, device=dev)
    mean, invstd, xmax = f32(Cc), f32(Cc), f32(1)
    Cp = 16
    xp = torch.empty(B, PH, PW, Cp, dtype=torch.bfloat16, device=dev)
    scratch = torch.zeros(int(lib.nn_stage_scratch_bytes(Cc)) + 64, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    a = StageArgs()
    a.in_, a.B, a.C, a.H, a.W, a.pool = x_in.data_ptr(), B, Cc, H, W, 1
    a.pooled, a.argmax, a.gamma, a.beta = pooled.data_ptr(), amax.data_ptr(), gamma.data_ptr(), beta.data_ptr()
    a.running_mean, a.running_var, a.momentum, a.eps = None, None, 0.1, 1e-5
    a.mean, a.invstd, a.act_max, a.q_bits, a.q_hi, a.stochastic = mean.data_ptr(), invstd.data_ptr(), 5.0, 4, 5.0, 0.0
    a.u_inject, a.rng, a.xp, a.Cp, a.act, a.xmax_out, a.scratch = None, ops._fixed_rng(1, 1), xp.data_ptr(), Cp, None, xmax.data_ptr(), scratch.data_ptr()
    _lib.check(lib.nn_stage_fwd(C.byref(a), 0, st), "nn_stage_fwd")
    gup = torch.randn(B, Cc, PH, PW, generator=gen).to(dev)
    outs = []
    for layout in (0, PACK_SHIFT):
        b = StageBwdArgs()
        b.g, b.x, b.argmax = gup.data_ptr(), pooled.data_ptr(), amax.data_ptr()
        b.B, b.C, b.H, b.W, b.pool = B, Cc, H, W, 1
        b.mean, b.invstd, b.gamma, b.beta = mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(), beta.data_ptr()
        b.act_max, b.q_bits, b.q_hi = 5.0, 4, 5.0
        dg, db = f32(Cc), f32(Cc)
        b.dgamma, b.dbeta = dg.data_ptr(), db.data_ptr()
        if layout == 0:
            buf = torch.zeros(B, H, W, Cp, dtype=torch.bfloat16, device=dev)
        else:
            P = (B * vH * vW + 127) // 128 * 128
            buf = torch.zeros(Cp // 8, P, 8, dtype=torch.bfloat16, device=dev)
            b.gy_layout, b.virt_H, b.virt_W = PACK_SHIFT, vH, vW
        b.gyp, b.Cp, b.gy_f32, b.scratch = buf.data_ptr(), Cp, None, scratch.data_ptr()
        _lib.check(lib.nn_stage_bwd(C.byref(b), 0, st), "nn_stage_bwd")
        outs.append(buf)
    torch.cuda.synchronize()
    nhwc, planes = outs[0].float().cpu(), outs[1].float().cpu()
    P = planes.shape[1]
    grid = planes[:, :B * vH * vW].reshape(Cp // 8, B, vH, vW, 8)
    got = grid[:, :, :H, :W].permute(1, 2, 3, 0, 4).reshape(B, H, W, Cp)
    assert torch.equal(got, nhwc)
    mask = torch.ones(Cp // 8, B, vH, vW, 8, dtype=torch.bool)
    mask[:, :, :H, :W] = False
    assert float(grid[mask].abs().max()) == 0.0 and float(planes[:, B * vH * vW:].abs().max() if P > B * vH * vW else 0.0) == 0.0


@pytest.mark.parametrize("B,Cout,k", [(4, 65, 5), (3, 20, 3), (2, 4, 1), (2, 64, 3)])
def test_shift_fused_maxpool(dev, B, Cout, k):
    """pooled_out / argmax_out of the shift kernel == MaxPool2d(2,2) (values and first-maximum window position) of the
    output the same launch configuration writes without the fusion (same Philox stream -> bit-identical noise)."""
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import NOISE_MERGED, NOISE_NONE, PREC_BF16, ConvFwdArgs, ConvGeom
    import ctypes as C
    lib = _lib.load()
    H = 32
    g = ConvGeom(B, 3, H, H, Cout, k, k, 1, 0)
    OH = H - k + 1
    if OH % 2:
        pytest.skip("odd output size")
    assert lib.nn_conv_pool_fusable(C.byref(g), NOISE_MERGED, PREC_BF16) == 1
    gen = torch.Generator().manual_seed(B + Cout + k)
    s_a, ka, x, cw, wq, w_raw = _mk((B, 3, H, H, Cout, k), gen)
    xd, wqd, wrd = x.to(dev), wq.to(dev), w_raw.to(dev)
    scale = ops.tensor_stats(wrd)[1:2]
    for mode in (NOISE_MERGED, NOISE_NONE):
        kw = dict(precision="bf16", a_code_scale=s_a, w_code_scale=1.0 / 15.0, noise_mode=mode)
        if mode:
            kw.update(current=1.0, scale_dev=scale, rng=ops._fixed_rng(3, 9), want_y=False)
        ref = ops.noisy_conv_fwd(xd, wqd, wrd if mode else None, None, 1, 0, **kw)
        full = ref["y_noisy"] if mode else ref["y"]
        pv, pi = F.max_pool2d(full, 2, 2, return_indices=True)
        # window position from torch's flat index
        ih, iw = pi // OH, pi % OH
        pos = ((ih % 2) * 2 + (iw % 2)).to(torch.uint8)
        # fused launch through the C ABI
        a = ConvFwdArgs()
        a.g = g
        a.x, a.w_eff, a.w_raw = xd.data_ptr(), wqd.data_ptr(), wrd.data_ptr() if mode else None
        pooled = torch.empty(B, Cout, OH // 2, OH // 2, device=dev)
        arg = torch.empty(B, Cout, OH // 2, OH // 2, dtype=torch.uint8, device=dev)
        a.pooled_out, a.argmax_out = pooled.data_ptr(), arg.data_ptr()
        a.noise_mode = mode
        if mode:
            a.current, a.scale_dev, a.rng = 1.0, scale.data_ptr(), ops._fixed_rng(3, 9)
        a.precision, a.a_code_scale, a.w_code_scale = PREC_BF16, s_a, 1.0 / 15.0
        ws = torch.empty(int(lib.nn_conv_workspace_bytes(C.byref(g), PREC_BF16)) + 4096, dtype=torch.uint8, device=dev)
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        # ... and the batch statistics of the BatchNorm that follows the pool, from the same launch
        mean, invstd = torch.empty(Cout, device=dev), torch.empty(Cout, device=dev)
        rm, rv = torch.full((Cout,), 0.25, device=dev), torch.full((Cout,), 2.0, device=dev)
        scratch = torch.zeros(int(lib.nn_conv_bn_scratch_bytes(Cout)), dtype=torch.uint8, device=dev)
        zero = torch.full((1,), 7.0, device=dev)
        a.bn_mean, a.bn_invstd, a.bn_running_mean, a.bn_running_var = mean.data_ptr(), invstd.data_ptr(), rm.data_ptr(), rv.data_ptr()
        a.bn_eps, a.bn_momentum, a.bn_eval_mode, a.bn_scratch, a.zero_out = 1e-5, 0.1, 0, scratch.data_ptr(), zero.data_ptr()
        for rep in range(2):                # twice: the arrival ticket resets itself, the running statistics move on
            _lib.check(lib.nn_noisy_conv_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream), "nn_noisy_conv_fwd")
            assert ops.error_flag() == 0
            assert torch.equal(pooled, pv)
            assert torch.equal(arg, pos)
            m_ref = pv.double().mean(dim=(0, 2, 3))
            v_ref = pv.double().var(dim=(0, 2, 3), unbiased=False)
            assert torch.allclose(mean.double(), m_ref, rtol=1e-5, atol=1e-6)
            assert torch.allclose(invstd.double(), 1.0 / torch.sqrt(v_ref + 1e-5), rtol=1e-5)
            assert zero.item() == 0.0
        n = pv[:, 0].numel()
        rm_ref, rv_ref = torch.full((Cout,), 0.25, dtype=torch.float64, device=dev), torch.full((Cout,), 2.0, dtype=torch.float64, device=dev)
        for rep in range(2):
            rm_ref = 0.9 * rm_ref + 0.1 * m_ref
            rv_ref = 0.9 * rv_ref + 0.1 * v_ref * n / (n - 1)
        assert torch.allclose(rm.double(), rm_ref, rtol=1e-5, atol=1e-6) and torch.allclose(rv.double(), rv_ref, rtol=1e-5)
        assert int(scratch[:4].view(torch.int32).item()) == 0
