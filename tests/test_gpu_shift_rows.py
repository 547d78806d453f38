"""The shift-GEMM forward on its row-plane input image: one K = 16 wgmma per (kernel row, plane pair).

- CPU: a Python restatement of make_shift_plan (planes, chain length, weight image bytes, stage bytes, shared memory,
  refusals), pinned against the library's byte queries and nn_conv_pack_layout.
- The row-plane image from nn_input_quant_pack_rows against a torch restatement, exactly (right-edge zeros, P = 2 and
  P = 4, stochastic and deterministic rounding), and its NHWC image bit-identical to nn_input_quant_pack's.
- The NN_PACK_SHIFT weight image of nn_prepare_weights against a restatement, exactly.
- The forward on prepacked operands at batch 512 (y exactly against float64, y_noisy against the tiled kernel to the
  sigma tolerance of test_gpu_shift.py, pooled values / window positions / bn1 statistics as test_pooled), the plane
  geometries (KH 1..7, P = 2 / 4 / 6, W not a multiple of 8, more tiles than SMs) and a geometry whose planes do not
  fit in shared memory, which runs on the tiled kernel with the same exact y.  Every launch asserts under
  torch.profiler which kernel ran.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

import __graft_entry__ as entry


def _pad(v, m):
    return (v + m - 1) // m * m


def planes(cin, kw):
    return 2 * ((kw * cin + 15) // 16)


def shift_plan(B, cin, H, W, cout, kh, kw, noisy):
    """make_shift_plan (csrc/nn_conv_umma.cu): None where the shift kernel does not serve the geometry"""
    if cin > 8 or kh > H or kw > W or W >= 4096 or B * H * W >= 1 << 31:
        return None
    n_t = _pad(cout, 8)
    n_mma = _pad(2 * n_t if noisy else n_t, 16)
    P = planes(cin, kw)
    steps = kh * P // 2
    if n_mma > 256 or steps > 64:
        return None
    a_plane = _pad(max(128 + (kh - 1) * W, (15 + kh - 1) * W + 8) * 16, 128)
    b_bytes = kh * P * n_mma * 16
    smem = 128 + b_bytes + 2 * P * a_plane + 32 + 96 + 4 * 64 + 16 + 12 * 1024 + 128 * (n_mma + 4) * 4
    if smem > 227 * 1024:
        return None
    return dict(P=P, steps=steps, n_mma=n_mma, b_bytes=b_bytes, a_stage=P * a_plane, smem=smem)


@pytest.fixture(scope="module")
def lib():
    entry.build()
    from noisynet_b200 import _lib
    return _lib.load()


PLAN_CASES = [  # B, Cin, H, W, Cout, k
    (512, 3, 32, 32, 65, 5),      # conv1: P = 2, a chain of 5
    (5, 8, 9, 11, 120, 3),        # P = 4, W = 11
    (2, 8, 20, 20, 16, 5),        # P = 6
    (2, 1, 16, 16, 33, 7),        # P = 2, KH = 7
    (1, 8, 100, 100, 16, 3),      # P = 4 on a 100-wide input: the planes do not fit
    (1, 8, 40, 40, 16, 7),        # P = 8, 28 steps, 40 wide: the planes do not fit
    (3, 3, 32, 32, 200, 5),       # 400 noisy columns: refused noisy, served plain
]


def test_plan_restated(lib):
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_NONE, PACK_SHIFT, PREC_BF16, ConvGeom, WPrepJob
    for B, cin, H, W, cout, k in PLAN_CASES:
        g = ConvGeom(B, cin, H, W, cout, k, k, 1, 0)
        assert lib.nn_conv_shift_planes_bytes(C.byref(g)) == planes(cin, k) * B * H * W * 16
        for noisy in (False, True):
            sp = shift_plan(B, cin, H, W, cout, k, k, noisy)
            layout = lib.nn_conv_pack_layout(C.byref(g), NOISE_EXTERNAL if noisy else NOISE_NONE, PREC_BF16)
            assert (layout == PACK_SHIFT) == (sp is not None), (B, cin, H, W, cout, k, noisy)
            jb = WPrepJob()
            jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.m_rows = cout, cin, k * k, 0, B
            jb.noise_mode, jb.layout = NOISE_EXTERNAL if noisy else NOISE_NONE, PACK_SHIFT
            n_mma = _pad(2 * _pad(cout, 8) if noisy else _pad(cout, 8), 16)
            assert lib.nn_weight_pack_bytes(C.byref(jb)) == _pad(k * planes(cin, k) * n_mma * 16, 1024)
            if sp is not None:
                ws = lib.nn_conv_workspace_bytes(C.byref(g), PREC_BF16)
                assert ws >= _pad(planes(cin, k) * B * H * W * 16, 1024) + _pad(sp["b_bytes"], 1024) + 1024
    assert shift_plan(512, 3, 32, 32, 65, 5, 5, True)["steps"] == 5
    assert shift_plan(512, 3, 32, 32, 65, 5, 5, True)["b_bytes"] == 23040
    assert shift_plan(1, 8, 100, 100, 16, 3, 3, False) is None and shift_plan(1, 8, 40, 40, 16, 7, 7, False) is None
    # non-square kernels are packed by the library itself; nn_prepare_weights refuses them
    jb = WPrepJob()
    jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.layout = 16, 3, 6, 0, PACK_SHIFT
    assert lib.nn_weight_pack_bytes(C.byref(jb)) == 0


# ---------------------------------------------------------------------------------------------------------------- GPU
def _profiled(fn, want):
    """fn() under torch.profiler, asserting that a kernel whose name contains `want` ran.  Late in a long test process the
    profiler sometimes records no device activity for a session (only the launch calls); the launches are deterministic,
    so such a call is profiled again, up to three times in all."""
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = [e.key for e in prof.key_averages()]
        if any(want in n for n in names):
            return out
    raise AssertionError((want, names))


def rows_ref(codes, kw):
    """the row-plane image of NHWC-ordered codes [B, C, H, W] (float): [P, B, H, W, 8]"""
    B, Cc, H, W = codes.shape
    P = planes(Cc, kw)
    out = torch.zeros(P * 8, B, H, W, dtype=codes.dtype)
    for e in range(min(P * 8, kw * Cc)):
        k, c = divmod(e, Cc)
        out[e, :, :, :W - k] = codes[:, c, :, k:]
    return out.reshape(P, 8, B, H, W).permute(0, 2, 3, 4, 1).contiguous()


def _run_pack_rows(lib, x, kw, q_bits, stoch, rng, want_xp=True, u=None):
    from noisynet_b200 import _lib
    B, Cc, H, W = x.shape
    g = _lib.ConvGeom(B, Cc, H, W, 8, kw, kw, 1, 0)
    n = int(lib.nn_conv_shift_planes_bytes(C.byref(g))) // 2
    pl = torch.full((n,), 7.0, dtype=torch.bfloat16, device=x.device)
    xp = torch.full((B, H, W, 8), 7.0, dtype=torch.bfloat16, device=x.device) if want_xp else None
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.nn_input_quant_pack_rows(x.data_ptr(), xp.data_ptr() if want_xp else None, pl.data_ptr(), B, Cc, H, W, kw,
                                            q_bits, 5.0, stoch, u.data_ptr() if u is not None else None, rng, 0, st),
               "nn_input_quant_pack_rows")
    torch.cuda.synchronize()
    return pl.reshape(planes(Cc, kw), B, H, W, 8), xp


@pytest.mark.gpu
@pytest.mark.parametrize("B,Cc,H,W,kw", [
    (8, 3, 32, 32, 5), (4, 4, 32, 32, 5), (3, 3, 20, 32, 3), (2, 1, 32, 32, 5),       # the 32-wide hot kernel: P = 2, 4, 2, 2
    (3, 3, 12, 12, 3), (2, 1, 16, 16, 5), (3, 8, 9, 11, 3), (2, 3, 10, 14, 7),      # the general one: P = 2, 2, 4, 4
    (2, 2, 8, 12, 4), (2, 6, 32, 32, 7), (2, 3, 32, 32, 4)])                        # P = 2, 6 (42 of 48), 2
@pytest.mark.parametrize("stoch", [0.0, 0.5])
def test_pack_rows_matches_restatement(lib, B, Cc, H, W, kw, stoch):
    """planes == the restatement of the NHWC codes of nn_input_quant_pack (same rng), which the same launch also writes"""
    from noisynet_b200 import _lib, ops
    gen = torch.Generator().manual_seed(B * 100 + Cc * 10 + kw)
    x = (torch.rand(B, Cc, H, W, generator=gen) * 6.0 - 0.5).cuda()
    rng = ops._fixed_rng(9, 4) if stoch else _lib.Rng(0, 0, None)
    ref = torch.zeros(B, H, W, 8, dtype=torch.bfloat16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.nn_input_quant_pack(x.data_ptr(), ref.data_ptr(), None, B, Cc, H * W, 8, 4, 5.0, stoch, None, rng, 0, st),
               "nn_input_quant_pack")
    pl, xp = _run_pack_rows(lib, x, kw, 4, stoch, rng)
    assert torch.equal(xp, ref)
    codes = ref.float().cpu().permute(0, 3, 1, 2)[:, :Cc]
    want = rows_ref(codes, kw)
    assert torch.equal(pl.float().cpu(), want)
    # the last column holds its own pixel's codes only: zero past them (right edge, and K past KW * Cin)
    assert float(pl[0, :, :, W - 1, Cc:].float().abs().sum()) == 0.0
    # from the NHWC codes alone (x = NULL): the same planes
    pl2 = torch.full_like(pl, 3.0)
    _lib.check(lib.nn_input_quant_pack_rows(None, ref.data_ptr(), pl2.data_ptr(), B, Cc, H, W, kw, 4, 5.0, stoch, None, rng, 0, st),
               "nn_input_quant_pack_rows")
    torch.cuda.synchronize()
    assert torch.equal(pl2, pl)
    # without the NHWC image: the same planes
    pl3, _ = _run_pack_rows(lib, x, kw, 4, stoch, rng, want_xp=False)
    assert torch.equal(pl3, pl)


@pytest.mark.gpu
def test_pack_rows_injected_draws(lib):
    from noisynet_b200 import _lib
    gen = torch.Generator().manual_seed(3)
    B, Cc, H, W = 4, 3, 32, 32
    x = (torch.rand(B, Cc, H, W, generator=gen) * 6.0).cuda()
    u = (torch.rand(B, Cc, H, W, generator=gen) - 0.5).cuda()
    ref = torch.zeros(B, H, W, 8, dtype=torch.bfloat16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.nn_input_quant_pack(x.data_ptr(), ref.data_ptr(), None, B, Cc, H * W, 8, 4, 5.0, 0.5, u.data_ptr(),
                                       _lib.Rng(0, 0, None), 0, st), "nn_input_quant_pack")
    pl, xp = _run_pack_rows(lib, x, 5, 4, 0.5, _lib.Rng(0, 0, None), u=u)
    assert torch.equal(xp, ref)
    assert torch.equal(pl.float().cpu(), rows_ref(ref.float().cpu().permute(0, 3, 1, 2)[:, :Cc], 5))


@pytest.mark.gpu
@pytest.mark.parametrize("cin,k,cout,noisy", [(3, 5, 65, True), (3, 5, 65, False), (8, 3, 120, True), (8, 5, 20, True), (1, 7, 9, True)])
def test_weight_image_matches_restatement(lib, cin, k, cout, noisy):
    from noisynet_b200 import _lib
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_NONE, PACK_SHIFT, WPrepJob
    gen = torch.Generator().manual_seed(cin * 7 + k + cout)
    w = (torch.randint(0, 16, (cout, cin, k, k), generator=gen) * 2 - 15).float()
    wd = w.cuda()
    jb = WPrepJob()
    jb.w_raw = wd.data_ptr()
    jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.m_rows = cout, cin, k * k, 0, 512
    jb.noise_mode, jb.want_wsum, jb.q_bits, jb.layout = NOISE_EXTERNAL if noisy else NOISE_NONE, 0, 0, PACK_SHIFT
    nbytes = int(lib.nn_weight_pack_bytes(C.byref(jb)))
    buf = torch.full((nbytes // 2,), 9.0, dtype=torch.bfloat16, device="cuda")
    jb.packed_out = buf.data_ptr()
    _lib.check(lib.nn_prepare_weights(C.byref(jb), 1, 0, torch.cuda.current_stream().cuda_stream), "nn_prepare_weights")
    torch.cuda.synchronize()
    n_t = _pad(cout, 8)
    n_mma = _pad(2 * n_t if noisy else n_t, 16)
    P = planes(cin, k)
    want = torch.zeros(k, P * 8, n_mma)
    a = w.abs()
    for kh in range(k):
        for e in range(k * cin):
            kw, c = divmod(e, cin)
            want[kh, e, :cout] = w[:, c, kh, kw]
            if noisy:
                want[kh, e, n_t:n_t + cout] = a[:, c, kh, kw] * a[:, c, kh, kw] + a[:, c, kh, kw]
    want = want.reshape(k, P, 8, n_mma).permute(0, 1, 3, 2).bfloat16().float()     # [kh][plane][row][8]
    got = buf[:k * P * n_mma * 8].reshape(k, P, n_mma, 8).float().cpu()
    assert torch.equal(got, want)


def _mk(B, cin, H, W, cout, kh, kw, seed):
    gen = torch.Generator().manual_seed(seed)
    s_a = 5.0 / 15.0
    ka = torch.randint(0, 16, (B, cin, H, W), generator=gen).float()
    cw = (torch.randint(0, 16, (cout, cin, kh, kw), generator=gen) * 2 - 15).float()
    return s_a, ka, cw


def _check_geometry(lib, B, cin, H, W, cout, kh, kw, want_kernel):
    """the library's own pack (fp32 x): plain y exactly against float64 and bit-identical to the tiled kernel's, noisy
    y_noisy to the sigma tolerance against the tiled kernel"""
    from noisynet_b200 import ops
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_NONE
    s_a, ka, cw = _mk(B, cin, H, W, cout, kh, kw, B + cin * 3 + H + cout + kh * 7 + kw)
    x, wq, wr = (ka * s_a).cuda(), (cw / 15.0).cuda(), (cw / 15.0 * 0.7).cuda()
    exact = F.conv2d(ka.double(), cw.double()) * (float(np.float32(s_a)) * float(np.float32(1.0 / 15.0)))
    kw_ = dict(precision="bf16", a_code_scale=s_a, w_code_scale=1.0 / 15.0)
    try:
        lib.nn_debug_shift_enable(1)
        a = _profiled(lambda: ops.noisy_conv_fwd(x, wq, None, None, 1, 0, noise_mode=NOISE_NONE, **kw_)["y"], want_kernel)
        assert ops.error_flag() == 0
        assert torch.allclose(a.cpu().double(), exact, rtol=1e-6, atol=1e-9)
        lib.nn_debug_shift_enable(0)
        b = ops.noisy_conv_fwd(x, wq, None, None, 1, 0, noise_mode=NOISE_NONE, **kw_)["y"]
        assert torch.equal(a, b)
        scale = ops.tensor_stats(x)[0:1]
        common = dict(noise_mode=NOISE_EXTERNAL, current=1.0, scale_dev=scale, **kw_)
        ref = ops.noisy_conv_fwd(x, wq, wr, None, 1, 0, rng=ops._fixed_rng(7, 3), want_z=True, want_sigma=True, **common)
        tol = 1e-5 * float(ref["sigma"].abs().max()) * float(ref["z"].abs().max()) + 1e-6
        lib.nn_debug_shift_enable(1)
        c = ops.noisy_conv_fwd(x, wq, wr, None, 1, 0, rng=ops._fixed_rng(7, 3), **common)
        assert ops.error_flag() == 0
        assert torch.equal(c["y"], ref["y"])
        assert (c["y_noisy"] - ref["y_noisy"]).abs().max().item() <= tol
    finally:
        lib.nn_debug_shift_enable(1)


GEOMS = [  # B, Cin, H, W, Cout, KH, KW
    (3, 3, 16, 16, 33, 1, 1),     # P = 2, one step
    (3, 2, 16, 18, 33, 2, 4),     # P = 2, 2 steps
    (3, 3, 14, 14, 40, 3, 3),     # P = 2, 3 steps
    (2, 4, 12, 12, 17, 4, 5),     # P = 4, 8 steps: a block of 5 and one of 3
    (3, 8, 9, 11, 120, 3, 3),     # P = 4, W = 11
    (2, 8, 16, 13, 24, 5, 5),     # P = 6, 15 steps, W = 13
    (2, 3, 20, 20, 16, 6, 6),     # P = 4 (18 of 32)
    (2, 2, 16, 16, 33, 7, 7),     # P = 2, KH = 7
    (2, 5, 12, 15, 9, 7, 2),      # P = 2, KH = 7, KW = 2
    (300, 2, 12, 12, 33, 3, 3),   # more tiles than SMs
]


@pytest.mark.gpu
@pytest.mark.parametrize("geom", GEOMS)
def test_plane_geometries(lib, geom):
    B, cin, H, W, cout, kh, kw = geom
    assert shift_plan(B, cin, H, W, cout, kh, kw, True) is not None
    _check_geometry(lib, *geom, "k_conv_shift<")


@pytest.mark.gpu
def test_refused_geometry_runs_tiled(lib):
    """Cin = 8 with a 3 x 3 kernel on a 100-wide input: 4 planes of 17 rows do not fit in shared memory (the tap-pair
    kernel served it) -- the tiled kernel computes the same exact y"""
    from noisynet_b200._lib import NOISE_NONE, PACK_TILED, PREC_BF16, ConvGeom
    assert shift_plan(1, 8, 100, 100, 16, 3, 3, False) is None
    g = ConvGeom(1, 8, 100, 100, 16, 3, 3, 1, 0)
    assert lib.nn_conv_pack_layout(C.byref(g), NOISE_NONE, PREC_BF16) == PACK_TILED
    _check_geometry(lib, 1, 8, 100, 100, 16, 3, 3, "k_conv_umma")


@pytest.mark.gpu
@pytest.mark.parametrize("pooled", [False, True])
def test_prepacked_forward_batch512(lib, pooled):
    """conv1 at batch 512 as the engine runs it: the row-plane image from nn_input_quant_pack_rows (stochastic rounding),
    the NN_PACK_SHIFT image from nn_prepare_weights, noisy (Philox) forward"""
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import NOISE_EXTERNAL, PACK_SHIFT, PREC_BF16, ConvFwdArgs, ConvGeom, WPrepJob
    B, cin, H, cout, k = 512, 3, 32, 65, 5
    OH = H - k + 1
    g = ConvGeom(B, cin, H, H, cout, k, k, 1, 0)
    assert lib.nn_conv_pack_layout(C.byref(g), NOISE_EXTERNAL, PREC_BF16) == PACK_SHIFT
    gen = torch.Generator().manual_seed(512)
    x = (torch.rand(B, cin, H, H, generator=gen) * 5.5).cuda()
    cw = (torch.randint(0, 16, (cout, cin, k, k), generator=gen) * 2 - 15).float()
    cwd = cw.cuda()
    st = torch.cuda.current_stream().cuda_stream
    pl, xp = _run_pack_rows(lib, x, k, 4, 0.5, ops._fixed_rng(21, 2))
    jb = WPrepJob()
    jb.w_raw = cwd.data_ptr()
    jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.m_rows = cout, cin, k * k, 0, B * OH * OH
    jb.noise_mode, jb.q_bits, jb.layout = NOISE_EXTERNAL, 0, PACK_SHIFT
    wbuf = torch.zeros(int(lib.nn_weight_pack_bytes(C.byref(jb))) + 1024, dtype=torch.uint8, device="cuda")
    jb.packed_out = (wbuf.data_ptr() + 1023) // 1024 * 1024
    _lib.check(lib.nn_prepare_weights(C.byref(jb), 1, 0, st), "nn_prepare_weights")
    s_a, wsc = 5.0 / 15.0, 1.0 / 15.0
    ka = xp.float().cpu()[..., :cin].permute(0, 3, 1, 2).contiguous()
    exact = F.conv2d(ka.double(), cw.double()) * (float(np.float32(s_a)) * float(np.float32(wsc)))
    scale = ops.tensor_stats(x)[0:1]
    ws = torch.empty(int(lib.nn_conv_workspace_bytes(C.byref(g), PREC_BF16)) + 4096, dtype=torch.uint8, device="cuda")

    def launch(y, yn, pooled_out=None, arg=None, bn=None):
        a = ConvFwdArgs()
        a.g = g
        a.x, a.x_packed, a.w_packed, a.w_packed_layout = None, pl.data_ptr(), jb.packed_out, PACK_SHIFT
        a.y, a.y_noisy = (y.data_ptr() if y is not None else None), (yn.data_ptr() if yn is not None else None)
        a.noise_mode, a.current, a.scale_dev, a.rng = NOISE_EXTERNAL, 1.0, scale.data_ptr(), ops._fixed_rng(5, 2)
        a.precision, a.a_code_scale, a.w_code_scale = PREC_BF16, s_a, wsc
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        if pooled_out is not None:
            a.pooled_out, a.argmax_out = pooled_out.data_ptr(), arg.data_ptr()
            mean, invstd, rm, rv, scratch = bn
            a.bn_mean, a.bn_invstd, a.bn_running_mean, a.bn_running_var = mean.data_ptr(), invstd.data_ptr(), rm.data_ptr(), rv.data_ptr()
            a.bn_eps, a.bn_momentum, a.bn_eval_mode, a.bn_scratch = 1e-5, 0.1, 0, scratch.data_ptr()
        return _lib.check(lib.nn_noisy_conv_fwd(C.byref(a), 0, st), "nn_noisy_conv_fwd")

    y, yn = torch.empty(B, cout, OH, OH, device="cuda"), torch.empty(B, cout, OH, OH, device="cuda")
    _profiled(lambda: launch(y, yn), "k_conv_shift<1, 16, false>")
    assert ops.error_flag() == 0
    assert torch.allclose(y.cpu().double(), exact, rtol=1e-6, atol=1e-9)
    if not pooled:
        # the tiled kernel on the same codes (fp32 input = codes x s_a, weights = codes x wsc, sigma rows from |codes|)
        try:
            lib.nn_debug_shift_enable(0)
            ref = ops.noisy_conv_fwd((ka * s_a).cuda(), (cw * wsc).cuda(), cwd, None, 1, 0, noise_mode=NOISE_EXTERNAL, current=1.0,
                                     scale_dev=scale, rng=ops._fixed_rng(5, 2), want_z=True, want_sigma=True, precision="bf16",
                                     a_code_scale=s_a, w_code_scale=wsc)
        finally:
            lib.nn_debug_shift_enable(1)
        assert torch.equal(ref["y"], y)
        tol = 1e-5 * float(ref["sigma"].abs().max()) * float(ref["z"].abs().max()) + 1e-6
        assert (yn - ref["y_noisy"]).abs().max().item() <= tol
        return
    pv, pi = F.max_pool2d(yn, 2, 2, return_indices=True)
    ih, iw = pi // OH, pi % OH
    pos = ((ih % 2) * 2 + (iw % 2)).to(torch.uint8)
    po = torch.empty(B, cout, OH // 2, OH // 2, device="cuda")
    arg = torch.empty(B, cout, OH // 2, OH // 2, dtype=torch.uint8, device="cuda")
    bn = (torch.empty(cout, device="cuda"), torch.empty(cout, device="cuda"), torch.zeros(cout, device="cuda"),
          torch.ones(cout, device="cuda"), torch.zeros(int(lib.nn_conv_bn_scratch_bytes(cout)), dtype=torch.uint8, device="cuda"))
    _profiled(lambda: launch(None, None, po, arg, bn), "k_conv_shift<1, 16, true>")
    assert ops.error_flag() == 0
    assert torch.equal(po, pv)
    assert torch.equal(arg, pos)
    m_ref = pv.double().mean(dim=(0, 2, 3))
    v_ref = pv.double().var(dim=(0, 2, 3), unbiased=False)
    assert torch.allclose(bn[0].double(), m_ref, rtol=1e-5, atol=1e-6)
    assert torch.allclose(bn[1].double(), 1.0 / torch.sqrt(v_ref + 1e-5), rtol=1e-5)
