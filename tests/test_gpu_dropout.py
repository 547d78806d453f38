"""Dropout in the stage kernels (noisynet.py:456-457, :512-513, :565-566) and in the NoisyNetEngine step.

Forward: BN -> ReLU -> clamp -> x * mask * k (k = fl(1 / fl(1 - p))) -> quantize, restated in torch with the kernel's own
BatchNorm statistics and op order ((x - mean) * invstd, then one fused multiply-add with gamma and beta), so codes are
compared exactly.  Backward: torch autograd through the same chain with the same mask.  The keep mask of the Philox
stream is checked bit for bit against ``philox_keep_mask``.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import noisynet_oracle as O
from test_oracle_dropout import OracleNetDropout, apply_dropout, philox_keep_mask, philox_stage_uniform

pytestmark = pytest.mark.gpu

ACT_MAX, Q_HI, ST = 5.0, 4.0, 0.5


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__ as entry
    entry.build()
    return torch.device("cuda:0")


def _inputs(shape, seed):
    g = torch.Generator().manual_seed(seed)
    B, Cc = shape[0], shape[1]
    x = torch.randn(shape, generator=g) * 1.5 + 0.3
    gamma, beta = torch.rand(Cc, generator=g) + 0.5, torch.randn(Cc, generator=g) * 0.5 + 0.5
    return g, x, gamma, beta


def _fwd(dev, x, gamma, beta, pool, bits, p, *, u=None, keep_in=None, act=False, rng=(21, 4), drop_rng=(33, 8), stats=None,
         stoch=ST):
    """nn_stage_fwd with dropout.  stats = (mean, invstd) on the device: stats_ready launch (pool must be 0)."""
    from noisynet_b200 import _lib, ops
    lib = _lib.load()
    B, Cc, H, W = x.shape
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    Cp = (Cc + 7) // 8 * 8
    r = dict(pooled=torch.empty(B, Cc, PH, PW, device=dev), amax=torch.empty(B, Cc, PH, PW, dtype=torch.uint8, device=dev),
             mean=torch.empty(Cc, device=dev), invstd=torch.empty(Cc, device=dev),
             xp=torch.full((B, PH, PW, Cp), 7.0, dtype=torch.bfloat16, device=dev), act=torch.empty(B, Cc, PH, PW, device=dev),
             xmax=torch.zeros(1, device=dev), keep=torch.full((B, Cc, PH, PW), 9, dtype=torch.uint8, device=dev),
             scratch=torch.zeros(int(lib.nn_stage_scratch_bytes(Cc)) + 64, dtype=torch.uint8, device=dev),
             rm=torch.zeros(Cc, device=dev), rv=torch.ones(Cc, device=dev), x=x, gamma=gamma, beta=beta)
    if stats is not None:
        r["mean"].copy_(stats[0]); r["invstd"].copy_(stats[1])
    a = _lib.StageArgs()
    a.in_ = x.data_ptr(); a.B, a.C, a.H, a.W, a.pool = B, Cc, H, W, pool
    a.pooled, a.argmax = r["pooled"].data_ptr(), r["amax"].data_ptr()
    a.gamma, a.beta, a.running_mean, a.running_var = gamma.data_ptr(), beta.data_ptr(), r["rm"].data_ptr(), r["rv"].data_ptr()
    a.momentum, a.eps = 0.1, 1e-5
    a.mean, a.invstd = r["mean"].data_ptr(), r["invstd"].data_ptr()
    a.act_max, a.q_bits, a.q_hi, a.stochastic = ACT_MAX, bits, Q_HI, stoch
    a.u_inject = None if u is None else u.data_ptr()
    a.rng = ops._fixed_rng(*rng)
    a.xp, a.Cp, a.act, a.xmax_out, a.scratch = r["xp"].data_ptr(), Cp, r["act"].data_ptr() if act else None, \
        r["xmax"].data_ptr(), r["scratch"].data_ptr()
    a.stats_ready = 1 if stats is not None else 0
    a.drop_p, a.keep = p, r["keep"].data_ptr()
    a.keep_inject = None if keep_in is None else keep_in.data_ptr()
    a.drop_rng = ops._fixed_rng(*drop_rng)
    _lib.check(lib.nn_stage_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream), "nn_stage_fwd")
    torch.cuda.synchronize()
    r["bn_in"] = r["pooled"] if pool else x
    return r


def _ref_fwd(r, bits, p, u, keep):
    """The kernel's arithmetic in torch (CPU): v = fma((x - mean) * invstd, gamma, beta), ReLU, clamp, dropout, quantize."""
    x = r["bn_in"].cpu()
    Cc = x.shape[1]
    sh = (1, Cc) + (1,) * (x.dim() - 2)
    mean, invstd = r["mean"].cpu().view(sh), r["invstd"].cpu().view(sh)
    t = (x - mean) * invstd
    v = (t.double() * r["gamma"].cpu().view(sh).double() + r["beta"].cpu().view(sh).double()).float()
    v = torch.clamp(F.relu(v), max=ACT_MAX)
    v = apply_dropout(v, keep.cpu().bool(), p)
    if bits == 0:
        return v.bfloat16().float(), v
    codes = O.uniform_quantize_codes(v, bits, 0.0, Q_HI, ST, u.cpu())
    scale, _ = O.quant_scale(bits, 0.0, Q_HI)
    return codes, codes * np.float32(scale)


def _codes(r, Cc):
    xp = r["xp"].float().cpu()
    assert torch.all(xp[..., Cc:] == 0)
    return xp[..., :Cc].permute(0, 3, 1, 2)


# shape, pool, stats_ready, bits, the kernel nn_stage_fwd dispatches on the Philox path (no injected draws, no fp32 copy;
# injected draws or the fp32 copy route every case to k_bn_act_pack<true>)
FWD_CASES = [((6, 65, 28, 28), 1, False, 4, "k_bn_act_pack_tiled<true>"),      # stage 1, separate pool
             ((5, 65, 14, 14), 0, True, 4, "k_bn_act_pack_tiled<true>"),       # stage 1 after the fused conv1 pool
             ((7, 120, 10, 10), 1, False, 4, "k_bn_act_pack_lean<true>"),      # stage 2
             ((33, 390, 1, 1), 0, False, 4, "k_bn_act_pack_lean<true>"),       # stage 3
             ((40, 390, 1, 1), 0, True, 4, "k_bn_act_pack_lean<true>"),        # stage 3 after fc1's split-K statistics
             ((4, 7, 6, 6), 1, False, 4, "k_bn_act_pack_lean<true>"),          # ragged chunk
             ((6, 65, 28, 28), 1, False, 0, "k_bn_act_pack<true>"),            # q = 0: bf16 values, general kernel
             ((33, 390, 1, 1), 0, True, 0, "k_bn_act_pack<true>")]


def _stats_for(dev, x, pool):
    xin = F.max_pool2d(x, 2, 2) if pool else x
    dims = [0] + list(range(2, xin.dim()))
    m = xin.double().mean(dim=dims)
    var = xin.double().var(dim=dims, unbiased=False)
    return xin, (m.float().to(dev), (1.0 / torch.sqrt(var + 1e-5)).float().to(dev))


@pytest.mark.parametrize("shape,pool,ready,bits,hot", FWD_CASES)
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_stage_fwd_dropout_vs_torch(dev, shape, pool, ready, bits, hot, p):
    """Injected u and mask (general kernel) and the Philox path (hot kernel, u and mask from the numpy restatement of the
    stream): codes, fp32 copy and xmax exactly equal to the torch restatement."""
    g, x, gamma, beta = _inputs(shape, seed=sum(shape) + bits)
    xin, stats = _stats_for(dev, x, pool)
    B, Cc = shape[0], shape[1]
    if ready:
        x, pool, stats_arg = xin, 0, stats
    else:
        stats_arg = None
    PH, PW = (shape[2] // 2, shape[3] // 2) if (pool and not ready) else (x.shape[2], x.shape[3])
    xd, gd, bd = x.to(dev), gamma.to(dev), beta.to(dev)
    # ---- injected draws: general kernel
    u = (torch.rand(B, Cc, PH, PW, generator=g) - 0.5)
    keep = (torch.rand(B, Cc, PH, PW, generator=g) >= p).to(torch.uint8)
    r = _fwd(dev, xd, gd, bd, pool, bits, p, u=u.to(dev) if bits else None, keep_in=keep.to(dev), act=True, stats=stats_arg)
    assert torch.equal(r["keep"].cpu(), keep)
    codes_ref, act_ref = _ref_fwd(r, bits, p, u, keep)
    assert torch.equal(_codes(r, Cc), codes_ref)
    assert torch.equal(r["act"].cpu(), act_ref)
    assert r["xmax"].item() == act_ref.max().item()
    # ---- Philox draws: the hot kernel (q = 0 has no hot kernel: the general one draws the same stream)
    r = _fwd(dev, xd, gd, bd, pool, bits, p, stats=stats_arg)
    Cp = (Cc + 7) // 8 * 8
    kmask = torch.from_numpy(philox_keep_mask(B, Cc, PH * PW, Cp, p, 33, 8).reshape(B, Cc, PH, PW))
    assert torch.equal(r["keep"].cpu(), kmask)
    uu = torch.from_numpy(philox_stage_uniform(B, Cc, PH * PW, Cp, ST, 21, 4).reshape(B, Cc, PH, PW))
    codes_ref, act_ref = _ref_fwd(r, bits, p, uu, kmask)
    assert torch.equal(_codes(r, Cc), codes_ref)
    assert r["xmax"].item() == act_ref.max().item()


@pytest.mark.parametrize("shape,pool,ready,bits,hot", [c for c in FWD_CASES if c[3] == 4])
def test_stage_fwd_dropout_hot_matches_general(dev, shape, pool, ready, bits, hot):
    """Same Philox streams: the hot kernel (no fp32 copy) and the general kernel (fp32 copy requested) give bit-identical
    codes, masks and xmax with dropout on.  (Which kernel runs follows from nn_stage_fwd's dispatch
    conditions.)"""
    _, x, gamma, beta = _inputs(shape, seed=3 + sum(shape))
    xin, stats = _stats_for(dev, x, pool)
    if ready:
        x, pool = xin, 0
    xd, gd, bd = x.to(dev), gamma.to(dev), beta.to(dev)
    kw = dict(stats=stats if ready else None, rng=(5, 12), drop_rng=(6, 1 << 32))
    hot_r = _fwd(dev, xd, gd, bd, pool, bits, 0.2, **kw)
    gen_r = _fwd(dev, xd, gd, bd, pool, bits, 0.2, act=True, **kw)
    assert torch.equal(hot_r["xp"], gen_r["xp"]) and torch.equal(hot_r["keep"], gen_r["keep"])
    assert hot_r["xmax"].item() == gen_r["xmax"].item()


@pytest.mark.parametrize("shape,pool", [((64, 65, 28, 28), 1), ((512, 120, 10, 10), 1), ((512, 390, 1, 1), 0)])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_mask_is_the_philox_restatement(dev, shape, pool, p):
    """The in-kernel mask equals philox_keep_mask bit for bit, its kept fraction is within 5 sigma of 1 - p, and dropped
    elements leave code 0.  (The rounding draws' independence of the keep stream is what the Philox branch of
    test_stage_fwd_dropout_vs_torch checks: its restated u does not depend on p.)"""
    _, x, gamma, beta = _inputs(shape, seed=7)
    xd, gd, bd = x.to(dev), gamma.to(dev), beta.to(dev)
    B, Cc, H, W = shape
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    r = _fwd(dev, xd, gd, bd, pool, 4, p, drop_rng=(1234, 77))
    m = r["keep"].cpu().numpy()
    assert np.array_equal(m, philox_keep_mask(B, Cc, PH * PW, (Cc + 7) // 8 * 8, p, 1234, 77).reshape(m.shape))
    n = m.size
    assert abs(m.mean() - (1 - p)) <= 5 * np.sqrt(p * (1 - p) / n), m.mean()
    assert torch.all(_codes(r, Cc)[torch.from_numpy(m == 0)] == 0)


def _bwd(dev, r, gout, pool, bits, p, keep, planes=False, f32=False):
    from noisynet_b200 import _lib
    lib = _lib.load()
    x = r["x"]
    B, Cc, H, W = x.shape
    Cp = (Cc + 7) // 8 * 8
    if planes:
        vH, vW = H + 4, W + 4
        stride = (B * vH * vW + 127) // 128 * 128
        gyp = torch.zeros(Cp // 8 * stride * 8, dtype=torch.bfloat16, device=dev)
    else:
        gyp = torch.full((B, H, W, Cp), 3.0, dtype=torch.bfloat16, device=dev)
    gyf = torch.empty(B, Cc, H, W, device=dev)
    dg, db = torch.empty(Cc, device=dev), torch.empty(Cc, device=dev)
    b = _lib.StageBwdArgs()
    b.g = gout.data_ptr()
    b.x = r["bn_in"].data_ptr(); b.argmax = r["amax"].data_ptr()
    b.B, b.C, b.H, b.W, b.pool = B, Cc, H, W, pool
    b.mean, b.invstd, b.gamma, b.beta = r["mean"].data_ptr(), r["invstd"].data_ptr(), r["gamma"].data_ptr(), r["beta"].data_ptr()
    b.act_max, b.q_bits, b.q_hi = ACT_MAX, bits, Q_HI
    b.dgamma, b.dbeta = dg.data_ptr(), db.data_ptr()
    b.gyp, b.Cp, b.gy_f32, b.scratch = gyp.data_ptr(), Cp, gyf.data_ptr() if f32 else None, r["scratch"].data_ptr()
    if planes:
        b.gy_layout, b.virt_H, b.virt_W = 1, vH, vW
    b.drop_p, b.keep = p, keep.data_ptr()
    _lib.check(lib.nn_stage_bwd(C.byref(b), 0, torch.cuda.current_stream().cuda_stream), "nn_stage_bwd")
    torch.cuda.synchronize()
    if planes:       # planes layout [chunk][plane_stride][8] on the vH x vW grid -> NHWC [B, H, W, Cp]
        g5 = gyp.view(Cp // 8, stride, 8)[:, :B * vH * vW].view(Cp // 8, B, vH, vW, 8)[:, :, :H, :W]
        packed = g5.permute(1, 2, 3, 0, 4).reshape(B, H, W, Cp)
    else:
        packed = gyp
    return dict(packed=packed.float().cpu(), gyf=gyf.cpu(), dg=dg.cpu(), db=db.cpu())


# shape, pool, planes, the kernel nn_stage_bwd dispatches without the fp32 copy (with it: k_bn_bwd_apply<true>)
BWD_CASES = [((6, 120, 10, 10), 1, False, "k_bn_bwd_apply_img<true>"),
             ((3, 65, 28, 28), 1, False, "k_bn_bwd_apply_lean<true, false, true>"),
             ((3, 65, 28, 28), 1, True, "k_bn_bwd_apply_lean<true, true, true>"),
             ((40, 390, 1, 1), 0, False, "k_bn_bwd_apply_lean<false, false, true>"),
             ((4, 16, 6, 6), 0, True, "k_bn_bwd_apply_lean<false, true, true>")]


@pytest.mark.parametrize("shape,pool,planes,hot", BWD_CASES)
@pytest.mark.parametrize("bits", [4, 0])
def test_stage_bwd_dropout_vs_autograd(dev, shape, pool, planes, hot, bits):
    """Backward (STE on v*k, g*mask*k, clamp, ReLU, BN backward, pool routing) against torch autograd with the same
    mask; hot kernels bit-identical to the general kernel."""
    p = 0.2
    g, x, gamma, beta = _inputs(shape, seed=5 + sum(shape))
    B, Cc, H, W = shape
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    u = torch.rand(B, Cc, PH, PW, generator=g) - 0.5
    keep = (torch.rand(B, Cc, PH, PW, generator=g) >= p).to(torch.uint8)
    gout = torch.randn(B, Cc, PH, PW, generator=g)
    # ---- torch autograd
    xr = x.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    pooled = F.max_pool2d(xr, 2, 2) if pool else xr
    bn = F.batch_norm(pooled, torch.zeros(Cc), torch.ones(Cc), gr, br, True, 0.1, 1e-5)
    h = apply_dropout(torch.clamp(F.relu(bn), max=ACT_MAX), keep.bool(), p)
    q = O.OracleNet._STEQuant.apply(h, bits, 0.0, Q_HI, ST, u) if bits else h
    q.backward(gout)
    ref = xr.grad
    # ---- kernels
    xd = x.to(dev)
    r = _fwd(dev, xd, gamma.to(dev), beta.to(dev), pool, bits, p, u=u.to(dev) if bits else None, keep_in=keep.to(dev))
    gd = gout.to(dev)
    gen = _bwd(dev, r, gd, pool, bits, p, r["keep"], planes=planes, f32=True)
    hot_r = _bwd(dev, r, gd, pool, bits, p, r["keep"], planes=planes)
    tol = 2e-5 * max(1.0, ref.abs().max().item())
    assert (gen["gyf"] - ref).abs().max().item() <= tol, (gen["gyf"] - ref).abs().max()
    assert torch.allclose(gen["dg"], gr.grad, rtol=1e-4, atol=1e-4) and torch.allclose(gen["db"], br.grad, rtol=1e-4, atol=1e-4)
    packed = gen["packed"][..., :Cc].permute(0, 3, 1, 2)
    assert (packed - ref).abs().max().item() <= 4e-3 * ref.abs().max().item() + 1e-6
    assert torch.equal(hot_r["packed"][..., :Cc], gen["packed"][..., :Cc])
    assert torch.equal(hot_r["dg"], gen["dg"]) and torch.equal(hot_r["db"], gen["db"])
    assert hot_r["packed"].abs().sum().item() > 0


def test_stage_rejects_bad_dropout_arguments(dev):
    from noisynet_b200 import _lib, ops
    lib = _lib.load()
    _, x, gamma, beta = _inputs((2, 8, 4, 4), seed=1)
    xd, gd, bd = x.to(dev), gamma.to(dev), beta.to(dev)
    for p, keep in ((1.0, True), (-0.1, True), (0.2, False)):
        a = _lib.StageArgs()
        buf = torch.zeros(2, 8, 4, 4, device=dev)
        xp = torch.zeros(2, 4, 4, 8, dtype=torch.bfloat16, device=dev)
        sc = torch.zeros(int(lib.nn_stage_scratch_bytes(8)) + 64, dtype=torch.uint8, device=dev)
        km = torch.zeros(2, 8, 4, 4, dtype=torch.uint8, device=dev)
        a.in_, a.B, a.C, a.H, a.W = xd.data_ptr(), 2, 8, 4, 4
        a.gamma, a.beta, a.mean, a.invstd = gd.data_ptr(), bd.data_ptr(), buf.data_ptr(), buf.data_ptr()
        a.xp, a.Cp, a.scratch, a.rng = xp.data_ptr(), 8, sc.data_ptr(), ops._fixed_rng(1, 1)
        a.drop_p, a.keep = p, km.data_ptr() if keep else None
        assert lib.nn_stage_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream) != 0
        b = _lib.StageBwdArgs()
        b.g, b.x, b.gyp, b.scratch = buf.data_ptr(), buf.data_ptr(), xp.data_ptr(), sc.data_ptr()
        b.drop_p, b.keep = p, km.data_ptr() if keep else None
        assert lib.nn_stage_bwd(C.byref(b), 0, torch.cuda.current_stream().cuda_stream) != 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------ the engine step
def _keep_masks(oa, B, p, seed):
    g = torch.Generator().manual_seed(seed)
    C1, C2, FC = oa.fm1 * oa.width, oa.fm2 * oa.width, oa.fc * oa.width
    shapes = {"keep1": (B, C1, 14, 14), "keep2": (B, C2, 5, 5), "keep3": (B, FC)}
    return {k: (torch.rand(s, generator=g) >= p).to(torch.uint8) for k, s in shapes.items()}


def _engine_pair(dev, widths, B, current, q, p, seed=1, x_seed=10, rnd_seed=100, rec=None, **extra):
    from noisynet_b200.engine import NoisyNetEngine
    from noisynet_b200.net import NoisyNet, default_args, make_fused_optimizer, with_quant
    from test_gpu_net import _make_rnd
    qkw = dict(quant_max2=4.0, quant_max4=4.5) if q else {}
    oa = O.default_args(q_a=q, q_w=q, current=current, dropout=p, dropout_conv=p, **qkw, **widths, **extra)
    torch.manual_seed(seed)
    om = OracleNetDropout(oa).init_like_reference()
    am = float(extra.get("act_max", 5.0))
    nkw = {k: v for k, v in extra.items() if k != "act_max"}
    na = with_quant(default_args(layer_currents=[current] * 4, dropout=p, dropout_conv=p, act_max=am, act_max1=am, act_max2=am,
                                 act_max3=am, **nkw, **widths), q, q)
    nm = NoisyNet(na, fused=True, precision="bf16").to(dev)
    nm.load_state_dict(om.state_dict(), strict=False)
    if q:
        nm.quantize2.running_max = torch.tensor(4.0, device=dev)
        nm.quantize4.running_max = torch.tensor(4.5, device=dev)
    om.train(), nm.train()
    oopt = O.make_optimizer(om, oa)
    eng = NoisyNetEngine(nm, B, opt=make_fused_optimizer(nm, na))
    if rec is not None:                 # record the oracle's activation codes, quantizer by quantizer
        orig_q = om._q

        def rec_q(t, bits, lo, hi, r, name):
            y = orig_q(t, bits, lo, hi, r, name)
            if name.startswith("ua"):
                rec[name] = torch.round((y.detach() - lo) / O.quant_scale(bits, lo, hi)[0])
            return y
        om._q = rec_q
    x, lab = O.synthetic_cifar(B, seed=x_seed)
    rnd = _make_rnd(oa, B, q, rnd_seed)
    rnd.update(_keep_masks(oa, B, p, rnd_seed + 1))
    oloss, _ = O.train_step(om, oopt, x, lab, i=100, rnd=rnd)
    eng.inject = dict(u=[rnd[k].to(dev) for k in ("ua1", "ua2", "ua3", "ua4")] if q else [],
                      uw=[rnd[k].to(dev) for k in ("uw0", "uw1", "uw2", "uw3")] if q else [],
                      z=[rnd[k].to(dev) for k in ("z0", "z1", "z2", "z3")] if current > 0 else [],
                      keep=[rnd[k].to(dev) for k in ("keep1", "keep2", "keep3")] if p > 0 else [])
    loss = eng.train_step(x.to(dev), lab.to(dev))
    return om, nm, eng, oloss, loss, x, lab, rnd


def test_engine_dropout_exact_vs_oracle(dev):
    """I = 0, q4, small widths, injected u and masks: exact integer tensor-core forward -> loss within 1e-5, every
    injected mask consumed, and the masks the kernels stored are the injected ones."""
    from noisynet_b200 import ops
    om, nm, eng, oloss, loss, x, lab, rnd = _engine_pair(dev, dict(fm1=9, fm2=12, fc=24), 8, 0.0, 4, 0.2)
    assert ops.error_flag() == 0 and not eng.inject["keep"] and not eng.inject["u"]
    assert abs(loss.item() - oloss.item()) < 1e-5, (loss.item(), oloss.item())
    for i, k in enumerate(("keep1", "keep2", "keep3")):
        assert torch.equal(eng.keep[i].cpu().reshape(rnd[k].shape), rnd[k]), k
    for k in ("bn1", "bn2", "bn3", "bn4"):
        assert torch.allclose(getattr(nm, k).running_mean.cpu(), getattr(om, k).running_mean, rtol=1e-4, atol=1e-5), k


def test_engine_dropout_conv_site_follows_the_flag(dev):
    """--dropout without --dropout_conv: no mask at the conv site (noisynet.py:456), masks after relu2 and relu3."""
    from noisynet_b200.engine import NoisyNetEngine
    from noisynet_b200.net import NoisyNet, default_args, with_quant
    nm = NoisyNet(with_quant(default_args(fm1=9, fm2=12, fc=24, dropout=0.1), 4, 4), fused=True, precision="bf16").to(dev)
    nm.quantize2.running_max = torch.tensor(4.0, device=dev)
    nm.quantize4.running_max = torch.tensor(4.5, device=dev)
    eng = NoisyNetEngine(nm, 8)
    assert eng.keep[0] is None and eng.keep[1] is not None and eng.keep[2] is not None
    nm2 = NoisyNet(with_quant(default_args(fm1=9, fm2=12, fc=24), 4, 4), fused=True, precision="bf16").to(dev)
    assert NoisyNetEngine(nm2, 8).keep == [None, None, None]


GRAD_REL_TOL, GRAD_COS_TOL = 0.25, 0.98


@pytest.mark.parametrize("fuse_pool", ["1", "0"])
def test_engine_dropout_benchmark_config_vs_oracle(dev, monkeypatch, fuse_pool):
    """The benchmarked configuration (batch 512, full widths, q4, I = 1 nA) with --dropout 0.1 --dropout_conv: the
    tolerances of test_engine_benchmark_config_vs_oracle (DESIGN.md section 2)."""
    monkeypatch.setenv("NN_ENGINE_FUSE_POOL", fuse_pool)
    from noisynet_b200 import ops
    B, rec = 512, {}
    om, nm, eng, oloss, loss, x, lab, rnd = _engine_pair(dev, {}, B, 1.0, 4, 0.1, seed=3, x_seed=20, rnd_seed=300, rec=rec)
    assert ops.error_flag() == 0 and not eng.inject["keep"] and not eng.inject["z"] and not eng.inject["uw"]
    report = {"loss": (loss.item(), oloss.item())}
    codes = {"ua1": eng.xp1[..., :3].permute(0, 3, 1, 2), "ua2": eng.xp2[..., :65].permute(0, 3, 1, 2),
             "ua3": eng.xp3[..., :120].permute(0, 3, 1, 2).reshape(B, -1), "ua4": eng.xp4[:, :390]}
    for k, c in codes.items():
        d = (c.float().cpu() - rec[k].reshape(c.shape)).abs()
        report[k] = ((d > 0).float().mean().item(), d.max().item())
    og = dict(om.named_parameters())
    for k, p in nm.named_parameters():
        a, b = p.grad.cpu().flatten().double(), og[k].grad.flatten().double()
        report["g:" + k] = (((a - b).norm() / (b.norm() + 1e-30)).item(), (a @ b / (a.norm() * b.norm() + 1e-30)).item())
    print("engine vs oracle, benchmark config with dropout:", report)
    assert abs(loss.item() - oloss.item()) <= 2e-3, report
    for k, tol in {"ua1": 0.0, "ua2": 5e-4, "ua3": 1e-2, "ua4": 5e-2}.items():
        assert report[k][0] <= tol and report[k][1] <= 1.0, (k, report)
    for k, rt in (("bn1", 2e-3), ("bn2", 2e-3), ("bn3", 3e-2), ("bn4", 3e-2)):
        assert torch.allclose(getattr(nm, k).running_mean.cpu(), getattr(om, k).running_mean, rtol=rt, atol=2e-3), k
        assert torch.allclose(getattr(nm, k).running_var.cpu(), getattr(om, k).running_var, rtol=rt, atol=1e-4), k
    for k, v in report.items():
        if k.startswith("g:"):
            assert v[0] <= GRAD_REL_TOL and v[1] >= GRAD_COS_TOL, (k, v, report)


def test_engine_readme_baseline_vs_oracle(dev):
    """The README's noise-free baseline (--L2 0.0005 --dropout 0.1: q = 0, I = 0, act_max = 0) on the engine against the
    oracle with the same masks.  The engine's operands are bf16-rounded (the input too), so near-tied 2x2 pooling windows
    route some gradients to another pixel -- the analogue of the code flips of DESIGN.md section 2, whose tolerances apply:
    loss within 1.5e-2 (bf16 training tolerance), per-parameter gradient rel-L2 <= 0.25 and cosine >= 0.98.  The same
    pair at p = 0 is the control: with dropout the errors must stay of the same order (a wrong mask, scale or STE would
    show as an error many times the control's)."""
    from noisynet_b200 import ops
    l2 = dict(L2_1=5e-4, L2_2=5e-4, L2_3=5e-4, L2_4=5e-4)
    reports = {}
    for p in (0.1, 0.0):
        om, nm, eng, oloss, loss, x, lab, rnd = _engine_pair(dev, {}, 64, 0.0, 0, p, act_max=0.0, **l2)
        assert ops.error_flag() == 0 and not eng.inject.get("keep")
        assert (p > 0) == all(k is not None for k in eng.keep)
        rep = {"loss": (loss.item(), oloss.item())}
        og = dict(om.named_parameters())
        for k, prm in nm.named_parameters():
            a, b = prm.grad.cpu().flatten().double(), og[k].grad.flatten().double()
            rep[k] = (((a - b).norm() / (b.norm() + 1e-30)).item(), (a @ b / (a.norm() * b.norm() + 1e-30)).item())
        reports[p] = rep
    print("README baseline, engine vs oracle (p = 0.1, control p = 0):", reports)
    rep, ctl = reports[0.1], reports[0.0]
    assert abs(rep["loss"][0] - rep["loss"][1]) <= 1.5e-2, rep
    for k, v in rep.items():
        if k != "loss":
            assert v[0] <= GRAD_REL_TOL and v[1] >= GRAD_COS_TOL, (k, v, reports)
            assert v[0] <= 4 * ctl[k][0] + 2e-2, (k, v, ctl[k])


def test_engine_dropout_graph_trains(dev):
    """The step with dropout captures as one CUDA graph: 25 replays, loss finite and falling, a fresh mask on every replay;
    eval_forward ignores p (same logits as a p = 0 engine on the same state)."""
    from noisynet_b200 import ops
    from noisynet_b200.engine import NoisyNetEngine
    from noisynet_b200.net import NoisyNet, default_args, init_like_reference, make_fused_optimizer, with_quant
    B = 256
    na = with_quant(default_args(dropout=0.1, dropout_conv=0.1), 4, 4)
    torch.manual_seed(6)
    nm = init_like_reference(NoisyNet(na, fused=True, precision="bf16")).to(dev)
    nm.quantize2.running_max = torch.tensor(5.0, device=dev)
    nm.quantize4.running_max = torch.tensor(5.0, device=dev)
    nm.collect_stats = False
    nm.train()
    eng = NoisyNetEngine(nm, B, opt=make_fused_optimizer(nm, na))
    x, lab = O.synthetic_cifar(B, seed=8)
    sx, sy = x.to(dev), lab.to(dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            eng.train_step(sx, sy)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    loss_out = torch.zeros((), device=dev)
    ctr = torch.zeros(1, dtype=torch.int64, device=dev)
    graph = torch.cuda.CUDAGraph()
    with ops.graph_rng(ctr, seed=11):
        with torch.cuda.graph(graph):
            loss_out.copy_(eng.train_step(sx, sy)[0])
            ops.rng_advance(ctr, 1)
    torch.cuda.synchronize()
    losses, masks = [], []
    for _ in range(25):
        graph.replay()
        losses.append(loss_out.item())
        masks.append(eng.keep[1].clone())
    assert ops.error_flag() == 0
    assert all(np.isfinite(losses)) and np.mean(losses[-5:]) < np.mean(losses[:5]), losses
    for a, b in zip(masks, masks[1:]):
        assert not torch.equal(a, b)
    frac = torch.stack(masks).float().mean().item()
    assert abs(frac - 0.9) < 0.01, frac
    # eval: dropout is the identity -> the same logits as a p = 0 engine on the same state and noise seed
    nm.eval()
    torch.manual_seed(5)
    out1 = eng.eval_forward(sx).clone()
    nm0 = NoisyNet(with_quant(default_args(), 4, 4), fused=True, precision="bf16").to(dev)
    nm0.load_state_dict(nm.state_dict())
    nm0.quantize3.max_value = nm.quantize3.max_value           # the same quantize3 range: compare the dropout switch alone
    nm0.eval()
    eng0 = NoisyNetEngine(nm0, B)
    torch.manual_seed(5)
    out0 = eng0.eval_forward(sx).clone()
    assert ops.error_flag() == 0
    assert torch.isfinite(out1).all() and torch.equal(out1, out0)
