"""Fused between-layer stages (SURVEY section 8f.1) and the NoisyNetEngine training step.

Stage kernels are compared with the torch ops the reference script composes (MaxPool2d, BatchNorm, ReLU,
clamp, the oracle quantizer) -- fp32, tolerance 1e-5; quantisation codes may flip where the BN output sits
within rounding of a code boundary, hence a mismatch-fraction criterion (<= 2e-4) for codes.
The whole engine step (bf16 tensor-core contractions, bf16 gradients) is compared with the CPU oracle's step:
forward loss within 2e-3, gradients within 2e-2 of each tensor's max (bf16 training tolerance).
"""
import ctypes as C

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


def _stage_call(dev, x, gamma, beta, rm, rv, pool, act_max, bits, q_hi, u):
    from noisynet_b200 import _lib
    lib = _lib.load()
    B, Cc, H, W = x.shape
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    Cp = (Cc + 7) // 8 * 8
    pooled = torch.empty(B, Cc, PH, PW, device=dev)
    amax = torch.empty(B, Cc, PH, PW, dtype=torch.uint8, device=dev)
    mean, invstd = torch.empty(Cc, device=dev), torch.empty(Cc, device=dev)
    xp = torch.zeros(B, PH, PW, Cp, dtype=torch.bfloat16, device=dev)
    act = torch.empty(B, Cc, PH, PW, device=dev)
    xmax = torch.zeros(1, device=dev)
    scratch = torch.zeros(int(lib.nn_stage_scratch_bytes(Cc)) + 64, dtype=torch.uint8, device=dev)
    a = _lib.StageArgs()
    a.in_ = x.data_ptr(); a.B, a.C, a.H, a.W, a.pool = B, Cc, H, W, pool
    a.pooled, a.argmax = pooled.data_ptr(), amax.data_ptr()
    a.gamma, a.beta, a.running_mean, a.running_var = gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr()
    a.momentum, a.eps = 0.1, 1e-5
    a.mean, a.invstd = mean.data_ptr(), invstd.data_ptr()
    a.act_max, a.q_bits, a.q_hi, a.stochastic = act_max, bits, q_hi, 0.5
    a.u_inject = u.data_ptr()
    a.rng = _lib.Rng(0, 0, None)
    a.xp, a.Cp, a.act, a.xmax_out, a.scratch = xp.data_ptr(), Cp, act.data_ptr(), xmax.data_ptr(), scratch.data_ptr()
    _lib.check(lib.nn_stage_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream), "nn_stage_fwd")
    return dict(pooled=pooled, amax=amax, mean=mean, invstd=invstd, xp=xp, act=act, xmax=xmax, scratch=scratch)


@pytest.mark.parametrize("shape,pool", [((6, 65, 28, 28), 1), ((5, 120, 10, 10), 1), ((33, 390, 1, 1), 0), ((4, 7, 6, 6), 1)])
def test_stage_fwd_bwd_vs_torch(dev, shape, pool):
    from noisynet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(sum(shape))
    B, Cc, H, W = shape
    x = torch.randn(shape, generator=g) * 1.5 + 0.3
    gamma, beta = torch.rand(Cc, generator=g) + 0.5, torch.randn(Cc, generator=g) * 0.5 + 0.5
    act_max, bits, q_hi = 5.0, 4, 4.0
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    u = torch.rand(B, Cc, PH, PW, generator=g) - 0.5
    gout = torch.randn(B, Cc, PH, PW, generator=g)
    # ---- torch / oracle reference
    xr = x.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rm, rv = torch.zeros(Cc), torch.ones(Cc)
    pooled = F.max_pool2d(xr, 2, 2) if pool else xr
    bn = F.batch_norm(pooled, rm, rv, gr, br, True, 0.1, 1e-5)
    h = torch.clamp(F.relu(bn), max=act_max)
    q = O.OracleNet._STEQuant.apply(h, bits, 0.0, q_hi, 0.5, u)
    q.backward(gout)
    codes_ref = O.uniform_quantize_codes(h.detach(), bits, 0.0, q_hi, 0.5, u)
    # ---- kernels
    xd = x.to(dev)
    rmd, rvd = torch.zeros(Cc, device=dev), torch.ones(Cc, device=dev)
    r = _stage_call(dev, xd, gamma.to(dev), beta.to(dev), rmd, rvd, pool, act_max, bits, q_hi, u.to(dev))
    if pool:
        assert torch.equal(r["pooled"].cpu(), pooled.detach())
    assert torch.allclose(rmd.cpu(), rm, rtol=1e-5, atol=1e-6) and torch.allclose(rvd.cpu(), rv, rtol=1e-4, atol=1e-6)
    codes = r["xp"].float().cpu()[..., :Cc].permute(0, 3, 1, 2)
    bad = (codes != codes_ref).float().mean().item()
    assert bad <= 2e-4, bad
    assert torch.all(r["xp"].float().cpu()[..., Cc:] == 0)
    assert (r["act"].cpu() - q.detach()).abs().max().item() <= (q_hi / 15) + 1e-5 and \
        ((r["act"].cpu() - q.detach()).abs() > 1e-5).float().mean().item() <= 2e-4
    assert r["xmax"].item() == pytest.approx(r["act"].max().item())
    # ---- backward
    Cp = (Cc + 7) // 8 * 8
    gyp = torch.zeros(B, H, W, Cp, dtype=torch.bfloat16, device=dev)
    gyf = torch.empty(B, Cc, H, W, device=dev)
    dg, db = torch.empty(Cc, device=dev), torch.empty(Cc, device=dev)
    b = _lib.StageBwdArgs()
    b.g = gout.to(dev).data_ptr()
    gkeep = gout.to(dev)
    b.g = gkeep.data_ptr()
    b.x = (r["pooled"] if pool else xd).data_ptr(); b.argmax = r["amax"].data_ptr()
    b.B, b.C, b.H, b.W, b.pool = B, Cc, H, W, pool
    gd, bd = gamma.to(dev), beta.to(dev)
    b.mean, b.invstd, b.gamma, b.beta = r["mean"].data_ptr(), r["invstd"].data_ptr(), gd.data_ptr(), bd.data_ptr()
    b.act_max, b.q_bits, b.q_hi = act_max, bits, q_hi
    b.dgamma, b.dbeta = dg.data_ptr(), db.data_ptr()
    b.gyp, b.Cp, b.gy_f32, b.scratch = gyp.data_ptr(), Cp, gyf.data_ptr(), r["scratch"].data_ptr()
    _lib.check(lib.nn_stage_bwd(C.byref(b), 0, torch.cuda.current_stream().cuda_stream), "nn_stage_bwd")
    ref = xr.grad
    tol = 2e-5 * max(1.0, ref.abs().max().item())
    assert (gyf.cpu() - ref).abs().max().item() <= tol, (gyf.cpu() - ref).abs().max()
    assert torch.allclose(dg.cpu(), gr.grad, rtol=1e-4, atol=1e-4) and torch.allclose(db.cpu(), br.grad, rtol=1e-4, atol=1e-4)
    packed = gyp.float().cpu()[..., :Cc].permute(0, 3, 1, 2)
    assert (packed - ref).abs().max().item() <= 4e-3 * ref.abs().max().item() + 1e-6       # bf16 rounding of the pack


@pytest.mark.parametrize("shape,pool", [((7, 65, 28, 28), 1), ((5, 120, 10, 10), 1), ((3, 16, 12, 12), 0), ((40, 390, 1, 1), 0)])
def test_stage_fwd_hot_path_kernels_match_general(dev, shape, pool):
    """The training hot path (Philox stochastic rounding, no fp32 copy) runs k_bn_act_pack_tiled (HW >= 32) or
    k_bn_act_pack_lean; asking for the fp32 copy routes the same call through the general kernel.  Same Philox counter
    per (pixel, chunk) -> the packed codes must be bit-identical (ragged last tile, even/odd chunk counts)."""
    from noisynet_b200 import _lib, ops
    lib = _lib.load()
    g = torch.Generator().manual_seed(11 + sum(shape))
    B, Cc, H, W = shape
    x = (torch.randn(shape, generator=g) * 1.5 + 0.3).to(dev)
    gamma, beta = (torch.rand(Cc, generator=g) + 0.5).to(dev), (torch.randn(Cc, generator=g) * 0.5 + 0.5).to(dev)
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    Cp = (Cc + 7) // 8 * 8
    outs = []
    for want_act in (False, True):
        pooled = torch.empty(B, Cc, PH, PW, device=dev)
        amax = torch.empty(B, Cc, PH, PW, dtype=torch.uint8, device=dev)
        mean, invstd = torch.empty(Cc, device=dev), torch.empty(Cc, device=dev)
        rm, rv = torch.zeros(Cc, device=dev), torch.ones(Cc, device=dev)
        xp = torch.full((B, PH, PW, Cp), 7.0, dtype=torch.bfloat16, device=dev)
        act = torch.empty(B, Cc, PH, PW, device=dev)
        xmax = torch.zeros(1, device=dev)
        scratch = torch.zeros(int(lib.nn_stage_scratch_bytes(Cc)) + 64, dtype=torch.uint8, device=dev)
        a = _lib.StageArgs()
        a.in_ = x.data_ptr(); a.B, a.C, a.H, a.W, a.pool = B, Cc, H, W, pool
        a.pooled, a.argmax = pooled.data_ptr(), amax.data_ptr()
        a.gamma, a.beta, a.running_mean, a.running_var = gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr()
        a.momentum, a.eps = 0.1, 1e-5
        a.mean, a.invstd = mean.data_ptr(), invstd.data_ptr()
        a.act_max, a.q_bits, a.q_hi, a.stochastic = 5.0, 4, 4.0, 0.5
        a.u_inject = None
        a.rng = ops._fixed_rng(21, 4)
        a.xp, a.Cp, a.act, a.xmax_out, a.scratch = xp.data_ptr(), Cp, act.data_ptr() if want_act else None, xmax.data_ptr(), scratch.data_ptr()
        _lib.check(lib.nn_stage_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream), "nn_stage_fwd")
        torch.cuda.synchronize()
        outs.append((xp.float().cpu(), xmax.item()))
    assert torch.equal(outs[0][0], outs[1][0])
    assert outs[0][1] == outs[1][1]
    assert 0.0 < outs[0][0][..., :Cc].mean().item() < 15.0 and torch.all(outs[0][0][..., Cc:] == 0)


@pytest.mark.parametrize("B,Cc", [(7, 3), (2, 1), (5, 4)])
def test_input_quant_pack_hot_path_matches_general(dev, B, Cc):
    """nn_input_quant_pack: the 4-pixels-per-thread kernel of the training hot path (no fp32 copy) against the general kernel
    (fp32 copy requested) with the same Philox stream: bit-identical codes; the codes dequantise to the fp32 copy."""
    from noisynet_b200 import _lib, ops
    lib = _lib.load()
    g = torch.Generator().manual_seed(B * 10 + Cc)
    x = (torch.rand(B, Cc, 32, 32, generator=g)).to(dev)
    outs = []
    for want_act in (False, True):
        xp = torch.full((B, 32, 32, 8), 9.0, dtype=torch.bfloat16, device=dev)
        act = torch.empty_like(x)
        _lib.check(lib.nn_input_quant_pack(x.data_ptr(), xp.data_ptr(), act.data_ptr() if want_act else None, B, Cc, 32 * 32, 8, 4, 1.0, 0.5,
                                           None, ops._fixed_rng(5, 17), 0, torch.cuda.current_stream().cuda_stream), "nn_input_quant_pack")
        torch.cuda.synchronize()
        outs.append((xp.float().cpu(), act.cpu()))
    assert torch.equal(outs[0][0], outs[1][0])
    codes = outs[0][0][..., :Cc].permute(0, 3, 1, 2)
    assert torch.all(outs[0][0][..., Cc:] == 0) and codes.max() <= 15 and codes.min() >= 0
    assert torch.allclose(codes * np.float32(1.0 / 15.0), outs[1][1], rtol=0, atol=1e-7)
    assert (codes - x.cpu() * 15).abs().max() <= 1.0 + 1e-4            # stochastic rounding moves a value by less than one level


@pytest.mark.parametrize("shape,pool", [((6, 120, 10, 10), 1), ((3, 65, 28, 28), 1), ((5, 16, 12, 12), 1), ((40, 390, 1, 1), 0)])
def test_stage_bwd_hot_path_kernels_match_general(dev, shape, pool):
    """nn_stage_bwd without the fp32 copy runs the hot-path kernels (k_bn_bwd_apply_img for pooled NHWC stages whose
    image fits shared memory, k_bn_bwd_apply_lean otherwise); with gy_f32 it runs the general kernel.  Same arithmetic ->
    the packed bf16 gradients must be bit-identical."""
    from noisynet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(5 + sum(shape))
    B, Cc, H, W = shape
    x = (torch.randn(shape, generator=g) * 1.5 + 0.3).to(dev)
    gamma, beta = (torch.rand(Cc, generator=g) + 0.5).to(dev), (torch.randn(Cc, generator=g) * 0.5 + 0.5).to(dev)
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    u = (torch.rand(B, Cc, PH, PW, generator=g) - 0.5).to(dev)
    gout = torch.randn(B, Cc, PH, PW, generator=g).to(dev)
    rm, rv = torch.zeros(Cc, device=dev), torch.ones(Cc, device=dev)
    r = _stage_call(dev, x, gamma, beta, rm, rv, pool, 5.0, 4, 4.0, u)
    Cp = (Cc + 7) // 8 * 8
    outs = []
    for want_f32 in (False, True):
        gyp = torch.full((B, H, W, Cp), 3.0, dtype=torch.bfloat16, device=dev)
        gyf = torch.empty(B, Cc, H, W, device=dev)
        dg, db = torch.empty(Cc, device=dev), torch.empty(Cc, device=dev)
        b = _lib.StageBwdArgs()
        b.g = gout.data_ptr()
        b.x = (r["pooled"] if pool else x).data_ptr(); b.argmax = r["amax"].data_ptr()
        b.B, b.C, b.H, b.W, b.pool = B, Cc, H, W, pool
        b.mean, b.invstd, b.gamma, b.beta = r["mean"].data_ptr(), r["invstd"].data_ptr(), gamma.data_ptr(), beta.data_ptr()
        b.act_max, b.q_bits, b.q_hi = 5.0, 4, 4.0
        b.dgamma, b.dbeta = dg.data_ptr(), db.data_ptr()
        b.gyp, b.Cp, b.gy_f32, b.scratch = gyp.data_ptr(), Cp, gyf.data_ptr() if want_f32 else None, r["scratch"].data_ptr()
        _lib.check(lib.nn_stage_bwd(C.byref(b), 0, torch.cuda.current_stream().cuda_stream), "nn_stage_bwd")
        torch.cuda.synchronize()
        outs.append((gyp.float().cpu(), dg.cpu(), db.cpu()))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
    assert outs[0][0].abs().sum().item() > 0


@pytest.mark.parametrize("B", [200, 512, 37, 1500])      # 1500 > 1024 rows: the strided single-block kernel
def test_head_vs_torch(dev, B):
    from noisynet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(3)
    Cc = 10
    z = torch.randn(B, Cc, generator=g) * 2
    lab = torch.randint(0, Cc, (B,), generator=g)
    gamma, beta = torch.rand(Cc, generator=g) + 0.5, torch.randn(Cc, generator=g) * 0.1
    zr = z.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rm, rv = torch.zeros(Cc), torch.ones(Cc)
    out = F.batch_norm(zr, rm, rv, gr, br, True, 0.1, 1e-5)
    loss = F.cross_entropy(out, lab)
    loss.backward()
    zd, ld = z.to(dev), lab.to(dev)
    gd, bd, rmd, rvd = gamma.to(dev), beta.to(dev), torch.zeros(Cc, device=dev), torch.ones(Cc, device=dev)
    lo, o, gg = torch.zeros(1, device=dev), torch.empty(B, Cc, device=dev), torch.empty(B, Cc, device=dev)
    gp = torch.zeros(B, 16, dtype=torch.bfloat16, device=dev)
    dg, db = torch.empty(Cc, device=dev), torch.empty(Cc, device=dev)
    _lib.check(lib.nn_head_fwd_bwd(zd.data_ptr(), ld.data_ptr(), B, Cc, gd.data_ptr(), bd.data_ptr(), rmd.data_ptr(),
                                   rvd.data_ptr(), 0.1, 1e-5, lo.data_ptr(), o.data_ptr(), gg.data_ptr(), gp.data_ptr(), 16,
                                   dg.data_ptr(), db.data_ptr(), 0, torch.cuda.current_stream().cuda_stream))
    assert abs(lo.item() - loss.item()) < 1e-5
    assert torch.allclose(o.cpu(), out.detach(), rtol=1e-5, atol=1e-5)
    assert torch.allclose(gg.cpu(), zr.grad, rtol=1e-4, atol=1e-7)
    assert torch.allclose(dg.cpu(), gr.grad, rtol=1e-4, atol=1e-6) and torch.allclose(db.cpu(), br.grad, rtol=1e-4, atol=1e-6)
    assert torch.allclose(rmd.cpu(), rm, rtol=1e-5, atol=1e-6) and torch.allclose(rvd.cpu(), rv, rtol=1e-4, atol=1e-6)
    assert torch.allclose(gp.float().cpu()[:, :Cc], zr.grad, rtol=1e-2, atol=1e-6)


def _engine_pair(dev, widths, B, current):
    from noisynet_b200.engine import NoisyNetEngine
    from noisynet_b200.net import NoisyNet, default_args, make_fused_optimizer, with_quant
    from test_gpu_net import _make_rnd
    q = 4
    oa = O.default_args(q_a=q, q_w=q, quant_max2=4.0, quant_max4=4.5, current=current, **widths)
    torch.manual_seed(1)
    om = O.OracleNet(oa).init_like_reference()
    na = with_quant(default_args(layer_currents=[current] * 4, **widths), q, q)
    nm = NoisyNet(na, fused=True, precision="bf16").to(dev)
    nm.load_state_dict(om.state_dict(), strict=False)
    nm.quantize2.running_max = torch.tensor(4.0, device=dev)
    nm.quantize4.running_max = torch.tensor(4.5, device=dev)
    om.train(), nm.train()
    oopt = O.make_optimizer(om, oa)
    eng = NoisyNetEngine(nm, B, opt=make_fused_optimizer(nm, na))
    x, lab = O.synthetic_cifar(B, seed=10)
    rnd = _make_rnd(oa, B, q, 100)
    oloss, _ = O.train_step(om, oopt, x, lab, i=100, rnd=rnd)
    eng.inject = dict(u=[rnd[k].to(dev) for k in ("ua1", "ua2", "ua3", "ua4")],
                      uw=[rnd[k].to(dev) for k in ("uw0", "uw1", "uw2", "uw3")],
                      z=[rnd[k].to(dev) for k in ("z0", "z1", "z2", "z3")] if current > 0 else [])
    loss = eng.train_step(x.to(dev), lab.to(dev))
    return om, nm, eng, oloss, loss, x, lab


def test_engine_forward_exact_vs_oracle(dev):
    """I = 0 (no analog noise): the tensor-core forward is exact integer arithmetic, the engine's 4-bit codes
    equal the oracle's and the loss agrees to 1e-5.  (Gradients are NOT compared here: noise-free conv outputs
    sit on a discrete grid, 2x2 pooling windows tie, and tie-breaking under 1e-7 rounding differences routes
    the gradient differently -- both valid.)"""
    from noisynet_b200 import ops
    om, nm, eng, oloss, loss, x, lab = _engine_pair(dev, dict(fm1=9, fm2=12, fc=24), 8, 0.0)
    assert ops.error_flag() == 0 and not eng.inject["u"]
    assert abs(loss.item() - oloss.item()) < 1e-5, (loss.item(), oloss.item())
    for k in ("bn1", "bn2", "bn3", "bn4"):
        assert torch.allclose(getattr(nm, k).running_mean.cpu(), getattr(om, k).running_mean, rtol=1e-4, atol=1e-5), k
        assert torch.allclose(getattr(nm, k).running_var.cpu(), getattr(om, k).running_var, rtol=1e-3, atol=1e-5), k
    assert nm.conv1.weight.abs().max().item() <= torch.tensor(0.3).item()


@pytest.mark.parametrize("widths,B", [(dict(fm1=9, fm2=12, fc=24), 8), ({}, 16)])
def test_engine_step_vs_module_path(dev, widths, B):
    """Wiring check at I = 1 nA: the engine (stage kernels, packed operands, explicit backward) against the
    autograd module path (NoisyNet(fused=True, precision='bf16'): same tensor-core contractions, torch pool / BN /
    ReLU / clamp, nn_quantize kernels) with identical injected draws.  The module path itself is pinned to the
    oracle in test_gpu_net.py (fp32) and its bf16 kernels to the fp32 ones in test_gpu_umma*.py.
    Tolerance: loss 2e-3, gradients rel-L2 2e-2 (rare 4-bit code flips from 1e-7 BatchNorm rounding differences)."""
    from noisynet_b200 import ops
    from noisynet_b200.engine import NoisyNetEngine
    from noisynet_b200.net import NoisyNet, default_args, with_quant
    from test_gpu_net import _make_rnd
    q = 4
    torch.manual_seed(2)
    na = with_quant(default_args(**widths), q, q)
    ref = NoisyNet(na, fused=True, precision="bf16").to(dev)
    eng_m = NoisyNet(na, fused=True, precision="bf16").to(dev)
    eng_m.load_state_dict(ref.state_dict())
    for mdl in (ref, eng_m):
        mdl.quantize2.running_max = torch.tensor(4.0, device=dev)
        mdl.quantize4.running_max = torch.tensor(4.5, device=dev)
        mdl.collect_stats = False
        mdl.train()
    oa = O.default_args(q_a=q, q_w=q, **widths)
    x, lab = O.synthetic_cifar(B, seed=11)
    x, lab = x.to(dev), lab.to(dev)
    rnd = _make_rnd(oa, B, q, 200)
    us = [rnd[k].to(dev) for k in ("ua1", "uw0", "ua2", "uw1", "ua3", "uw2", "ua4", "uw3")]
    zs = [rnd[k].to(dev) for k in ("z0", "z1", "z2", "z3")]
    with ops.inject_random(list(us), list(zs)):
        out = ref(x, 0, 100)
        rloss = F.cross_entropy(out, lab)
        rloss.backward()
    eng = NoisyNetEngine(eng_m, B, opt=None)
    eng.inject = dict(u=[us[0], us[2], us[4], us[6]], uw=[us[1], us[3], us[5], us[7]], z=list(zs))
    loss = eng.train_step(x, lab)
    assert ops.error_flag() == 0 and not eng.inject["u"] and not eng.inject["z"]
    assert abs(loss.item() - rloss.item()) < 2e-3, (loss.item(), rloss.item())
    rg = dict(ref.named_parameters())
    for k, p in eng_m.named_parameters():
        g_ref = rg[k].grad
        rel = ((p.grad - g_ref).norm() / (g_ref.norm() + 1e-12)).item()
        assert rel < 2e-2, (k, rel)
    for k in ("bn1", "bn2", "bn3", "bn4"):
        assert torch.allclose(getattr(eng_m, k).running_mean, getattr(ref, k).running_mean, rtol=1e-3, atol=1e-4), k
        assert torch.allclose(getattr(eng_m, k).running_var, getattr(ref, k).running_var, rtol=2e-3, atol=1e-4), k


def test_engine_step_with_noise(dev):
    """I = 1 nA: sigma is computed from bf16 weights (3e-3 relative), which flips a few 4-bit codes downstream
    (discrete, chaotic amplification) -- the per-layer noise maths is pinned in test_gpu_umma.py; here the whole
    step must stay close in loss and keep training."""
    from noisynet_b200 import ops
    om, nm, eng, oloss, loss, x, lab = _engine_pair(dev, dict(fm1=9, fm2=12, fc=24), 8, 1.0)
    assert ops.error_flag() == 0 and not eng.inject["u"] and not eng.inject["z"]
    assert abs(loss.item() - oloss.item()) < 0.1, (loss.item(), oloss.item())
    eng.inject = None
    losses = [eng.train_step(x.to(dev), lab.to(dev)).item() for _ in range(25)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    assert ops.error_flag() == 0


def test_engine_eval_forward_vs_oracle(dev):
    """model.eval() forward (noisynet.py:1560-1567) on the engine's kernels: BatchNorm with running statistics, no
    stochastic rounding.  I = 0: exact integer tensor-core arithmetic -> logits equal the oracle's to 2e-4 after a
    training step has moved the running statistics.  I = 1 nA: the accurate noise model is injected in eval too
    (hardware_model.py:43) -> logits differ from the noise-free ones, reproducibly for a fixed seed."""
    from noisynet_b200 import ops
    om, nm, eng, oloss, loss, x, lab = _engine_pair(dev, dict(fm1=9, fm2=12, fc=24), 8, 0.0)
    om.eval(), nm.eval()
    with torch.no_grad():
        ref = om(x, i=100)
    out = eng.eval_forward(x.to(dev)).cpu()
    assert ops.error_flag() == 0
    eng.sync_bn_counters()
    assert int(nm.bn1.num_batches_tracked) == 1
    # both models took one (slightly different: bf16 gradients) optimizer step: compare on the ORACLE's state
    nm.load_state_dict(om.state_dict(), strict=False)
    nm.w_absmax.clear()
    out = eng.eval_forward(x.to(dev)).cpu()
    assert torch.allclose(out, ref, rtol=2e-4, atol=2e-4), (out - ref).abs().max()
    assert int(nm.bn1.num_batches_tracked) == int(om.bn1.num_batches_tracked) == 1
    om1, nm1, eng1, _, _, x1, _ = _engine_pair(dev, dict(fm1=9, fm2=12, fc=24), 8, 1.0)
    nm1.eval()
    torch.manual_seed(5)
    a = eng1.eval_forward(x1.to(dev)).clone()
    b = eng1.eval_forward(x1.to(dev), currents=[1e9] * 4).clone()         # practically noise-free
    torch.manual_seed(5)
    c = eng1.eval_forward(x1.to(dev)).clone()
    assert torch.isfinite(a).all() and (a - b).abs().max().item() > 1e-3
    assert torch.equal(a, c)


GRAD_REL_TOL, GRAD_COS_TOL = 0.25, 0.98        # a few % of fc2's input codes differ (see below)


@pytest.mark.parametrize("fuse_pool", ["1", "0"])
def test_engine_benchmark_config_vs_oracle(dev, monkeypatch, fuse_pool):
    """The configuration bench.py measures -- NoisyNetEngine.train_step at batch 512, full widths (65 / 120 / 390),
    q_a = q_w = 4, I = 1 nA on every layer -- against the CPU oracle's training step (oracle/noisynet_oracle.py, pinned to
    the unmodified reference by tests/golden) with the SAME injected draws (stochastic-rounding uniforms of the four
    activation and four weight quantizers, the four Gaussian noise tensors).

    What can differ: the engine's sigma uses bf16-rounded g(|w|) (<= 3e-3 relative), its BatchNorm statistics are summed
    in a different order (1e-6), the Box-Muller-free injected z is identical.  A perturbation of 1e-3 sigma moves a
    pre-quantizer activation by ~1e-4 of a 4-bit step (5/15), so a small FRACTION of codes lands on the other side of a
    rounding boundary; every flipped code is a full-step difference that the next layer sees.  Stated tolerances:
      * loss: |d| <= 2e-3;
      * 4-bit codes entering conv1 identical; entering conv2 <= 0.05 %, fc1 <= 1 %, fc2 <= 5 % differ (every flipped code
        perturbs the next layer: the fraction grows with depth), none by more than one level;
      * BatchNorm running statistics: rtol 2e-3 (bn1, bn2), 3e-2 behind the flipped codes (bn3, bn4);
      * gradients of every parameter against the ORACLE's: relative L2 error <= GRAD_REL_TOL, cosine >= GRAD_COS_TOL
        (bf16 grad_output operands + the flipped codes, whose STE masks and ReLU gates switch whole gradient paths).
    """
    monkeypatch.setenv("NN_ENGINE_FUSE_POOL", fuse_pool)      # conv1 + pool + bn1 statistics in one launch / separate stage
    from noisynet_b200 import ops
    from noisynet_b200.engine import NoisyNetEngine
    from noisynet_b200.net import NoisyNet, default_args, make_fused_optimizer, with_quant
    from test_gpu_net import _make_rnd
    B, q, current = 512, 4, 1.0
    oa = O.default_args(q_a=q, q_w=q, quant_max2=5.0, quant_max4=5.0, current=current)
    torch.manual_seed(3)
    om = O.OracleNet(oa).init_like_reference()
    na = with_quant(default_args(layer_currents=[current] * 4), q, q)
    nm = NoisyNet(na, fused=True, precision="bf16").to(dev)
    nm.load_state_dict(om.state_dict(), strict=False)
    nm.quantize2.running_max = torch.tensor(5.0, device=dev)
    nm.quantize4.running_max = torch.tensor(5.0, device=dev)
    om.train(), nm.train()
    oopt = O.make_optimizer(om, oa)
    eng = NoisyNetEngine(nm, B, opt=make_fused_optimizer(nm, na))
    x, lab = O.synthetic_cifar(B, seed=20)
    rnd = _make_rnd(oa, B, q, 300)
    rec = {}
    orig_q = om._q

    def rec_q(t, bits, lo, hi, r, name):
        y = orig_q(t, bits, lo, hi, r, name)
        if name.startswith("ua"):
            s = O.quant_scale(bits, lo, hi)[0]
            rec[name] = torch.round((y.detach() - lo) / s)
        return y
    om._q = rec_q
    oloss, _ = O.train_step(om, oopt, x, lab, i=100, rnd=rnd)
    eng.inject = dict(u=[rnd[k].to(dev) for k in ("ua1", "ua2", "ua3", "ua4")],
                      uw=[rnd[k].to(dev) for k in ("uw0", "uw1", "uw2", "uw3")],
                      z=[rnd[k].to(dev) for k in ("z0", "z1", "z2", "z3")])
    loss = eng.train_step(x.to(dev), lab.to(dev))
    assert ops.error_flag() == 0 and not eng.inject["u"] and not eng.inject["z"] and not eng.inject["uw"]
    report = {"loss": (loss.item(), oloss.item())}
    # 4-bit activation codes, layer by layer
    codes = {"ua1": eng.xp1[..., :3].permute(0, 3, 1, 2), "ua2": eng.xp2[..., :65].permute(0, 3, 1, 2),
             "ua3": eng.xp3[..., :120].permute(0, 3, 1, 2).reshape(B, -1), "ua4": eng.xp4[:, :390]}
    for k, c in codes.items():
        d = (c.float().cpu() - rec[k].reshape(c.shape)).abs()
        report[k] = ((d > 0).float().mean().item(), d.max().item())
    og = dict(om.named_parameters())
    for k, p in nm.named_parameters():
        a, b = p.grad.cpu().flatten().double(), og[k].grad.flatten().double()
        rel = ((a - b).norm() / (b.norm() + 1e-30)).item()
        cos = (a @ b / (a.norm() * b.norm() + 1e-30)).item()
        report["g:" + k] = (rel, cos)
    print("engine vs oracle at the benchmark configuration:", report)
    assert abs(loss.item() - oloss.item()) <= 2e-3, report
    flip_tol = {"ua1": 0.0, "ua2": 5e-4, "ua3": 1e-2, "ua4": 5e-2}
    for k, tol in flip_tol.items():
        assert report[k][0] <= tol and report[k][1] <= 1.0, (k, report)
    for k, rt in (("bn1", 2e-3), ("bn2", 2e-3), ("bn3", 3e-2), ("bn4", 3e-2)):      # behind the flipped codes: looser
        assert torch.allclose(getattr(nm, k).running_mean.cpu(), getattr(om, k).running_mean, rtol=rt, atol=2e-3), k
        assert torch.allclose(getattr(nm, k).running_var.cpu(), getattr(om, k).running_var, rtol=rt, atol=1e-4), k
    for k, v in report.items():
        if k.startswith("g:"):
            assert v[0] <= GRAD_REL_TOL and v[1] >= GRAD_COS_TOL, (k, v, report)


@pytest.mark.parametrize("B,current", [(512, 1.0), (200, 1.0), (96, 0.0)])
def test_classifier_tail_matches_separate_kernels(dev, B, current):
    """nn_classifier_tail (one 8-CTA cluster) == nn_noisy_conv_fwd (integer-code tensor-core path, same Philox stream) ->
    nn_head_fwd_bwd -> nn_noisy_conv_dgrad on the same inputs.  The main contraction is exact in both; sigma^2 is the
    same bf16 operands summed in a different fp32 order (1e-6 relative), everything after is fp32 on equal inputs."""
    import ctypes as C
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_NONE, PREC_BF16, ConvDgradArgs, ConvGeom, TailArgs
    lib = _lib.load()
    K, Cc, Kp = 390, 10, 392
    gen = torch.Generator().manual_seed(B)
    s_a, w_cs = 5.0 / 15.0, 1.0 / 15.0
    ka = torch.randint(0, 16, (B, K), generator=gen).float() * (torch.rand(B, K, generator=gen) > 0.4).float()
    codes = (torch.randint(0, 16, (Cc, K), generator=gen) * 2 - 15).to(torch.int8)
    w_raw = torch.randn(Cc, K, generator=gen) * 0.2
    lab = torch.randint(0, Cc, (B,), generator=gen)
    gamma, beta = torch.rand(Cc, generator=gen) + 0.5, torch.randn(Cc, generator=gen) * 0.1
    xp = torch.zeros(B, Kp, dtype=torch.bfloat16)
    xp[:, :K] = ka.bfloat16()
    xpd, cd, wrd, labd = xp.to(dev), codes.to(dev), w_raw.to(dev), lab.to(dev)
    gd, bd = gamma.to(dev), beta.to(dev)
    xd = (ka * s_a).float().to(dev).view(B, K, 1, 1)
    wqd = (codes.float() * w_cs).to(dev).view(Cc, K, 1, 1)
    scale = ops.tensor_stats(xd)[0:1]
    mode = NOISE_EXTERNAL if current > 0 else NOISE_NONE
    st = torch.cuda.current_stream().cuda_stream
    f32 = lambda *s: torch.zeros(*s, device=dev)
    # --- separate kernels
    kw = dict(precision="bf16", a_code_scale=s_a, w_code_scale=w_cs, noise_mode=mode)
    if mode:
        kw.update(current=current, scale_dev=scale, rng=ops._fixed_rng(21, 4), want_y=False)
    r = ops.noisy_conv_fwd(xd, wqd, wrd.view(Cc, K, 1, 1) if mode else None, None, 1, 0, **kw)
    logits = (r["y_noisy"] if mode else r["y"]).view(B, Cc).contiguous()
    loss0, g0, gp0, dg0, db0 = f32(1), f32(B, Cc), torch.zeros(B, 16, dtype=torch.bfloat16, device=dev), f32(Cc), f32(Cc)
    rm0, rv0 = f32(Cc), torch.ones(Cc, device=dev)
    _lib.check(lib.nn_head_fwd_bwd(logits.data_ptr(), labd.data_ptr(), B, Cc, gd.data_ptr(), bd.data_ptr(), rm0.data_ptr(),
                                   rv0.data_ptr(), 0.1, 1e-5, loss0.data_ptr(), None, g0.data_ptr(), gp0.data_ptr(), 16,
                                   dg0.data_ptr(), db0.data_ptr(), 0, st), "nn_head_fwd_bwd")
    gx0 = ops.conv_dgrad(gp0[:, :Cc].float().view(B, Cc, 1, 1).contiguous(), wqd, (B, K, 1, 1), precision="bf16", w_code_scale=w_cs)
    # --- fused
    a = TailArgs()
    a.xp, a.B, a.K, a.Kp, a.C = xpd.data_ptr(), B, K, Kp, Cc
    a.w_codes, a.w_raw, a.a_code_scale, a.w_code_scale = cd.data_ptr(), wrd.data_ptr(), s_a, w_cs
    a.noise_mode = mode
    if mode:
        a.current, a.scale_dev, a.rng = current, scale.data_ptr(), ops._fixed_rng(21, 4)
    a.labels, a.gamma, a.beta = labd.data_ptr(), gd.data_ptr(), bd.data_ptr()
    rm1, rv1 = f32(Cc), torch.ones(Cc, device=dev)
    a.running_mean, a.running_var, a.momentum, a.eps = rm1.data_ptr(), rv1.data_ptr(), 0.1, 1e-5
    loss1, lg1, g1, gp1 = f32(1), f32(B, Cc), f32(B, Cc), torch.zeros(B, 16, dtype=torch.bfloat16, device=dev)
    gx1, dg1, db1 = f32(B, K), f32(Cc), f32(Cc)
    a.loss_out, a.logits_out, a.g, a.g_packed, a.Cp_g = loss1.data_ptr(), lg1.data_ptr(), g1.data_ptr(), gp1.data_ptr(), 16
    a.gx, a.dgamma, a.dbeta = gx1.data_ptr(), dg1.data_ptr(), db1.data_ptr()
    _lib.check(lib.nn_classifier_tail(C.byref(a), 0, st), "nn_classifier_tail")
    torch.cuda.synchronize()
    assert torch.allclose(lg1, logits, rtol=1e-5, atol=1e-5)
    assert torch.allclose(loss1, loss0, rtol=1e-5, atol=1e-6)
    assert torch.allclose(g1, g0, rtol=1e-4, atol=2e-7)
    assert torch.allclose(dg1, dg0, rtol=1e-4, atol=1e-6) and torch.allclose(db1, db0, rtol=1e-4, atol=1e-6)
    assert torch.allclose(rm1, rm0, rtol=1e-5, atol=1e-6) and torch.allclose(rv1, rv0, rtol=1e-5, atol=1e-6)
    assert (gp1.float() - gp0.float()).abs().max().item() <= 1e-2 * g0.abs().max().item()      # one bf16 ulp where g differs by 1e-7
    assert torch.allclose(gx1, gx0.view(B, K), rtol=1e-3, atol=2e-3 * gx0.abs().max().item())
