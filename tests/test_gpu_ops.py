"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle and the golden
fixtures minted from the reference.  Tolerances are stated per test:
  * quantizer / STE / AddNoise / clamp: BIT-EXACT (fp32 op-for-op restatement);
  * fp32 CUDA-core contractions: 1e-5 relative to the fp32 oracle (summation order only);
  * in-kernel Philox normals vs the numpy restatement: mean abs error < 5e-6, max < 2e-3 (MUFU lg2/sqrt/sin/cos).
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


def T(a):
    return torch.from_numpy(np.asarray(a))


def test_device_info(dev):
    import ctypes as C
    from noisynet_b200 import _lib
    sm, ma, mi = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.load().nn_device_info(0, C.byref(sm), C.byref(ma), C.byref(mi)))
    assert (ma.value, mi.value) == (9, 0) and sm.value >= 100


# ------------------------------------------------------------------------------ a1 / a2
def test_quantize_golden_bit_exact(dev, golden):
    from noisynet_b200 import ops
    g = golden("quant")
    x = T(g["kat_hm_x"]).to(dev)
    assert torch.equal(ops.quantize_fwd(x, 4, 0.0, 5.0).cpu(), T(g["kat_hm_y"]))
    assert torch.equal(ops.quantize_bwd(x, torch.arange(1.0, 12.0, device=dev), 0.0, 5.0).cpu(), T(g["kat_hm_g"]))
    assert torch.equal(ops.quantize_fwd(T(g["wq_x"]).to(dev), 4, -1.0, 1.0).cpu(), T(g["wq_y"]))
    assert torch.equal(ops.quantize_fwd(T(g["floor_x"]).to(dev), 4, 0.0, 0.0).cpu(), T(g["floor_y"]))
    for ci, (bits, lo, hi, st) in enumerate(g["r_params"]):
        x, u = T(g[f"r{ci}_x"]).to(dev), T(g[f"r{ci}_u"]).to(dev)
        y = ops.quantize_fwd(x, int(bits), lo, hi, st, u=u if st > 0 else None)
        assert torch.equal(y.cpu(), T(g[f"r{ci}_y"])), ci
        gin = ops.quantize_bwd(x, T(g[f"r{ci}_gout"]).to(dev), lo, hi)
        assert torch.equal(gin.cpu(), T(g[f"r{ci}_gin"])), ci


def test_quantize_philox_matches_spec(dev):
    """In-kernel Philox uniform == numpy restatement, bit-exact, incl. ragged tail and odd sizes."""
    from noisynet_b200 import ops
    for n in (1, 3, 4, 5, 1023, 4099):
        x = torch.rand(n, generator=torch.Generator().manual_seed(n)) * 6 - 0.5
        y = ops.quantize_fwd(x.to(dev), 4, 0.0, 5.0, 0.5, rng=ops._fixed_rng(77, 12345))
        u = torch.from_numpy(O.philox_uniform_sym(n, 77, 12345, 0.5))
        assert torch.equal(y.cpu(), O.uniform_quantize_fwd(x, 4, 0.0, 5.0, 0.5, u)), n


def test_quantize_autograd_function_and_inplace(dev):
    from noisynet_b200.hardware_model import QuantMeasure, UniformQuantize
    x = (torch.rand(3, 5, 7, device=dev) * 7 - 1).requires_grad_(True)
    y = UniformQuantize().apply(x, 4, 0.0, 5.0, 0, False, False)       # the reference's call form
    y.backward(torch.ones_like(y))
    assert torch.equal(x.grad.cpu(), ((x.detach() >= 0) & (x.detach() <= 5)).float().cpu())
    assert torch.equal(y.detach().cpu(), O.uniform_quantize_fwd(x.detach().cpu(), 4, 0.0, 5.0))
    qm = QuantMeasure(4, max_value=5.0, inplace=True).to(dev).eval()
    h = x.detach().clone() * 1.0
    out = qm(h)
    assert out.data_ptr() == h.data_ptr()
    assert torch.equal(out.cpu(), O.uniform_quantize_fwd(x.detach().cpu(), 4, 0.0, 5.0))
    # stochastic rounding is unbiased: mean code error ~ 0, and it is off in eval
    qt = QuantMeasure(4, max_value=5.0).to(dev).train()
    big = torch.full((400000,), 1.1, device=dev)        # 1.1 / (5/15) = 3.3 -> code 3 w.p. 0.7, code 4 w.p. 0.3
    m = qt(big).mean().item()
    assert abs(m - 1.1) < 3e-3
    assert torch.equal(qt.eval()(big), torch.full_like(big, O.uniform_quantize_fwd(torch.tensor([1.1]), 4, 0, 5.0).item()))


def test_quantize_empty_and_large(dev):
    from noisynet_b200 import ops
    assert ops.quantize_fwd(torch.empty(0, device=dev), 4, 0.0, 1.0).numel() == 0
    n = 512 * 65 * 14 * 14 + 3
    x = torch.rand(n, device=dev) * 6
    y = ops.quantize_fwd(x, 4, 0.0, 5.0)
    codes = torch.round(y / (5.0 / 15))
    assert codes.min() >= 0 and codes.max() <= 15
    assert torch.equal(ops.quantize_fwd(y, 4, 0.0, 5.0), y)          # idempotent on the grid


def test_quant_measure_ranges(dev, golden):
    from noisynet_b200 import hardware_model as hm, quant as q
    g = golden("quant")
    x = T(g["qm_run_x"]).to(dev)
    qm = hm.QuantMeasure(4, stochastic=0.5, pctl=99.0, calculate_running=True).to(dev).train()
    qm(x)
    assert torch.equal(qm.running_list[0].cpu(), T(g["qm_run_pctl"]))
    qm.calculate_running = False
    qm.running_max = torch.tensor(qm.running_list, device=dev).mean()      # as noisynet.py:1258
    assert torch.equal(qm.eval()(x).cpu(), T(g["qm_fixed_y"]))
    w = T(g["qm_w_x"]).to(dev)
    qmw = hm.QuantMeasure(4, min_value=-1.0, max_value=1.0, pctl=99.0, calculate_running=True).to(dev).eval()
    assert torch.equal(qmw(w).cpu(), T(g["qm_w_y"]))
    assert torch.equal(qmw.running_max.cpu(), T(g["qm_w_max"]))
    assert qmw.calculate_running is False
    qq = q.QuantMeasure(4, pctl=0.99, calculate_running=True).to(dev).train()
    qq(x)
    assert torch.equal(qq.running_list[0].cpu(), T(g["qq_pctl"]))


@pytest.mark.parametrize("n,pctl", [(1000, 99.0), (65 * 14 * 14 * 64, 99.98), (3000 * 512 + 7, 90.0), (37, 50.0)])
def test_range_select_matches_kthvalue(dev, n, pctl):
    """SURVEY 8f.2: the device radix select is torch.kthvalue bit for bit (hardware_model.py:249, :233-235), and the max."""
    from noisynet_b200 import ops
    gen = torch.Generator().manual_seed(n)
    x = (torch.randn(n, generator=gen).abs() * 2).to(dev)
    x[::7] = 0.0                                            # ties and zeros, as after ReLU
    k = int(n * pctl / 100.)
    out = ops.range_select(x, mode=0, min_value=0.0, k_rank=k).cpu()
    ref, _ = torch.kthvalue(x.flatten().cpu(), k)
    assert out[0].item() == ref.item() and out[1].item() == x.max().item()
    assert out[2].item() == 0.0 and out[3].item() == x.max().item()
    w = torch.randn(n, generator=gen).to(dev) * 0.3
    o1 = ops.range_select(w, pctl, mode=1).cpu()
    wc = w.cpu()
    pos, neg = wc[wc > 0], wc[wc < 0].abs()
    rp, _ = torch.kthvalue(pos, int(pos.numel() * pctl / 100.))
    rn, _ = torch.kthvalue(neg, int(neg.numel() * pctl / 100.))
    assert o1[1].item() == rp.item() and o1[0].item() == -rn.item()
    assert o1[2].item() == -rn.item() and o1[3].item() == rp.item()


def test_quant_measure_calibration_has_no_host_sync(dev, golden):
    """While calibrating (noisynet.py:1251-1259) the reference syncs twice per QuantMeasure call (kthvalue result kept on
    the device, input.max().item()); the drop-in selects the range on the device and hands it to the quantizer kernels
    as a pointer: forward AND backward run under torch's sync-debug mode 'error'.  Output = the reference's (golden)."""
    from noisynet_b200 import hardware_model as hm, ops, quant as q
    g = golden("quant")
    x = T(g["qm_run_x"]).to(dev).requires_grad_(True)
    u = T(g["qm_run_u"]).to(dev)
    qm = hm.QuantMeasure(4, stochastic=0.5, pctl=99.0, calculate_running=True).to(dev).train()
    qq = q.QuantMeasure(4, pctl=0.99, calculate_running=True).to(dev).train()
    gy = torch.ones_like(x)
    qfix = hm.QuantMeasure(4, stochastic=0.0).to(dev).eval()          # running_max == 0, max_value == 0 -> live input.max()
    qfix(x.detach())                                                  # (reads the running_max buffer once; cached until it changes)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with ops.inject_random([u], []):
            y = qm(x)
        y.backward(gy)
        y2 = qq(x.detach())
        y3 = qfix(x.detach())
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(y.detach().cpu(), T(g["qm_run_y"]))
    assert torch.equal(qm.running_list[0].cpu(), T(g["qm_run_pctl"]))
    xc = x.detach().cpu()
    assert torch.equal(x.grad.cpu(), ((xc >= 0) & (xc <= xc.max())).float())
    assert torch.equal(qq.running_list[0].cpu(), T(g["qq_pctl"]))
    assert torch.equal(y3.cpu(), O.uniform_quantize_fwd(xc, 4, 0.0, xc.max().item(), 0.0))
    assert y2.shape == x.shape


# ------------------------------------------------------------------------------ a4 / a9 / stats
def test_weight_noise(dev, golden):
    from noisynet_b200 import ops
    g = golden("layers")
    y = ops.weight_noise(T(g["an_w"]).to(dev), 0.3, u=T(g["an_u"]).to(dev))
    assert torch.equal(y.cpu(), T(g["an_y"]))
    w = torch.randn(1001)
    y = ops.weight_noise(w.to(dev), 0.2, rng=ops._fixed_rng(5, 8))
    u = torch.from_numpy(O.philox_uniform_sym(1001, 5, 8, 0.2))
    assert torch.equal(y.cpu(), O.add_weight_noise(w, 0.2, u))


def test_clamp_and_stats(dev):
    from noisynet_b200 import ops
    w = torch.randn(195000 + 7) * 0.2
    wd = w.to(dev)
    amax = ops.clamp_absmax_(wd, 0.3)
    assert torch.equal(wd.cpu(), w.clamp(-0.3, 0.3)) and amax.item() == pytest.approx(0.3)
    amax = ops.clamp_absmax_(wd, 0.0)                      # w_max == 0: no clamp (noisynet.py:1534 guards)
    assert torch.equal(wd.cpu(), w.clamp(-0.3, 0.3))
    x = torch.relu(torch.randn(4, 9, 7, 7)) - 0.0
    x[0, 0, 0, 0] = -3.5
    s = ops.tensor_stats(x.to(dev)).cpu()
    assert s[0].item() == x.max().item() and s[1].item() == x.abs().max().item()
    assert s[2].item() == (x > 0).sum().item()


# ------------------------------------------------------------------------------ a5/a6/a7/a10 fp32 kernels
def _conv_modes(ci, cfg):
    return dict(bw=int(cfg[0]), nz=cfg[1], train=bool(cfg[2]), stride=int(cfg[3]), pad=int(cfg[4]), bias=bool(cfg[5]))


def test_noisy_conv2d_module_vs_reference_golden(dev, golden):
    """hardware_model.NoisyConv2d forward + backward against the reference's own outputs."""
    from noisynet_b200 import hardware_model as hm, ops
    g = golden("layers")
    for ci, cfg in enumerate(g["conv_cfgs"]):
        c = _conv_modes(ci, cfg)
        m = hm.NoisyConv2d(6, 10, 3, stride=c["stride"], padding=c["pad"], bias=c["bias"], num_bits=0,
                           num_bits_weight=c["bw"], noise=c["nz"], stochastic=0.5).to(dev)
        m.precision = "fp32"
        with torch.no_grad():
            m.weight.copy_(T(g[f"conv{ci}_w"]))
            if c["bias"]:
                m.bias.copy_(T(g[f"conv{ci}_b"]))
        m.train(c["train"])
        x = T(g[f"conv{ci}_x"]).to(dev).requires_grad_(True)
        stochastic_draw = (c["bw"] > 0 and c["train"]) or (c["nz"] > 0 and c["train"])
        if stochastic_draw:
            # replay the reference's uniform draw: compute the effective weight with the injected u
            u = T(g[f"conv{ci}_u"]).to(dev)
            if c["bw"] > 0:
                w_eff = ops.quantize_fwd(m.weight.detach(), c["bw"], -1.0, 1.0, 0.5, u=u)
                y = ops.ConvFn.apply(x, w_eff, m.bias, c["stride"], c["pad"], "fp32", m.weight, -1.0, 1.0)
            else:
                w_eff = ops.AddNoise.apply(m.weight, c["nz"], False, u)
                b_eff = ops.AddNoise.apply(m.bias, c["nz"], False, T(g[f"conv{ci}_ub"]).to(dev)) if c["bias"] else None
                y = ops.ConvFn.apply(x, w_eff, b_eff, c["stride"], c["pad"], "fp32")
        else:
            y = m(x)
        y.backward(T(g[f"conv{ci}_gy"]).to(dev))
        assert torch.allclose(y.cpu(), T(g[f"conv{ci}_y"]), rtol=1e-5, atol=2e-6), ci
        assert torch.allclose(x.grad.cpu(), T(g[f"conv{ci}_gx"]), rtol=1e-5, atol=2e-6), ci
        assert torch.allclose(m.weight.grad.cpu(), T(g[f"conv{ci}_gw"]), rtol=1e-5, atol=2e-5), ci
        if c["bias"]:
            assert torch.allclose(m.bias.grad.cpu(), T(g[f"conv{ci}_gb"]), rtol=1e-5, atol=2e-5), ci


def test_noisy_linear_module_vs_reference_golden(dev, golden):
    from noisynet_b200 import hardware_model as hm, ops
    g = golden("layers")
    for ci, cfg in enumerate(g["lin_cfgs"]):
        bw, nz, train, bias = int(cfg[0]), cfg[1], bool(cfg[2]), bool(cfg[3])
        m = hm.NoisyLinear(37, 11, bias=bias, num_bits=0, num_bits_weight=bw, noise=nz, stochastic=0.5).to(dev)
        m.precision = "fp32"
        with torch.no_grad():
            m.weight.copy_(T(g[f"lin{ci}_w"]))
            if bias:
                m.bias.copy_(T(g[f"lin{ci}_b"]))
        m.train(train)
        x = T(g[f"lin{ci}_x"]).to(dev).requires_grad_(True)
        draws = train and ((0 < bw < 8) or (not (0 < bw < 8) and nz > 0))
        if draws:
            u = T(g[f"lin{ci}_u"]).to(dev)
            x4 = x.view(x.shape[0], -1, 1, 1)
            if 0 < bw < 8:
                w_eff = ops.quantize_fwd(m.weight.detach(), bw, -1.0, 1.0, 0.5, u=u)
                y = ops.ConvFn.apply(x4, w_eff.view(11, 37, 1, 1), m.bias, 1, 0, "fp32", m.weight.view(11, 37, 1, 1), -1.0, 1.0)
            else:
                w_eff = ops.AddNoise.apply(m.weight, nz, False, u)
                b_eff = ops.AddNoise.apply(m.bias, nz, False, T(g[f"lin{ci}_ub"]).to(dev)) if bias else None
                y = ops.ConvFn.apply(x4, w_eff.view(11, 37, 1, 1), b_eff, 1, 0, "fp32")
            y = y.view(x.shape[0], -1)
        else:
            y = m(x)
        y.backward(T(g[f"lin{ci}_gy"]).to(dev))
        assert torch.allclose(y.cpu(), T(g[f"lin{ci}_y"]), rtol=1e-5, atol=2e-6), ci
        assert torch.allclose(x.grad.cpu(), T(g[f"lin{ci}_gx"]), rtol=1e-5, atol=1e-5), ci
        assert torch.allclose(m.weight.grad.cpu(), T(g[f"lin{ci}_gw"]), rtol=1e-5, atol=1e-5), ci


def test_conv_with_own_input_quantizer(dev, golden):
    """ResNet-style NoisyConv2d(num_bits=4, num_bits_weight=4) (hardware_model.py:337-343)."""
    from noisynet_b200 import ops
    g = golden("layers")
    x = T(g["cq_x"]).to(dev).requires_grad_(True)
    w = T(g["cq_w"]).to(dev).requires_grad_(True)
    xq = ops.UniformQuantize.apply(x, 4, 0.0, 2.0, 0.5, False, False, T(g["cq_ua"]).to(dev))
    wq = ops.quantize_fwd(w.detach(), 4, -1.0, 1.0, 0.5, u=T(g["cq_uw"]).to(dev))
    y = ops.ConvFn.apply(xq, wq, None, 1, 1, "fp32", w, -1.0, 1.0)
    y.backward(T(g["cq_gy"]).to(dev))
    assert torch.allclose(y.cpu(), T(g["cq_y"]), rtol=1e-5, atol=2e-6)
    assert torch.allclose(x.grad.cpu(), T(g["cq_gx"]), rtol=1e-5, atol=1e-5)
    assert torch.allclose(w.grad.cpu(), T(g["cq_gw"]), rtol=1e-5, atol=2e-5)


def _dummy_model():
    from types import SimpleNamespace
    return SimpleNamespace(training=True, power=[[] for _ in range(4)], nsr=[[] for _ in range(4)],
                           input_sparsity=[[] for _ in range(4)])


def test_current_noise_vs_reference_golden(dev, golden):
    """add_noise_calculate_power accurate model with the reference's own z (noise-only launch) and the
    single-launch fused kernel; stats (power, nsr, sparsity) as appended at hardware_model.py:86-88."""
    from noisynet_b200 import ops
    from noisynet_b200._lib import NOISE_EXTERNAL, NOISE_MERGED
    g = golden("noise")
    for ci, (kind, merged, cur) in enumerate(g["n_meta"]):
        x, w, y, z = (T(g[f"n{ci}_{k}"]).to(dev) for k in "xwyz")
        if kind == 1:
            x4, w4, y4, z4 = x.view(*x.shape, 1, 1), w.view(*w.shape, 1, 1), y.view(*y.shape, 1, 1), z.view(*z.shape, 1, 1)
        else:
            x4, w4, y4, z4 = x, w, y, z
        mode = NOISE_MERGED if merged else NOISE_EXTERNAL
        scale = ops.tensor_stats(w)[1:2] if merged else ops.tensor_stats(x)[0:1]
        stats = torch.tensor([0.0, 0.0, float("-inf")], device=dev)
        r = ops.noisy_conv_fwd(x4, None, w4, None, 1, 0, noise_mode=mode, current=cur, scale_dev=scale, z=z4,
                               stats=stats, precision="fp32", y_in=y4)
        ref = T(g[f"n{ci}_out"])
        assert torch.allclose(r["y_noisy"].cpu().view_as(ref), ref, rtol=1e-5, atol=2e-6), ci
        s = stats.tolist()
        xs = ops.tensor_stats(x).tolist()
        mean_sum = s[0] / x.shape[0]
        p = 1.2e-6 * cur * mean_sum / (xs[0] * scale.item()) if merged else 1.2e-6 * cur * mean_sum / xs[0]
        got = [p, s[1] / y.numel() / s[2], xs[2] / x.numel()]
        assert np.allclose(got, g[f"n{ci}_stats"], rtol=2e-4), (ci, got, g[f"n{ci}_stats"])
        # fused single launch: main + sigma^2 contraction + epilogue
        r2 = ops.noisy_conv_fwd(x4, w4, w4, None, 1, 0, noise_mode=mode, current=cur, scale_dev=scale, z=z4,
                                precision="fp32", want_sigma=True)
        assert torch.allclose(r2["y"].cpu().view_as(ref), T(g[f"n{ci}_y"]), rtol=1e-5, atol=2e-6), ci
        assert torch.allclose(r2["y_noisy"].cpu().view_as(ref), ref, rtol=1e-5, atol=3e-6), ci
        sig, *_ = O.noise_sigma(x.cpu(), w.cpu(), cur, "conv" if kind == 0 else "linear", bool(merged))
        assert torch.allclose(r2["sigma"].cpu().view_as(sig), sig, rtol=1e-5, atol=1e-6), ci


def test_add_noise_calculate_power_entry_point(dev, golden):
    """The drop-in function with the reference's signature (in-kernel Philox z): statistical check +
    exact consistency with the exported z; zero sigma gives exactly zero noise (SURVEY section 7)."""
    from noisynet_b200 import hardware_model as hm, ops
    from noisynet_b200._lib import NOISE_MERGED
    from noisynet_b200.net import default_args
    g = golden("noise")
    x, w, y = (T(g[f"n2_{k}"]).to(dev) for k in "xwy")
    model = _dummy_model()
    args = default_args(layer_currents=[10.0] * 4)
    torch.manual_seed(5)
    out = hm.add_noise_calculate_power(model, args, [], x, w, y, layer_type='conv', i=0, layer_num=0, merged_dac=True)
    ref_stats = g["n2_stats"]
    assert model.power[0][0] == pytest.approx(ref_stats[0], rel=1e-4)
    assert model.input_sparsity[0][0] == pytest.approx(ref_stats[2], rel=1e-6)
    assert model.nsr[0][0] == pytest.approx(ref_stats[1], rel=0.05)         # different z draw: statistical
    sig, *_ = O.noise_sigma(x.cpu(), w.cpu(), 10.0, "conv", True)
    zhat = ((out - y).cpu() / sig)
    zhat = zhat[sig > 1e-6]
    assert abs(zhat.mean().item()) < 0.02 and abs(zhat.std().item() - 1.0) < 0.02
    # reproducible under torch.manual_seed, different between consecutive calls
    torch.manual_seed(5)
    out2 = hm.add_noise_calculate_power(model, args, [], x, w, y, layer_type='conv', i=99, layer_num=0, merged_dac=True)
    out3 = hm.add_noise_calculate_power(model, args, [], x, w, y, layer_type='conv', i=99, layer_num=0, merged_dac=True)
    assert torch.equal(out, out2) and not torch.equal(out2, out3)
    assert len(model.power[0]) == 1                                          # i >= 20: no stats appended
    # sigma == 0 (all-zero patches from zero-padded crops) -> exactly zero noise
    xz = torch.zeros_like(x)
    yz = torch.zeros_like(y)
    outz = hm.add_noise_calculate_power(model, args, [], xz, w, yz, layer_type='conv', i=99, layer_num=0, merged_dac=True)
    assert torch.count_nonzero(outz).item() == 0
    # gradient is identity w.r.t. output
    yg = y.clone().requires_grad_(True)
    o = hm.add_noise_calculate_power(model, args, [], x, w, yg, layer_type='conv', i=99, layer_num=0, merged_dac=True)
    o.backward(torch.ones_like(o))
    assert torch.equal(yg.grad, torch.ones_like(yg))


def test_philox_normal_epilogue_matches_spec(dev):
    """z exported by the fused kernel == numpy Philox/Box-Muller restatement (mapping (m, n) -> group)."""
    from noisynet_b200 import ops
    from noisynet_b200._lib import NOISE_MERGED
    x = torch.rand(3, 4, 9, 9)
    w = torch.randn(13, 4, 3, 3) * 0.2
    xd, wd = x.to(dev), w.to(dev)
    scale = ops.tensor_stats(wd)[1:2]
    r = ops.noisy_conv_fwd(xd, wd, wd, None, 1, 0, noise_mode=NOISE_MERGED, current=2.0, scale_dev=scale,
                           want_z=True, want_sigma=True, precision="fp32", rng=ops._fixed_rng(4242, 17))
    z = r["z"].cpu()                                        # [B, N, OH, OW]
    B, N, OH, OW = z.shape
    zs = torch.from_numpy(O.philox_normal_mn(B * OH * OW, N, 4242, 17)).view(B, OH, OW, N).permute(0, 3, 1, 2)
    assert (z - zs).abs().max().item() < 2e-3 and (z - zs).abs().mean().item() < 5e-6    # MUFU approximations
    assert torch.allclose(r["y_noisy"].cpu(), r["y"].cpu() + z * r["sigma"].cpu(), rtol=0, atol=1e-6)
    # distribution of a large draw
    xb = torch.rand(64, 3, 32, 32, device=dev)
    wb = torch.randn(65, 3, 5, 5, device=dev) * 0.1
    rb = ops.noisy_conv_fwd(xb, wb, wb, None, 1, 0, noise_mode=NOISE_MERGED, current=1.0,
                            scale_dev=ops.tensor_stats(wb)[1:2], want_z=True, precision="fp32")
    zb = rb["z"].flatten()
    assert abs(zb.mean().item()) < 2e-3 and abs(zb.std().item() - 1) < 2e-3
    assert abs((zb ** 3).mean().item()) < 1e-2 and abs((zb ** 4).mean().item() - 3) < 3e-2
    # independent across channels / pixels: lag correlations ~ 0
    zc = rb["z"]
    assert abs((zc[:, 0] * zc[:, 1]).mean().item()) < 2e-2        # 50k samples: sigma = 4.5e-3
    assert abs((zc[:, :, :, :-1] * zc[:, :, :, 1:]).mean().item()) < 3e-3   # 3.1M samples: sigma = 5.6e-4


def test_alt_noise_models(dev, golden):
    from noisynet_b200 import ops
    g = golden("noise")
    for kind in ("uniform_ind", "uniform_dep", "normal_ind", "normal_dep"):
        y = T(g[f"alt_{kind}_y"]).to(dev)
        out = ops.alt_noise(y, kind, 0.2, rnd=T(g[f"alt_{kind}_rnd"]).to(dev))
        assert torch.allclose(out.cpu(), T(g[f"alt_{kind}"]), rtol=1e-5, atol=2e-6), kind


def test_fp32_conv_geometries_vs_oracle(dev):
    """Strided / padded / ragged shapes incl. sizes that do not divide the tiles, NoisyNet's own
    layer shapes and ResNet-18 style 3x3 / 1x1-s2 / 7x7-s2 convs (SURVEY section 8a)."""
    from noisynet_b200 import ops
    gen = torch.Generator().manual_seed(11)
    cases = [(2, 3, 32, 32, 65, 5, 1, 0), (2, 65, 14, 14, 120, 5, 1, 0), (5, 3000, 1, 1, 390, 1, 1, 0),
             (7, 390, 1, 1, 10, 1, 1, 0), (1, 1, 5, 5, 1, 5, 1, 0), (2, 16, 15, 15, 24, 3, 1, 1),
             (2, 16, 14, 14, 32, 1, 2, 0), (1, 3, 33, 33, 16, 7, 2, 3), (3, 5, 9, 11, 7, 3, 2, 1)]
    for (B, Cin, H, W, Cout, k, s, p) in cases:
        x = torch.randn(B, Cin, H, W, generator=gen)
        w = torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5
        y = F.conv2d(x, w, None, s, p)
        gy = torch.randn(y.shape, generator=gen)
        xd, wd, gyd = x.to(dev), w.to(dev), gy.to(dev)
        r = ops.noisy_conv_fwd(xd, wd, None, None, s, p, precision="fp32")
        assert torch.allclose(r["y"].cpu(), y, rtol=1e-4, atol=1e-5), (B, Cin, H, W, Cout, k, s, p)
        gx = ops.conv_dgrad(gyd, wd, x.shape, s, p, precision="fp32").cpu()
        gw = ops.conv_wgrad(gyd, xd, w.shape, s, p, precision="fp32").cpu()
        assert torch.allclose(gx, torch.nn.grad.conv2d_input(x.shape, w, gy, s, p), rtol=1e-4, atol=1e-5)
        ref_gw = torch.nn.grad.conv2d_weight(x, w.shape, gy, s, p)
        assert torch.allclose(gw, ref_gw, rtol=1e-4, atol=1e-4 * ref_gw.abs().max().item())


def test_linearity_and_determinism_at_full_size(dev):
    """BASELINE config-2 sizes (batch 512): size-independent properties instead of a CPU oracle run."""
    from noisynet_b200 import ops
    from noisynet_b200._lib import NOISE_EXTERNAL
    B = 512
    x1 = torch.rand(B, 65, 14, 14, device=dev)
    x2 = torch.rand(B, 65, 14, 14, device=dev)
    w = torch.randn(120, 65, 5, 5, device=dev) * 0.05
    y1 = ops.noisy_conv_fwd(x1, w, precision="fp32")["y"]
    y2 = ops.noisy_conv_fwd(x2, w, precision="fp32")["y"]
    y12 = ops.noisy_conv_fwd(x1 + x2, w, precision="fp32")["y"]
    assert torch.allclose(y12, y1 + y2, rtol=1e-4, atol=1e-4)
    # per-sample independence: a batch slice equals the same samples run alone
    ys = ops.noisy_conv_fwd(x1[100:104].contiguous(), w, precision="fp32")["y"]
    assert torch.equal(ys, y1[100:104])
    # deterministic wgrad (fixed-order split reduction)
    gy = torch.randn_like(y1)
    g1 = ops.conv_wgrad(gy, x1, w.shape, precision="fp32")
    g2 = ops.conv_wgrad(gy, x1, w.shape, precision="fp32")
    assert torch.equal(g1, g2)
    # <gy, conv(x, w)> == <dgrad(gy), x> == <wgrad(gy, x), w>   (adjoint identities)
    a = (gy * y1).sum().item()
    b = (ops.conv_dgrad(gy, w, x1.shape, precision="fp32") * x1).sum().item()
    c = (g1 * w).sum().item()
    assert abs(a - b) < 2e-3 * abs(a) + 1e-2 and abs(a - c) < 2e-3 * abs(a) + 1e-2
    # sigma^2 >= 0 and noise scales like 1/sqrt(I)
    sc = ops.tensor_stats(x1)[0:1]
    r1 = ops.noisy_conv_fwd(x1, w, w, None, noise_mode=NOISE_EXTERNAL, current=1.0, scale_dev=sc, want_sigma=True,
                            precision="fp32")
    r4 = ops.noisy_conv_fwd(x1, w, w, None, noise_mode=NOISE_EXTERNAL, current=4.0, scale_dev=sc, want_sigma=True,
                            precision="fp32")
    assert (r1["sigma"] >= 0).all() and torch.allclose(r1["sigma"], 2.0 * r4["sigma"], rtol=1e-5, atol=1e-7)


def test_distort_tensor_semantics(dev):
    """hardware_model.distort_tensor (reference hardware_model.py:426-458, called by the ImageNet models' forward,
    models/resnet.py:40-55): fixed Gaussian offsets drawn once per tensor slot (--offset), or a fresh uniform
    multiplicative distortion x * (1 + U(-noise, noise)) per call."""
    from types import SimpleNamespace
    from noisynet_b200 import hardware_model as hm
    torch.manual_seed(0)
    x = torch.randn(8, 16, 12, 12, device=dev)
    owner = SimpleNamespace(generate_offsets=True)
    args = SimpleNamespace(offset=0.1, offset_input=0.0, noise=0.0, debug=False)
    y1 = hm.distort_tensor(owner, args, x, scale=0.1)
    assert torch.equal(y1 - x, owner.act1_offsets) or torch.allclose(y1 - x, owner.act1_offsets, atol=1e-6)
    assert owner.act1_offsets.std().item() == pytest.approx(0.1, rel=0.1) and owner.generate_offsets
    y2 = hm.distort_tensor(owner, args, x * 2, scale=0.1, stop=True)            # last layer: offsets are frozen afterwards
    assert not owner.generate_offsets and torch.allclose(y2 - 2 * x, owner.act2_offsets, atol=1e-6)
    frozen = owner.act1_offsets.clone()
    y3 = hm.distort_tensor(owner, args, x, scale=0.1)
    assert torch.equal(owner.act1_offsets, frozen) and torch.allclose(y3, x + frozen, atol=1e-6)
    # multiplicative distortion (nn_alt_noise kind "distort_act"): |y / x - 1| <= noise, fresh per call, mean ~ 0
    args = SimpleNamespace(offset=0.0, offset_input=0.0, noise=0.05, debug=False)
    ya, yb = hm.distort_tensor(owner, args, x), hm.distort_tensor(owner, args, x)
    r = ya / x - 1.0
    assert r.abs().max().item() <= 0.05 + 1e-5 and abs(r.mean().item()) < 2e-3
    assert r.std().item() == pytest.approx(0.05 / 3 ** 0.5, rel=0.05)
    assert not torch.equal(ya, yb)
