"""Mint golden fixtures by running the UNMODIFIED reference modules (CPU, shimmed).

Needs a checkout of the reference (michaelklachko/NoisyNet) named by NOISYNET_REFERENCE:
    NOISYNET_REFERENCE=<checkout> python -m oracle.gen_golden
Writes small .npz files under tests/golden/.  The tests read only those fixtures, never the
reference itself.  Every case stores the inputs, the random tensors the reference consumed
(recovered by re-seeding the generator) and the reference's outputs.
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def net_args(**over):
    """The argparse namespace fields noisynet.Net and add_noise_calculate_power read
    (noisynet.py:20-312 defaults + README flags)."""
    a = SimpleNamespace(
        train_act_max=False, train_w_max=False, q_a1=0, q_a2=0, q_a3=0, q_a4=0, stochastic=0.5,
        pctl=99.98, debug_quant=False, act_max=5.0, dropout=0.0, fm1=65, fm2=120, fc=390, fs=5,
        width=1, use_bias=False, q_w1=0, q_w2=0, q_w3=0, q_w4=0, n_w1=0, n_w2=0, n_w3=0, n_w4=0,
        n_w_test=0, debug_noise=False, batchnorm=True, track_running_stats=True, bn3=True, bn4=True,
        weightnorm=False, plot=False, write=False, merge_bn=False,
        current1=1.0, current2=1.0, current3=1.0, current4=1.0, distort_act=False, merged_dac=True,
        act_max1=5.0, act_max2=5.0, act_max3=5.0, L3_act=0, dropout_conv=0, resume=None,
        uniform_ind=0, uniform_dep=0, normal_ind=0, normal_dep=0, noise_test=False,
        layer_currents=[1.0, 1.0, 1.0, 1.0], plot_noise=False, plot_power=False, noise=0,
        debug=False, plot_basic=False, block_size=None)
    for k, v in over.items():
        setattr(a, k, v)
    return a


def t2n(d):
    return {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v))
            for k, v in d.items()}


def gen_quant(hm, q):
    out = {}
    x = torch.tensor([-0.2, 0, 0.1, 0.5, 1 / 6, 2.4, 2.5, 2.6, 5.0, 5.1, 7.0])
    for name, mod in (("hm", hm), ("q", q)):
        xi = x.clone().requires_grad_(True)
        y = mod.UniformQuantize().apply(xi, 4, 0.0, 5.0, 0, False, False)
        g = torch.arange(1.0, 12.0)
        y.backward(g.clone())
        out[f"kat_{name}_x"], out[f"kat_{name}_y"], out[f"kat_{name}_g"] = x, y, xi.grad
    # weight quantizer on [-1,1], eval
    w = torch.tensor([-1.3, -1, -0.95, -0.5, -0.07, 0, 0.06, 0.07, 0.3, 0.93, 1, 1.2])
    qm = hm.QuantMeasure(4, min_value=-1.0, max_value=1.0).eval()
    wi = w.clone().requires_grad_(True)
    yw = qm(wi)
    yw.backward(torch.ones_like(w))
    out["wq_x"], out["wq_y"], out["wq_g"] = w, yw, wi.grad
    # scale floor (max == min)
    xf = torch.tensor([0.0, 1e-6, 1.0])
    out["floor_x"] = xf
    out["floor_y"] = hm.UniformQuantize().apply(xf.clone(), 4, 0.0, 0.0, 0, False, False)
    # random tensors, several (bits, range), deterministic and stochastic
    g = torch.Generator().manual_seed(1234)
    cases = []
    for ci, (bits, lo, hi, st, shape) in enumerate([
            (4, 0.0, 1.0, 0.0, (4, 3, 8, 8)), (4, 0.0, 5.0, 0.5, (4, 7, 6, 6)),
            (2, 0.0, 3.0, 0.5, (5, 33)), (8, -1.0, 1.0, 0.5, (6, 3, 5, 5)),
            (4, -1.0, 1.0, 0.5, (65, 3, 5, 5)), (6, -0.37, 0.91, 0.25, (1000,)),
            (1, 0.0, 1.0, 0.5, (3, 50))]):
        xr = (torch.randn(shape, generator=g) * (hi - lo) * 0.7 + (hi + lo) / 2).float()
        torch.manual_seed(100 + ci)
        xi = xr.clone().requires_grad_(True)
        y = hm.UniformQuantize().apply(xi, bits, lo, hi, st, False, False)
        gr = torch.randn(shape, generator=g)
        y.backward(gr.clone())
        torch.manual_seed(100 + ci)
        u = xr.new(xr.shape).uniform_(-st, st) if st > 0 else torch.zeros_like(xr)
        out[f"r{ci}_x"], out[f"r{ci}_u"], out[f"r{ci}_y"] = xr, u, y
        out[f"r{ci}_gout"], out[f"r{ci}_gin"] = gr, xi.grad
        cases.append([bits, lo, hi, st])
    out["r_params"] = np.asarray(cases, dtype=np.float64)
    # QuantMeasure range selection
    xa = torch.rand(4, 8, 6, 6, generator=g) * 3.0
    qm = hm.QuantMeasure(4, stochastic=0.5, pctl=99.0, calculate_running=True)
    qm.train()
    torch.manual_seed(7)
    ya = qm(xa)
    out["qm_run_x"], out["qm_run_y"] = xa, ya
    out["qm_run_pctl"] = qm.running_list[0]
    torch.manual_seed(7)
    out["qm_run_u"] = xa.new(xa.shape).uniform_(-0.5, 0.5)
    qm.calculate_running = False
    qm.running_max = torch.tensor(qm.running_list).mean()
    qm.eval()
    out["qm_fixed_y"] = qm(xa)
    wq = torch.randn(20, 9, 5, 5, generator=g) * 0.05
    qmw = hm.QuantMeasure(4, min_value=-1.0, max_value=1.0, pctl=99.0, calculate_running=True).eval()
    out["qm_w_x"], out["qm_w_y"] = wq, qmw(wq)
    out["qm_w_min"], out["qm_w_max"] = qmw.running_min, qmw.running_max
    qq = q.QuantMeasure(4, pctl=0.99, calculate_running=True)
    qq.train()
    torch.manual_seed(9)
    out["qq_y"] = qq(xa)
    out["qq_pctl"] = qq.running_list[0]
    torch.manual_seed(9)
    out["qq_u"] = xa.new(xa.shape).uniform_(-0.5, 0.5)
    np.savez_compressed(os.path.join(OUT, "quant.npz"), **t2n(out))
    print("quant.npz", len(out), "arrays")


def gen_layers(hm):
    out = {}
    g = torch.Generator().manual_seed(4321)
    # --- AddNoise
    w = torch.randn(5, 3, 3, 3, generator=g)
    torch.manual_seed(11)
    out["an_w"], out["an_y"] = w, hm.AddNoise().apply(w.clone(), 0.3, False)
    torch.manual_seed(11)
    out["an_u"] = w.new_empty(w.shape).uniform_(-0.3, 0.3)
    # --- NoisyConv2d: variants (bits_w, noise, training, stride, padding, bias)
    cfgs = [(0, 0.0, True, 1, 0, False), (4, 0.0, True, 1, 0, False), (4, 0.0, False, 1, 0, False),
            (0, 0.2, True, 1, 0, True), (4, 0.0, True, 2, 1, False), (0, 0.0, True, 1, 2, True)]
    out["conv_cfgs"] = np.asarray([[c[0], c[1], int(c[2]), c[3], c[4], int(c[5])] for c in cfgs], dtype=np.float64)
    for ci, (bw, nz, train, stride, pad, bias) in enumerate(cfgs):
        torch.manual_seed(50 + ci)
        m = hm.NoisyConv2d(6, 10, 3, stride=stride, padding=pad, bias=bias, num_bits=0,
                           num_bits_weight=bw, noise=nz, stochastic=0.5)
        with torch.no_grad():
            m.weight.mul_(2.0)
            if bias:
                m.bias.normal_(0, 0.1)
        m.train(train)
        x = torch.rand(3, 6, 9, 9, generator=g).requires_grad_(True)
        torch.manual_seed(500 + ci)
        y = m(x)
        gy = torch.randn(y.shape, generator=g)
        y.backward(gy)
        torch.manual_seed(500 + ci)
        if bw > 0 and train:
            u = m.weight.new(m.weight.shape).uniform_(-0.5, 0.5)
        elif nz > 0 and train:
            u = m.weight.new_empty(m.weight.shape).uniform_(-nz, nz)
            out[f"conv{ci}_ub"] = m.bias.new_empty(m.bias.shape).uniform_(-nz, nz)
        else:
            u = torch.zeros_like(m.weight)
        out[f"conv{ci}_x"], out[f"conv{ci}_w"], out[f"conv{ci}_u"] = x, m.weight, u
        if bias:
            out[f"conv{ci}_b"], out[f"conv{ci}_gb"] = m.bias, m.bias.grad
        out[f"conv{ci}_y"], out[f"conv{ci}_gy"] = y, gy
        out[f"conv{ci}_gx"], out[f"conv{ci}_gw"] = x.grad, m.weight.grad
    # --- NoisyConv2d with its own input quantizer (ResNet style, hardware_model.py:337-340)
    torch.manual_seed(77)
    m = hm.NoisyConv2d(4, 8, 3, padding=1, num_bits=4, num_bits_weight=4, stochastic=0.5)
    m.quantize_input.max_value = 2.0
    with torch.no_grad():
        m.weight.mul_(3.0)
    m.train()
    x = (torch.rand(2, 4, 7, 7, generator=g) * 2.5 - 0.2).requires_grad_(True)
    torch.manual_seed(770)
    y = m(x)
    gy = torch.randn(y.shape, generator=g)
    y.backward(gy)
    torch.manual_seed(770)
    out["cq_ua"] = x.new(x.shape).uniform_(-0.5, 0.5)
    out["cq_uw"] = m.weight.new(m.weight.shape).uniform_(-0.5, 0.5)
    out["cq_x"], out["cq_w"], out["cq_y"], out["cq_gy"] = x, m.weight, y, gy
    out["cq_gx"], out["cq_gw"] = x.grad, m.weight.grad
    # --- NoisyLinear
    lcfgs = [(0, 0.0, True, False), (4, 0.0, True, False), (4, 0.0, False, True), (0, 0.1, True, True),
             (8, 0.0, True, False)]
    out["lin_cfgs"] = np.asarray([[c[0], c[1], int(c[2]), int(c[3])] for c in lcfgs], dtype=np.float64)
    for ci, (bw, nz, train, bias) in enumerate(lcfgs):
        torch.manual_seed(60 + ci)
        m = hm.NoisyLinear(37, 11, bias=bias, num_bits=0, num_bits_weight=bw, noise=nz, stochastic=0.5)
        with torch.no_grad():
            m.weight.mul_(3.0)
        m.train(train)
        x = torch.rand(5, 37, generator=g).requires_grad_(True)
        torch.manual_seed(600 + ci)
        y = m(x)
        gy = torch.randn(y.shape, generator=g)
        y.backward(gy)
        torch.manual_seed(600 + ci)
        if 0 < bw < 8 and train:
            u = m.weight.new(m.weight.shape).uniform_(-0.5, 0.5)
        elif not (0 < bw < 8) and nz > 0 and train:
            u = m.weight.new_empty(m.weight.shape).uniform_(-nz, nz)
            if bias:
                out[f"lin{ci}_ub"] = m.bias.new_empty(m.bias.shape).uniform_(-nz, nz)
        else:
            u = torch.zeros_like(m.weight)
        out[f"lin{ci}_x"], out[f"lin{ci}_w"], out[f"lin{ci}_u"] = x, m.weight, u
        if bias:
            out[f"lin{ci}_b"] = m.bias
        out[f"lin{ci}_y"], out[f"lin{ci}_gy"] = y, gy
        out[f"lin{ci}_gx"], out[f"lin{ci}_gw"] = x.grad, m.weight.grad
    np.savez_compressed(os.path.join(OUT, "layers.npz"), **t2n(out))
    print("layers.npz", len(out), "arrays")


def gen_noise(hm):
    out = {}
    g = torch.Generator().manual_seed(999)
    model = SimpleNamespace(training=True, power=[[] for _ in range(4)], nsr=[[] for _ in range(4)],
                            input_sparsity=[[] for _ in range(4)])
    cases = [("conv", True, 1.0, (4, 3, 12, 12), (9, 3, 5, 5)),
             ("conv", False, 1.0, (4, 9, 8, 8), (12, 9, 5, 5)),
             ("conv", True, 10.0, (2, 3, 20, 20), (17, 3, 5, 5)),
             ("linear", True, 1.0, (6, 50), (20, 50)),
             ("linear", False, 3.0, (6, 20), (10, 20))]
    meta = []
    for ci, (kind, merged, cur, xs, ws) in enumerate(cases):
        x = torch.randint(0, 16, xs, generator=g).float() / 15.0
        if ci == 1:  # post-ReLU style input with zeros
            x = torch.relu(torch.randn(xs, generator=g)) * 1.5
        w = torch.randn(ws, generator=g) * 0.1
        y = torch.nn.functional.conv2d(x, w) if kind == "conv" else torch.nn.functional.linear(x, w)
        args = net_args(layer_currents=[cur] * 4)
        torch.manual_seed(900 + ci)
        yn = hm.add_noise_calculate_power(model, args, [], x, w, y, layer_type=kind, i=0,
                                          layer_num=ci % 4, merged_dac=merged)
        torch.manual_seed(900 + ci)
        z = torch.empty_like(y).normal_(0, 1)
        out[f"n{ci}_x"], out[f"n{ci}_w"], out[f"n{ci}_y"], out[f"n{ci}_z"], out[f"n{ci}_out"] = x, w, y, z, yn
        out[f"n{ci}_stats"] = np.asarray([model.power[ci % 4][-1], model.nsr[ci % 4][-1],
                                          model.input_sparsity[ci % 4][-1]])
        meta.append([0 if kind == "conv" else 1, int(merged), cur])
    out["n_meta"] = np.asarray(meta, dtype=np.float64)
    # alternative noise models (hardware_model.py:24-41) and distort_act (:17-20 needs torch.cuda -> skip)
    y = torch.randn(3, 5, 4, 4, generator=g)
    for kind in ("uniform_ind", "uniform_dep", "normal_ind", "normal_dep"):
        args = net_args(**{kind: 0.2})
        yk = y.abs() if kind == "normal_dep" else y   # torch.normal rejects the negative std of :39
        out[f"alt_{kind}_y"] = yk
        torch.manual_seed(42)
        out[f"alt_{kind}"] = hm.add_noise_calculate_power(model, args, [], yk, yk, yk)
        torch.manual_seed(42)
        if kind.startswith("uniform"):
            out[f"alt_{kind}_rnd"] = torch.rand(y.shape)
        else:
            out[f"alt_{kind}_rnd"] = torch.empty_like(y).normal_(0, 1)
    np.savez_compressed(os.path.join(OUT, "noise.npz"), **t2n(out))
    print("noise.npz", len(out), "arrays")


def gen_net():
    """One training step of the real noisynet.Net (class body executed from the reference file)
    on a tiny batch, README flags, with and without 4-bit quantization."""
    from oracle import noisynet_oracle as O
    out = {}
    for tag, q in (("fp", 0), ("q4", 4)):
        args = net_args(q_a1=q, q_a2=q, q_a3=q, q_a4=q, q_w1=q, q_w2=q, q_w3=q, q_w4=q,
                        fm1=9, fm2=12, fc=24)   # narrow net keeps the fixture small
        Net = ref_shims.load_reference_net_class(args)
        torch.manual_seed(2024)
        model = Net(args)
        if q:
            model.quantize2.running_max = torch.tensor(4.0)
            model.quantize4.running_max = torch.tensor(4.5)
        model.power = [[] for _ in range(4)]
        model.nsr = [[] for _ in range(4)]
        model.input_sparsity = [[] for _ in range(4)]
        x, lab = O.synthetic_cifar(8, seed=3)
        sd0 = {k: v.clone() for k, v in model.state_dict().items()}
        oa = O.default_args(q_a=q, q_w=q, quant_max2=4.0, quant_max4=4.5, fm1=9, fm2=12, fc=24)
        opt = O.make_optimizer(model, oa)
        model.train()
        torch.manual_seed(31337)
        logits = model(x, 0, 0, 1, 10.0)
        loss = torch.nn.CrossEntropyLoss()(logits, lab)
        opt.zero_grad()
        loss.backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        opt.step()
        model.conv1.weight.data.clamp_(-0.3, 0.3)
        for k, v in sd0.items():
            out[f"{tag}_sd0_{k}"] = v
        for k, v in grads.items():
            out[f"{tag}_grad_{k}"] = v
        for k, v in model.state_dict().items():
            out[f"{tag}_sd1_{k}"] = v
        out[f"{tag}_x"], out[f"{tag}_label"], out[f"{tag}_logits"], out[f"{tag}_loss"] = x, lab, logits, loss
        out[f"{tag}_power"] = np.asarray([p[0] for p in model.power])
        out[f"{tag}_nsr"] = np.asarray([p[0] for p in model.nsr])
        out[f"{tag}_sparsity"] = np.asarray([p[0] for p in model.input_sparsity])
    np.savez_compressed(os.path.join(OUT, "net_step.npz"), **t2n(out))
    print("net_step.npz", len(out), "arrays")


def main():
    os.makedirs(OUT, exist_ok=True)
    hm, q = ref_shims.import_reference_ops()
    gen_quant(hm, q)
    gen_layers(hm)
    gen_noise(hm)
    gen_net()


if __name__ == "__main__":
    main()
