"""The CIFAR NoisyNet of noisynet.py:326-695 built on the boundary modules.

``noisynet.Net`` lives inside a script whose module level runs the whole training, so it cannot be
imported; this class restates its forward (default flags: batchnorm on, no merge_bn, no plot/write)
with identical sub-module names / state_dict keys, calling exactly the operator API the script calls
(NoisyConv2d -> add_noise_calculate_power -> pool -> bn -> relu -> clamp -> QuantMeasure).

``fused=True`` replaces each (layer, add_noise_calculate_power) pair by ONE launch of the fused
noisy-conv kernel (main + sigma^2 contraction + Philox noise epilogue) -- same maths, one pass over x.
"""
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from ._lib import NOISE_EXTERNAL, NOISE_MERGED
from .hardware_model import (NoisyConv2d, NoisyLinear, QuantMeasure, _prepare_weight, _scalar_stats_buffer,
                             add_noise_calculate_power, code_scales)


def default_args(**over):
    """README flags (README.md:6-9) over the argparse defaults (noisynet.py:20-312)."""
    a = SimpleNamespace(
        fm1=65, fm2=120, fc=390, fs=5, width=1, use_bias=False, stochastic=0.5, pctl=99.98,
        q_a1=0, q_a2=0, q_a3=0, q_a4=0, q_w1=0, q_w2=0, q_w3=0, q_w4=0,
        n_w1=0.0, n_w2=0.0, n_w3=0.0, n_w4=0.0, n_w_test=0.0,
        act_max=5.0, act_max1=5.0, act_max2=5.0, act_max3=5.0, dropout=0.0, dropout_conv=0.0,
        w_max1=0.3, w_max2=0.0, w_max3=0.0, w_max4=0.0,
        current1=1.0, current2=1.0, current3=1.0, current4=1.0, layer_currents=[1.0, 1.0, 1.0, 1.0],
        merged_dac=True, batchnorm=True, bn3=True, bn4=True, track_running_stats=True,
        LR=0.005, L2_1=0.0005, L2_2=0.0002, L2_3=0.0, L2_4=0.0, L2_bn=0.0, amsgrad=False,
        distort_act=False, uniform_ind=0, uniform_dep=0, normal_ind=0, normal_dep=0, noise_test=False,
        noise=0, plot=False, write=False, debug_quant=False, debug_noise=False)
    for k, v in over.items():
        setattr(a, k, v)
    return a


def with_quant(args, q_a=4, q_w=4):
    """--q_a / --q_w broadcast (noisynet.py:861-862, 898-900)."""
    args.q_a1 = args.q_a2 = args.q_a3 = args.q_a4 = q_a
    args.q_w1 = args.q_w2 = args.q_w3 = args.q_w4 = q_w
    return args


class NoisyNet(nn.Module):
    def __init__(self, args, fused=False, precision=None):
        super().__init__()
        a = self.args = args
        self.fused = fused
        self.precision = precision
        self.pool = nn.MaxPool2d(2, 2)
        self.relu = nn.ReLU()
        self.quantize1 = QuantMeasure(a.q_a1, stochastic=a.stochastic, pctl=a.pctl, max_value=1.0, debug=a.debug_quant)
        self.quantize2 = QuantMeasure(a.q_a2, stochastic=a.stochastic, pctl=a.pctl, debug=a.debug_quant)
        self.quantize3 = QuantMeasure(a.q_a3, stochastic=a.stochastic, pctl=a.pctl,
                                      max_value=a.act_max / (1. - a.dropout), debug=a.debug_quant)
        self.quantize4 = QuantMeasure(a.q_a4, stochastic=a.stochastic, pctl=a.pctl, debug=a.debug_quant)
        self.conv1 = NoisyConv2d(3, a.fm1 * a.width, kernel_size=a.fs, bias=a.use_bias, num_bits=0,
                                 num_bits_weight=a.q_w1, noise=a.n_w1, test_noise=a.n_w_test,
                                 stochastic=a.stochastic, debug=a.debug_noise)
        self.conv2 = NoisyConv2d(a.fm1 * a.width, a.fm2 * a.width, kernel_size=a.fs, bias=a.use_bias, num_bits=0,
                                 num_bits_weight=a.q_w2, noise=a.n_w2, test_noise=a.n_w_test,
                                 stochastic=a.stochastic, debug=a.debug_noise)
        self.linear1 = NoisyLinear(a.fm2 * a.width * a.fs * a.fs, a.fc * a.width, bias=a.use_bias, num_bits=0,
                                   num_bits_weight=a.q_w3, noise=a.n_w3, test_noise=a.n_w_test,
                                   stochastic=a.stochastic, debug=a.debug_noise)
        self.linear2 = NoisyLinear(a.fc * a.width, 10, bias=a.use_bias, num_bits=0, num_bits_weight=a.q_w4,
                                   noise=a.n_w4, test_noise=a.n_w_test, stochastic=a.stochastic, debug=a.debug_noise)
        self.bn1 = nn.BatchNorm2d(a.fm1 * a.width, track_running_stats=a.track_running_stats)
        self.bn2 = nn.BatchNorm2d(a.fm2 * a.width, track_running_stats=a.track_running_stats)
        self.bn3 = nn.BatchNorm1d(a.fc * a.width, track_running_stats=a.track_running_stats)
        self.bn4 = nn.BatchNorm1d(10, track_running_stats=a.track_running_stats)
        if a.dropout > 0 or a.dropout_conv > 0:     # noisynet.py:375-376 (the script creates it for --dropout only and then
            self.dropout = nn.Dropout(p=a.dropout)   # fails on --dropout_conv alone; here p = --dropout in both cases)
        for m in (self.conv1, self.conv2, self.linear1, self.linear2):
            m.precision = precision
        self.power = [[] for _ in range(4)]
        self.nsr = [[] for _ in range(4)]
        self.input_sparsity = [[] for _ in range(4)]
        self.collect_stats = True      # False: never sync for the i < 20 side statistics (benchmark loops)
        self.w_absmax = {}             # layer index -> (param version, device scalar max|W|) from clamp_weights_()
        self._absmax_buf = None

    # --- one noisy layer -------------------------------------------------------------------------
    def _layer(self, x, mod, idx, kind, merged, i):
        a = self.args
        cur = a.layer_currents[idx]
        if not self.fused or cur <= 0 or a.distort_act:
            y = mod(x)                                                         # noisynet.py:398 / 462 / 522 / 571
            setattr(self, ("conv%d_" if kind == "conv" else "linear%d_") % (idx % 2 + 1), y)
            if cur > 0 or a.distort_act:                                       # noisynet.py:414-417
                return add_noise_calculate_power(self, a, [], x, mod.weight, y, layer_type=kind,
                                                 i=i if self.collect_stats else 10 ** 9, layer_num=idx,
                                                 merged_dac=merged)
            return y
        # ---- fused: one launch
        weight, bias, ste = _prepare_weight(mod, linear=(kind == "linear"))
        a_cs, w_cs = code_scales(x, weight)          # exact integer operands on the tensor-core path
        w_raw = mod.weight.detach()
        if kind == "linear":
            x4 = x.reshape(x.shape[0], -1, 1, 1)
            weight = weight.view(weight.shape[0], weight.shape[1], 1, 1)
            w_raw4 = w_raw.view(w_raw.shape[0], w_raw.shape[1], 1, 1)
        else:
            x4, w_raw4 = x, w_raw
        want_stats = self.collect_stats and i < 20
        xs = None
        if merged:
            hit = self.w_absmax.get(idx)               # (param version, device scalar) from clamp_weights_()
            scale_dev = hit[1] if (hit is not None and hit[0] == mod.weight._version) else \
                ops.tensor_stats(w_raw)[1:2]
        else:
            xs = ops.tensor_stats(x4.detach())
            scale_dev = xs[0:1]
        stats = _scalar_stats_buffer(x.device) if want_stats else None
        mode = NOISE_MERGED if merged else NOISE_EXTERNAL
        if ste is None:
            y, yn = ops.FusedNoisyConvFn.apply(x4, weight, bias, w_raw4, 1, 0, mode, float(cur), scale_dev, stats,
                                               None, self.precision, None, 0.0, 0.0, a_cs, w_cs)
        else:
            raw, lo, hi = ste
            raw4 = raw.view(raw.shape[0], raw.shape[1], 1, 1) if kind == "linear" else raw
            y, yn = ops.FusedNoisyConvFn.apply(x4, weight, bias, w_raw4, 1, 0, mode, float(cur), scale_dev, stats,
                                               None, self.precision, raw4, lo, hi, a_cs, w_cs)
        if kind == "linear":
            y, yn = y.view(y.shape[0], -1), yn.view(yn.shape[0], -1)
        if want_stats:
            if xs is None:
                xs = ops.tensor_stats(x4.detach())
            s, xl = stats.tolist(), xs.tolist()
            mean_sum = s[0] / x4.shape[0]
            if merged:
                p = 1.0e-6 * 1.2 * cur * mean_sum / (xl[0] * scale_dev.item())
            else:
                p = 1.0e-6 * 1.2 * cur * mean_sum / xl[0]
            self.power[idx].append(p)
            self.nsr[idx].append(s[1] / y.numel() / s[2])
            self.input_sparsity[idx].append(xl[2] / x4.numel())
        return yn

    def forward(self, input, epoch=0, i=0, s=0, acc=0.0):
        a = self.args
        x = self.quantize1(input) if a.q_a1 > 0 else input                     # noisynet.py:390-393
        h = self._layer(x, self.conv1, 0, "conv", a.merged_dac, i)             # :398-417
        h = self.bn1(self.pool(h))                                             # :419-422
        h = self.relu(h)                                                       # :430
        if a.act_max1 > 0:
            h = torch.clamp(h, max=a.act_max1)                                 # :438
        if a.dropout_conv > 0:
            h = self.dropout(h)                                                # :456-457
        if a.q_a2 > 0:
            h = self.quantize2(h)                                              # :460
        h = self._layer(h, self.conv2, 1, "conv", False, i)                    # :462-481
        h = self.relu(self.bn2(self.pool(h)))
        if a.act_max2 > 0:
            h = torch.clamp(h, max=a.act_max2)
        if a.dropout > 0:
            h = self.dropout(h)                                                # :512-513
        h = h.view(h.size(0), -1)                                              # :515
        if a.q_a3 > 0:
            h = self.quantize3(h)                                              # :520
        h = self._layer(h, self.linear1, 2, "linear", a.merged_dac, i)         # :522-538
        h = self.relu(self.bn3(h))
        if a.act_max3 > 0:
            h = torch.clamp(h, max=a.act_max3)
        if a.dropout > 0:
            h = self.dropout(h)                                                # :565-566
        if a.q_a4 > 0:
            h = self.quantize4(h)                                              # :569
        h = self._layer(h, self.linear2, 3, "linear", False, i)                # :571-591
        return self.bn4(h)                                                     # :594

    # --- noisynet.py:1527-1542 -----------------------------------------------------------------------
    def clamp_weights_(self):
        a = self.args
        for idx, (mod, wmax) in enumerate(((self.conv1, a.w_max1), (self.conv2, a.w_max2),
                                           (self.linear1, a.w_max3), (self.linear2, a.w_max4))):
            if self._absmax_buf is None or self._absmax_buf.device != mod.weight.device:
                self._absmax_buf = torch.zeros(4, dtype=torch.float32, device=mod.weight.device)
            amax = self._absmax_buf[idx:idx + 1]      # persistent storage: stable address under CUDA-graph replay
            ops.clamp_absmax_(mod.weight.data, wmax, out=amax)
            self.w_absmax[idx] = (mod.weight._version, amax)


def init_like_reference(model):
    """utils.py:203-216 then utils.py:244-299 with weight_init='default' (conv: N(0, sqrt(2/n)),
    linear: kaiming_normal fan_in drawn twice)."""
    import math
    for m in (model.conv1, model.conv2):
        n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
        m.weight.data.normal_(0, math.sqrt(2. / n))
    for m in (model.linear1, model.linear2):
        nn.init.kaiming_normal_(m.weight, mode='fan_in', nonlinearity='relu')
        nn.init.kaiming_normal_(m.weight, mode='fan_in', nonlinearity='relu')
    return model


def make_optimizer(model, args, fused=None, capturable=False):
    """noisynet.py:1135-1169."""
    a = args
    groups = [
        {'params': model.conv1.parameters(), 'weight_decay': a.L2_1, 'lr': a.LR},
        {'params': model.conv2.parameters(), 'weight_decay': a.L2_2, 'lr': a.LR},
        {'params': model.linear1.parameters(), 'weight_decay': a.L2_3, 'lr': a.LR},
        {'params': model.linear2.parameters(), 'weight_decay': a.L2_4, 'lr': a.LR},
        {'params': model.bn1.parameters(), 'weight_decay': a.L2_bn},
        {'params': model.bn2.parameters(), 'weight_decay': a.L2_bn},
        {'params': model.bn3.parameters(), 'weight_decay': a.L2_bn},
        {'params': model.bn4.parameters(), 'weight_decay': a.L2_bn}]
    kw = {}
    if fused is not None:
        kw["fused"] = fused
    if capturable:
        kw["capturable"] = True
    return torch.optim.AdamW(groups, lr=a.LR, amsgrad=a.amsgrad, **kw)


def train_step(model, opt, x, label, i=0):
    """noisynet.py:1276-1278, 1346, 1372, 1520, 1527-1542."""
    out = model(x, 0, i)
    loss = F.cross_entropy(out, label)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
    model.clamp_weights_()
    return loss.detach(), out.detach()


def make_fused_optimizer(model, args, grad_scale=1.0):
    """Same groups as noisynet.py:1135-1169, on the fused AdamW + clamp kernel; the per-layer clamp bounds
    (noisynet.py:1527-1542) ride along in the groups."""
    from .optim import FusedAdamW
    a = args
    groups = [
        {'params': model.conv1.parameters(), 'weight_decay': a.L2_1, 'lr': a.LR, 'clamp': a.w_max1},
        {'params': model.conv2.parameters(), 'weight_decay': a.L2_2, 'lr': a.LR, 'clamp': a.w_max2},
        {'params': model.linear1.parameters(), 'weight_decay': a.L2_3, 'lr': a.LR, 'clamp': a.w_max3},
        {'params': model.linear2.parameters(), 'weight_decay': a.L2_4, 'lr': a.LR, 'clamp': a.w_max4},
        {'params': list(model.bn1.parameters()) + list(model.bn2.parameters()) + list(model.bn3.parameters())
                   + list(model.bn4.parameters()), 'weight_decay': a.L2_bn, 'lr': a.LR}]
    return FusedAdamW(groups, lr=a.LR, weight_decay=0.0, grad_scale=grad_scale)


def bind_absmax(model, opt):
    """After the first fused step: the next forwards read max|W| from the optimizer's device scalars."""
    for idx, mod in enumerate((model.conv1, model.conv2, model.linear1, model.linear2)):
        model.w_absmax[idx] = (mod.weight._version, opt.absmax_of(mod.weight))


def train_step_fused(model, opt, x, label, i=0):
    """train_step with optimizer.step() + weight clamp + max|W| in one launch (FusedAdamW)."""
    out = model(x, 0, i)
    loss = F.cross_entropy(out, label)
    opt.zero_grad()
    loss.backward()
    opt.step()
    bind_absmax(model, opt)
    return loss.detach(), out.detach()
