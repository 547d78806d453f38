"""CPU restatement (torch-CPU fp32 + numpy) of the NoisyNet hot path.

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.  Every function cites
the reference lines (michaelklachko/NoisyNet, commit 34b7996) it restates.  The
arithmetic of the reference lives in PyTorch (ATen, fp32); this file therefore
uses torch CPU fp32 ops for the contractions and restates everything the
reference writes itself (quantizer, STE, weight noise, current noise, side
statistics, op order of the CIFAR net, weight clamp) line by line.

Random numbers: the reference draws from torch's global generator.  Every
function here takes the random tensor (``u`` / ``z``) as an explicit optional
argument so that (a) the reference can be matched with the same draws and
(b) the CUDA kernels can be matched through their z/u export/inject modes.
``philox_*`` below restates the generator the CUDA kernels use (Philox4x32-10 +
Box-Muller, documented in DESIGN.md) -- that part is a spec of OUR kernels, not
of the reference.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------
# a1/a2  UniformQuantize            hardware_model.py:133-183 (= quant.py:12-61)
# --------------------------------------------------------------------------

def quant_scale(num_bits, min_value, max_value):
    """hardware_model.py:148-151: scale = max((max-min)/(2^b-1), 1e-6) in Python doubles."""
    qmax = 2.0 ** num_bits - 1.0
    scale = (float(max_value) - float(min_value)) / (qmax - 0.0)
    return max(scale, 1e-6), qmax


def uniform_quantize_fwd(x, num_bits, min_value, max_value, stochastic=0.0, u=None):
    """hardware_model.py:153-170.

    y = round_half_even(clamp((x - min)/scale + U(-st, st), 0, 2^b-1)) * scale + min,
    every step a separate fp32 rounding (add_, div_, add_, clamp_, round_, mul_, add_).
    ``u`` is the tensor the reference would have drawn at :161 (already in [-st, st)).
    """
    scale, qmax = quant_scale(num_bits, min_value, max_value)
    out = x.detach().clone().float()
    out.add_(-float(min_value)).div_(scale).add_(0.0)
    if stochastic > 0:
        if u is None:
            u = out.new_empty(out.shape).uniform_(-stochastic, stochastic)
        out.add_(u)
    out.clamp_(0.0, qmax).round_()
    out.add_(-0.0).mul_(scale).add_(float(min_value))
    return out


def uniform_quantize_codes(x, num_bits, min_value, max_value, stochastic=0.0, u=None):
    """Integer codes k (before the dequantize step :170) -- used by the bit-exact tests."""
    scale, qmax = quant_scale(num_bits, min_value, max_value)
    out = x.detach().clone().float()
    out.add_(-float(min_value)).div_(scale)
    if stochastic > 0 and u is not None:
        out.add_(u)
    return out.clamp_(0.0, qmax).round_()


def uniform_quantize_bwd(x, grad_output, min_value, max_value):
    """hardware_model.py:176-183 saturated STE: g * 1[min <= x <= max].

    The reference zeroes ``grad_output`` in place; we return a new tensor (SURVEY §7:
    our op must not mutate its incoming grad)."""
    g = grad_output.clone()
    g[x > max_value] = 0
    g[x < min_value] = 0
    return g


# --------------------------------------------------------------------------
# a3  QuantMeasure range selection  hardware_model.py:227-288 / quant.py:99-137
# --------------------------------------------------------------------------

def kth_percentile(t, pctl_percent):
    """hardware_model.py:249: torch.kthvalue(flat, int(numel * pctl / 100))."""
    flat = t.detach().flatten()
    k = int(flat.numel() * pctl_percent / 100.0)
    return torch.kthvalue(flat, k)[0]


def weight_percentile_range(w, pctl_percent):
    """hardware_model.py:232-239: one-shot +-percentile for signed weights."""
    pos = w[w > 0].flatten()
    neg = torch.abs(w[w < 0]).flatten()
    p = torch.kthvalue(pos, int(pos.numel() * pctl_percent / 100.0))[0]
    n = torch.kthvalue(neg, int(neg.numel() * pctl_percent / 100.0))[0]
    return -n, p


# --------------------------------------------------------------------------
# a4  AddNoise                      hardware_model.py:291-307
# --------------------------------------------------------------------------

def add_weight_noise(w, noise, u=None):
    """w + w * U(-n, n); backward is identity (STE)."""
    out = w.detach().clone()
    if u is None:
        u = out.new_empty(out.shape).uniform_(-noise, noise)
    out.add_(out * u)
    return out


# --------------------------------------------------------------------------
# a5/a6  NoisyConv2d / NoisyLinear forward     hardware_model.py:328-366, 386-423
# --------------------------------------------------------------------------

def effective_weight(w, num_bits_weight=0, noise=0.0, test_noise=0.0, training=True,
                     stochastic=0.5, u=None, w_min=-1.0, w_max=1.0, linear=False):
    """Branch order of hardware_model.py:343-360 (conv) / :402-420 (linear)."""
    quant_on = (0 < num_bits_weight < 8) if linear else (num_bits_weight > 0)
    if quant_on:
        st = stochastic if training else 0.0           # :283-286
        return uniform_quantize_fwd(w, num_bits_weight, w_min, w_max, st, u)
    if test_noise > 0 and not training:
        return add_weight_noise(w, test_noise, u)
    if noise > 0 and training:
        return add_weight_noise(w, noise, u)
    return w.detach().clone()


def noisy_conv2d_fwd(x, w_eff, bias=None, stride=1, padding=0, dilation=1, groups=1):
    """hardware_model.py:362."""
    return F.conv2d(x, w_eff, bias, stride, padding, dilation, groups)


def noisy_linear_fwd(x, w_eff, bias=None):
    """hardware_model.py:421."""
    return F.linear(x, w_eff, bias)


# --------------------------------------------------------------------------
# a7  add_noise_calculate_power, accurate model   hardware_model.py:43-88, 122-127
# --------------------------------------------------------------------------

def noise_sigma(x, w_raw, current, layer_type="conv", merged_dac=True, stride=1, padding=0, want_plain=True):
    """Returns (sigma, S_plain, x_max, w_max).

    merged DAC  (:47-59):  S = conv(x,|W|),        sigma = sqrt(0.1 * (max|W| / I) * S)
    external DAC(:61-81):  S = conv(x,|W|^2+|W|),  sigma = sqrt(0.1 * (max(x) / I) * S)
    The reference calls F.conv2d with default stride/padding (:49, :65); NoisyNet's
    convs are stride 1 / pad 0 so this is the layer geometry.  ``stride``/``padding``
    generalise to the layer's own geometry (needed for S to have Y's shape).
    """
    absw = torch.abs(w_raw)
    x_max = torch.max(x)
    w_max = torch.max(absw)
    if layer_type == "conv":
        contract = lambda k: F.conv2d(x, k, None, stride, padding)
    else:
        contract = lambda k: F.linear(x, k, None)
    # the external-DAC branch needs conv(x,|W|) only for the i < 20 power statistic (:67-68, :74-75)
    s_plain = contract(absw) if (merged_dac or want_plain) else None
    if merged_dac:
        sig = torch.sqrt(0.1 * (w_max / current) * s_plain)
    else:
        s_sq = contract(absw.pow(2) + absw)
        sig = torch.sqrt(0.1 * (x_max / current) * s_sq)
    return sig, s_plain, x_max, w_max


def add_noise_calculate_power(x, w_raw, y, current, layer_type="conv", merged_dac=True,
                              z=None, want_stats=True, stride=1, padding=0):
    """Accurate-model branch.  Returns (y_noisy, stats) with stats = dict(power, nsr, sparsity)
    as appended at hardware_model.py:86-88 when i < 20."""
    with torch.no_grad():
        sig, s_plain, x_max, w_max = noise_sigma(x, w_raw, current, layer_type, merged_dac,
                                                 stride, padding, want_plain=want_stats)
        if z is None:
            z = torch.randn_like(sig)
        noise = z * sig                       # torch.normal(0, sig) == normal_(0,1) * sig
        stats = None
        if want_stats:
            dim = (1, 2, 3) if layer_type == "conv" else 1
            sample_sums = torch.sum(s_plain, dim=dim)
            if merged_dac:                    # :57
                p = 1.0e-6 * 1.2 * current * torch.mean(sample_sums) / (x_max * w_max)
            else:                             # :79
                p = 1.0e-6 * 1.2 * current * torch.mean(sample_sums) / x_max
            stats = dict(power=p.item(),
                         nsr=torch.mean(torch.abs(noise) / torch.max(y)).item(),
                         sparsity=x[x > 0].numel() / x.numel())
    return y + noise, stats


def alt_noise(y, kind, level, rnd):
    """Alternative output-noise models hardware_model.py:24-41 (+ :122-125).
    ``rnd`` is U[0,1) for the uniform models and N(0,1) for the normal ones."""
    with torch.no_grad():
        if kind == "uniform_ind":
            s = level * torch.max(torch.abs(y))
            return y + (rnd * 2 - 1) * s
        if kind == "uniform_dep":            # multiplicative, U(level, 1/level)
            return y * (level + rnd * (1.0 / level - level))
        if kind == "normal_ind":
            return y + rnd * (level * torch.max(torch.abs(y)))
        if kind == "normal_dep":
            return y + rnd * (level * y)
        if kind == "distort_act":            # :17-20, U(-n, n) multiplicative offset
            return y + y * ((rnd * 2 - 1) * level)
    raise ValueError(kind)


# --------------------------------------------------------------------------
# a8/a9 clamps          noisynet.py:434-441, 1527-1542
# --------------------------------------------------------------------------

def act_clamp(x, act_max):
    return torch.clamp(x, max=act_max) if act_max > 0 else x


def weight_clamp_(w, w_max):
    if w_max > 0:
        w.data.clamp_(-w_max, w_max)
    return w


# --------------------------------------------------------------------------
# The CIFAR net (noisynet.py:326-695) as a functional forward, and one
# training step (noisynet.py:1249-1542).  Used for whole-step parity and as
# the CPU arm of the benchmark.
# --------------------------------------------------------------------------

def default_args(**over):
    """README flags (README.md:6-9) + argparse defaults (noisynet.py:20-312)."""
    a = SimpleNamespace(
        fm1=65, fm2=120, fc=390, fs=5, width=1, use_bias=False,
        current=1.0, act_max=5.0, w_max1=0.3, w_max2=0.0, w_max3=0.0, w_max4=0.0,
        LR=0.005, L2_1=0.0005, L2_2=0.0002, L2_3=0.0, L2_4=0.0, L2_bn=0.0,
        q_a=0, q_w=0, stochastic=0.5, pctl=99.98, n_w=0.0, n_w_test=0.0,
        dropout=0.0, dropout_conv=0.0, batchnorm=True, bn3=True, bn4=True,
        merged_dac=True, amsgrad=False, track_running_stats=True,
        quant_max2=0.0, quant_max4=0.0)   # running_max of quantize2/4 after calibration
    for k, v in over.items():
        setattr(a, k, v)
    return a


class OracleNet(torch.nn.Module):
    """Parameters/buffers named exactly as noisynet.Net's state_dict (conv1.weight, bn1.*, ...)."""

    def __init__(self, args):
        super().__init__()
        a = args
        nn = torch.nn
        self.args = a
        self.conv1 = nn.Conv2d(3, a.fm1 * a.width, a.fs, bias=a.use_bias)
        self.conv2 = nn.Conv2d(a.fm1 * a.width, a.fm2 * a.width, a.fs, bias=a.use_bias)
        self.linear1 = nn.Linear(a.fm2 * a.width * a.fs * a.fs, a.fc * a.width, bias=a.use_bias)
        self.linear2 = nn.Linear(a.fc * a.width, 10, bias=a.use_bias)
        self.bn1 = nn.BatchNorm2d(a.fm1 * a.width)
        self.bn2 = nn.BatchNorm2d(a.fm2 * a.width)
        self.bn3 = nn.BatchNorm1d(a.fc * a.width)
        self.bn4 = nn.BatchNorm1d(10)
        self.power = [[] for _ in range(4)]
        self.nsr = [[] for _ in range(4)]
        self.input_sparsity = [[] for _ in range(4)]

    def init_like_reference(self):
        """utils.py:203-216 (weights_init) then utils.py:244-299 (init_model, weight_init='default')."""
        a = self.args
        for m in (self.conv1, self.conv2):
            n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
            m.weight.data.normal_(0, math.sqrt(2.0 / n))
        for m in (self.linear1, self.linear2):
            torch.nn.init.kaiming_normal_(m.weight, mode="fan_in", nonlinearity="relu")
            torch.nn.init.kaiming_normal_(m.weight, mode="fan_in", nonlinearity="relu")
        return self

    class _STEQuant(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, bits, lo, hi, st, u):
            ctx.save_for_backward(x)
            ctx.lo, ctx.hi = lo, hi
            return uniform_quantize_fwd(x, bits, lo, hi, st, u)

        @staticmethod
        def backward(ctx, g):
            (x,) = ctx.saved_tensors
            return uniform_quantize_bwd(x, g, ctx.lo, ctx.hi), None, None, None, None, None

    def _q(self, x, bits, lo, hi, rnd, name):
        st = self.args.stochastic if self.training else 0.0
        u = None
        if rnd is not None and st > 0:
            u = rnd.get(name)
        return OracleNet._STEQuant.apply(x, bits, lo, hi, st, u)

    def _layer(self, x, mod, idx, kind, merged, i, rnd):
        a = self.args
        w = mod.weight
        if a.q_w > 0:
            w_eff = self._q(w, a.q_w, -1.0, 1.0, rnd, f"uw{idx}")          # hardware_model.py:343
        elif a.n_w > 0 and self.training:
            un = rnd.get(f"uw{idx}") if rnd is not None else None
            w_eff = w + (add_weight_noise(w, a.n_w, un) - w).detach()       # STE identity :303-307
        else:
            w_eff = w
        y = F.conv2d(x, w_eff) if kind == "conv" else F.linear(x, w_eff)    # :362 / :421
        if a.current > 0:
            z = rnd.get(f"z{idx}") if rnd is not None else None
            out, st = add_noise_calculate_power(x.detach(), w.detach(), y, a.current, kind, merged,
                                                z=z, want_stats=(i < 20))
            if st is not None:
                self.power[idx].append(st["power"])
                self.nsr[idx].append(st["nsr"])
                self.input_sparsity[idx].append(st["sparsity"])
            return out
        return y

    def forward(self, x, i=0, rnd=None):
        """noisynet.py:378-594 with default flags (batchnorm, no merge_bn, no dropout)."""
        a = self.args
        if a.q_a > 0:
            x = self._q(x, a.q_a, 0.0, 1.0, rnd, "ua1")                      # quantize1 :344, 390
        c1 = self._layer(x, self.conv1, 0, "conv", a.merged_dac, i, rnd)     # :398-415
        h = F.max_pool2d(c1, 2, 2)                                           # :419
        h = self.bn1(h)                                                      # :422
        h = act_clamp(F.relu(h), a.act_max)                                  # :430-438
        if a.q_a > 0:
            h = self._q(h, a.q_a, 0.0, a.quant_max2 if a.quant_max2 > 0 else float(h.max()),
                        rnd, "ua2")                                          # quantize2 :345, 460
        c2 = self._layer(h, self.conv2, 1, "conv", False, i, rnd)            # :462-479
        h = F.max_pool2d(c2, 2, 2)
        h = self.bn2(h)
        h = act_clamp(F.relu(h), a.act_max)
        h = h.view(h.size(0), -1)                                            # :515
        if a.q_a > 0:
            h = self._q(h, a.q_a, 0.0, a.act_max / (1.0 - a.dropout), rnd, "ua3")   # quantize3 :346
        l1 = self._layer(h, self.linear1, 2, "linear", a.merged_dac, i, rnd)       # :522-536
        h = self.bn3(l1)
        h = act_clamp(F.relu(h), a.act_max)
        if a.q_a > 0:
            h = self._q(h, a.q_a, 0.0, a.quant_max4 if a.quant_max4 > 0 else float(h.max()),
                        rnd, "ua4")
        l2 = self._layer(h, self.linear2, 3, "linear", False, i, rnd)        # :571-589
        return self.bn4(l2)                                                  # :594


def make_optimizer(model, args):
    """noisynet.py:1135-1169: AdamW, per-layer lr / weight decay groups."""
    a = args
    groups = [
        {"params": model.conv1.parameters(), "weight_decay": a.L2_1, "lr": a.LR},
        {"params": model.conv2.parameters(), "weight_decay": a.L2_2, "lr": a.LR},
        {"params": model.linear1.parameters(), "weight_decay": a.L2_3, "lr": a.LR},
        {"params": model.linear2.parameters(), "weight_decay": a.L2_4, "lr": a.LR},
        {"params": model.bn1.parameters(), "weight_decay": a.L2_bn},
        {"params": model.bn2.parameters(), "weight_decay": a.L2_bn},
        {"params": model.bn3.parameters(), "weight_decay": a.L2_bn},
        {"params": model.bn4.parameters(), "weight_decay": a.L2_bn},
    ]
    return torch.optim.AdamW(groups, lr=a.LR, amsgrad=a.amsgrad)


def train_step(model, opt, x, label, i=0, rnd=None):
    """noisynet.py:1276-1278, 1346, 1372, 1520, 1527-1542."""
    a = model.args
    out = model(x, i=i, rnd=rnd)
    loss = F.cross_entropy(out, label)
    opt.zero_grad()
    loss.backward()
    opt.step()
    weight_clamp_(model.conv1.weight, a.w_max1)
    weight_clamp_(model.conv2.weight, a.w_max2)
    weight_clamp_(model.linear1.weight, a.w_max3)
    weight_clamp_(model.linear2.weight, a.w_max4)
    return loss.detach(), out.detach()


def synthetic_cifar(n, seed=0):
    """SURVEY §8d / BASELINE.md §3: 4-bit CIFAR-shaped inputs in {0..15}/15, labels 0..9."""
    rng = np.random.default_rng(seed)
    x = (rng.integers(0, 16, (n, 3, 32, 32)).astype(np.float32) / 15.0).astype(np.float32)
    y = rng.integers(0, 10, n).astype(np.int64)
    return torch.from_numpy(x), torch.from_numpy(y)


# --------------------------------------------------------------------------
# Spec of the CUDA kernels' generator (NOT a restatement of the reference):
# Philox4x32-10, key = seed, counter = (offset_lo, offset_hi, group_lo, group_hi).
# --------------------------------------------------------------------------

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(group, seed, offset):
    """group: uint64 array of group indices.  Returns uint32 array [..., 4]."""
    group = np.asarray(group, dtype=np.uint64)
    c0 = np.full_like(group, np.uint64(offset) & _MASK)
    c1 = np.full_like(group, (np.uint64(offset) >> np.uint64(32)) & _MASK)
    c2 = group & _MASK
    c3 = (group >> np.uint64(32)) & _MASK
    k0 = np.uint64(seed) & _MASK
    k1 = (np.uint64(seed) >> np.uint64(32)) & _MASK
    for _ in range(10):
        p0 = _M0 * c0
        p1 = _M1 * c2
        hi0, lo0 = (p0 >> np.uint64(32)) & _MASK, p0 & _MASK
        hi1, lo1 = (p1 >> np.uint64(32)) & _MASK, p1 & _MASK
        c0, c1, c2, c3 = (hi1 ^ c1 ^ k0) & _MASK, lo1, (hi0 ^ c3 ^ k1) & _MASK, lo0
        k0 = (k0 + _W0) & _MASK
        k1 = (k1 + _W1) & _MASK
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def philox_uniform01(r):
    """u = (r >> 8) * 2^-24 in [0, 1)  (exact in fp32)."""
    return ((r >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)).astype(np.float32)


def philox_uniform_sym(n, seed, offset, s):
    """Per-element U[-s, s): element i uses group i//4, word i%4; v = fl(fl(u*2s) - s)."""
    groups = np.arange((n + 3) // 4, dtype=np.uint64)
    r = philox4x32_10(groups, seed, offset).reshape(-1)[:n]
    u = philox_uniform01(r)
    two_s = np.float32(np.float32(2.0) * np.float32(s))
    return (u * two_s).astype(np.float32) - np.float32(s)


def philox_normal_groups(groups, seed, offset):
    """Box-Muller on (r0,r1) and (r2,r3): u1 = fma(r, 2^-32, 2^-33) in (0,1], theta = fma(u2, 2pi, -pi) with
    u2 = (r>>8)*2^-24; z_even = rad*cos(theta), z_odd = rad*sin(theta), rad = sqrt(-2 ln u1).
    The kernels evaluate log2 / sqrt / sin / cos with the MUFU approximations (abs error ~1e-6 typical);
    this restatement evaluates them exactly.  Returns float32 [..., 4]."""
    r = philox4x32_10(groups, seed, offset)
    out = np.empty(r.shape, dtype=np.float32)
    for j in (0, 2):
        ra, rb = r[..., j], r[..., j + 1]
        u1 = (ra.astype(np.float32).astype(np.float64) * 2.0 ** -32 + 2.0 ** -33).astype(np.float32)
        u2 = philox_uniform01(rb)
        rad = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
        th = (u2.astype(np.float64) * float(np.float32(6.2831853071795865)) + float(np.float32(-3.14159265358979324))).astype(np.float32)
        out[..., j] = (rad * np.cos(th.astype(np.float64))).astype(np.float32)
        out[..., j + 1] = (rad * np.sin(th.astype(np.float64))).astype(np.float32)
    return out


def philox_normal_flat(n, seed, offset):
    """Element i -> group i//4, word i%4 (elementwise kernels)."""
    groups = np.arange((n + 3) // 4, dtype=np.uint64)
    return philox_normal_groups(groups, seed, offset).reshape(-1)[:n]


def philox_normal_mn(M, N, seed, offset):
    """Conv/linear epilogue mapping: element (m, n) -> group m*ceil(N/4) + n//4, word n%4.
    Returns [M, N] float32 (m = (b*OH + oh)*OW + ow for conv, n = output channel)."""
    ng = (N + 3) // 4
    groups = (np.arange(M, dtype=np.uint64)[:, None] * np.uint64(ng)
              + np.arange(ng, dtype=np.uint64)[None, :])
    z = philox_normal_groups(groups, seed, offset)          # [M, ng, 4]
    return z.reshape(M, ng * 4)[:, :N]
