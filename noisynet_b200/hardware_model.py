"""Drop-in replacement for the reference's ``hardware_model`` module (hardware_model.py).

Same names, signatures, state_dict keys and error behaviour; every arithmetic op runs in the
sm_90a kernels behind the C ABI (include/noisynet_b200.h).  Put ``<repo>/dropin`` ahead of the
reference on ``sys.path`` and ``noisynet.py`` / ``models/resnet.py`` / ``main.py`` import this
instead (noisynet.py:14, models/resnet.py:11, main.py:37).

Reference lines are cited as hm:<line> (hardware_model.py) below.
"""
import torch
import torch.nn as nn

from . import ops
from ._lib import NOISE_EXTERNAL, NOISE_MERGED
from .ops import AddNoise, UniformQuantize  # noqa: F401  (re-exported names, hm:130, hm:291)

__all__ = ["add_noise_calculate_power", "UniformQuantize", "QuantMeasure", "AddNoise", "NoisyConv2d",
           "NoisyLinear", "distort_tensor"]


def _scalar_stats_buffer(device):
    return torch.tensor([0.0, 0.0, float("-inf")], dtype=torch.float32, device=device)


def _layer_geometry(input, weights, output, layer_type):
    """The reference contracts with default stride/padding (hm:49, hm:65); S must have the shape of
    ``output``, so the layer's own stride/padding are recovered from the shapes when they differ."""
    if layer_type == "linear":
        x2 = input.reshape(-1, input.shape[-1])
        return x2.view(x2.shape[0], x2.shape[1], 1, 1), weights.view(weights.shape[0], weights.shape[1], 1, 1), 1, 0
    kh = weights.shape[2]
    H, OH = input.shape[2], output.shape[2]
    for stride in (1, 2, 3, 4):
        for pad in range(0, kh):
            if (H + 2 * pad - kh) // stride + 1 == OH and (input.shape[3] + 2 * pad - weights.shape[3]) // stride + 1 == output.shape[3]:
                return input, weights, stride, pad
    raise ValueError("add_noise_calculate_power: cannot infer conv geometry from shapes %s %s %s"
                     % (tuple(input.shape), tuple(weights.shape), tuple(output.shape)))


def add_noise_calculate_power(self, args, arrays, input, weights, output, layer_type='conv', i=0, layer_num=0,
                              merged_dac=True):
    """hm:16-127.  ``self`` is the model (reads .training, appends to .power/.nsr/.input_sparsity)."""
    if args.distort_act:                                                       # hm:17-20
        return ops.StraightThrough.apply(output, ops.alt_noise(output.detach(), "distort_act", args.noise))

    training = self.training
    for kind in ("uniform_ind", "uniform_dep", "normal_ind", "normal_dep"):   # hm:24-41, first match wins
        level = getattr(args, kind, 0)
        if level > 0 and (training or args.noise_test):
            if kind == "uniform_dep":                                          # multiplicative (hm:122-123)
                return output * ops.alt_noise(torch.ones_like(output), kind, level)
            return ops.StraightThrough.apply(output, ops.alt_noise(output.detach(), kind, level))

    if args.plot or args.write:
        raise NotImplementedError("noisynet_b200: --plot/--write diagnostics (plot_histograms.py) are out of scope")

    current = float(args.layer_currents[layer_num])
    x = input.detach()
    w = weights.detach()
    x4, w4, stride, pad = _layer_geometry(x, w, output, layer_type)
    want_stats = i < 20                                                        # hm:54, hm:85
    mode = NOISE_MERGED if merged_dac else NOISE_EXTERNAL
    xs = None
    if merged_dac:
        scale_dev = ops.tensor_stats(w)[1:2]                                   # w_max = max|W|    (hm:47)
    else:
        xs = ops.tensor_stats(x)
        scale_dev = xs[0:1]                                                    # input_max         (hm:45)
    stats = _scalar_stats_buffer(output.device) if want_stats else None
    y4 = output if layer_type == "conv" else output.reshape(x4.shape[0], -1, 1, 1)
    noisy = ops.CurrentNoiseFn.apply(y4, x4, w4, stride, pad, mode, current, scale_dev, stats, None, None)
    noisy = noisy.view_as(output)

    if want_stats:                                                             # hm:55-57, 77-79, 85-88 (host sync,
        if xs is None:                                                         #  as the reference's .item() calls)
            xs = ops.tensor_stats(x)
        ws = ops.tensor_stats(w) if not merged_dac else None
        s = stats.tolist()
        xl = xs.tolist()
        batch = x4.shape[0]
        mean_sum = s[0] / batch
        if merged_dac:
            w_max = scale_dev.item()
            p = 1.0e-6 * 1.2 * current * mean_sum / (xl[0] * w_max)
        else:
            p = 1.0e-6 * 1.2 * current * mean_sum / xl[0]
        del ws
        self.power[layer_num].append(p)
        self.nsr[layer_num].append(s[1] / output.numel() / s[2])
        self.input_sparsity[layer_num].append(xl[2] / x.numel())
    return noisy


class QuantMeasure(nn.Module):
    """hm:186-288 -- range selection for the uniform quantizer; buffers ``running_min`` [1] and
    ``running_max`` [] keep the reference's state_dict keys."""

    def __init__(self, num_bits=8, momentum=0.0, stochastic=0.5, min_value=0., max_value=0., scale=1,
                 calculate_running=False, pctl=90., debug=False, inplace=False):
        super(QuantMeasure, self).__init__()
        self.register_buffer('running_min', torch.zeros(1))
        self.register_buffer('running_max', torch.zeros([]))
        self.momentum = momentum
        self.num_bits = num_bits
        self.stochastic = stochastic
        self.inplace = inplace
        self.debug = debug
        self.max_value = max_value
        self.min_value = min_value
        self.scale = scale
        self.calculate_running = calculate_running
        self.running_list = []
        self.pctl = pctl
        if pctl < 1:                                                           # hm:222-225
            print('\n\npctl is {} please check!!!\n\n\n'.format(pctl))
            raise (SystemExit)

    def _host(self, name):
        """Host value of a scalar buffer, re-read (one sync) only when the buffer object or its
        version changed -- the reference syncs on every call (hm:265-271)."""
        t = getattr(self, name)
        cache = self.__dict__.setdefault('_host_cache', {})
        hit = cache.get(name)
        # the cache holds the tensor OBJECT (a strong reference: the scripts replace the buffer, noisynet.py:1258, and a freed
        # wrapper's id can be reused) and its version counter
        if hit is None or hit[0] is not t or hit[1] != t._version:
            hit = (t, t._version, float(t.reshape(-1)[0].item()))
            cache[name] = hit
        return hit[2]

    def _range(self, input):
        """Returns (min_value, max_value, stoch, range_dev).  range_dev (float32[2] device tensor) is set where the
        reference reads the range back from the device per call (``input.max().item()``, ``running_max.item()`` right
        after computing it): there the range is selected ON the device (ops.range_select: exact radix-select kthvalue +
        atomic max, SURVEY 8f.2) and handed to the quantizer kernels as a device pointer -- no host sync."""
        range_dev = None
        with torch.no_grad():
            min_value = self.min_value
            max_value = self.max_value
            if self.calculate_running:
                if self.min_value < 0:                                         # hm:232-239 signed weights
                    out4 = ops.range_select(input.detach(), self.pctl, mode=1)
                    self.running_min = out4[0].reshape([])
                    self.running_max = out4[1].reshape([])
                    self.calculate_running = False
                    range_dev = out4[2:4]
                else:                                                          # hm:240-259
                    if 224 in list(input.shape):
                        pctl = torch.tensor(0.92) if self.num_bits == 4 else torch.tensor(1.0)
                        mx = ops.tensor_stats(input.detach())[0:1]
                        range_dev = torch.cat([torch.full_like(mx, float(min_value)), mx])
                    else:
                        out4 = ops.range_select(input.detach(), mode=0, min_value=min_value,
                                                k_rank=int(input.numel() * self.pctl / 100.))
                        pctl = out4[0].reshape([])
                        range_dev = out4[2:4]
                    self.running_list.append(pctl)
            else:                                                              # hm:260-274
                if self.min_value < 0 and self._host('running_min') < 0:
                    min_value = self._host('running_min')
                    max_value = self._host('running_max')
                elif self.max_value > 0:
                    max_value = self.max_value
                elif self._host('running_max') > 0:
                    max_value = self._host('running_max')
                else:
                    print('\n\nSetting max_value to input.max\nrunning_max is ', self._host('running_max'))
                    mx = ops.tensor_stats(input.detach())[0:1]
                    range_dev = torch.cat([torch.full_like(mx, float(min_value)), mx])
            stoch = self.stochastic if self.training else 0                    # hm:283-286
        return min_value, max_value, stoch, range_dev

    def forward(self, input):
        min_value, max_value, stoch, range_dev = self._range(input)
        if range_dev is not None:
            return UniformQuantize.apply(input, self.num_bits, None, None, stoch, self.inplace, False, None, range_dev)
        out = UniformQuantize.apply(input, self.num_bits, min_value, max_value, stoch, self.inplace, False)
        # tag for the integer-code tensor-core path (consumed by NoisyConv2d / NoisyLinear)
        out._nn_quant = (int(self.num_bits), float(min_value), float(max_value))
        return out


def _f32(v):
    return torch.tensor(v, dtype=torch.float32).item()


def code_scales(x, w):
    """Integer-code scales for the tensor-core path from the tags QuantMeasure / _prepare_weight leave on their
    outputs: activations on the grid k * s (min 0) -> a_code_scale = s; weights on a symmetric grid
    (2k - qmax) * s/2 -> w_code_scale = s/2.  0.0 = no exact code representation."""
    a_cs = w_cs = 0.0
    t = getattr(x, "_nn_quant", None)
    if t is not None and t[1] == 0.0 and t[2] > 0 and t[0] <= 8:
        a_cs = _f32(max((t[2] - t[1]) / (2.0 ** t[0] - 1.0), 1e-6))
    t = getattr(w, "_nn_quant", None)
    if t is not None and t[1] == -t[2] and t[2] > 0 and t[0] <= 8:
        w_cs = _f32(max((t[2] - t[1]) / (2.0 ** t[0] - 1.0), 1e-6)) / 2.0
    return a_cs, w_cs


def _prepare_weight(mod, linear):
    """Branch order of hm:343-360 / hm:402-420.  Returns (weight, bias, ste) where ste is None or
    (raw_parameter, lo, hi): the quantized weight is then produced outside autograd and the masked
    gradient is routed to the raw parameter by the fused wgrad."""
    weight, bias = mod.weight, mod.bias
    quant_on = (0 < mod.num_bits_weight < 8) if linear else (mod.num_bits_weight > 0)
    if quant_on:
        qm = mod.quantize_weights
        lo, hi, stoch, range_dev = qm._range(mod.weight)
        if range_dev is not None:        # percentile calibration of the weight range just ran (once per module, hm:232-239):
            lo, hi = range_dev.tolist()  # the STE bounds of the fused wgrad are host scalars -> one sync, this call only
        with torch.no_grad():
            wq = ops.quantize_fwd(mod.weight.detach(), qm.num_bits, lo, hi, stoch)
        wq._nn_quant = (int(qm.num_bits), float(lo), float(hi))
        return wq, bias, (mod.weight, lo, hi)
    if mod.test_noise > 0 and not mod.training:
        weight = AddNoise.apply(mod.weight, mod.test_noise, mod.debug)
        if mod.bias is not None:
            bias = AddNoise.apply(mod.bias, mod.test_noise, mod.debug)
    elif mod.noise > 0 and mod.training:
        weight = AddNoise.apply(mod.weight, mod.noise, mod.debug)
        if mod.bias is not None:
            bias = AddNoise.apply(mod.bias, mod.noise, mod.debug)
    return weight, bias, None


class NoisyConv2d(nn.Conv2d):
    """hm:310-366."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=False,
                 num_bits=0, num_bits_weight=0, noise=0.5, test_noise=0, stochastic=True, debug=False):
        super(NoisyConv2d, self).__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)
        self.num_bits = num_bits
        self.fms = out_channels
        self.fs = kernel_size
        self.noise = noise
        self.num_bits_weight = num_bits_weight
        if num_bits > 0:
            self.quantize_input = QuantMeasure(self.num_bits, stochastic=stochastic, debug=debug)
        if num_bits_weight > 0:
            self.quantize_weights = QuantMeasure(self.num_bits_weight, min_value=-1.0, max_value=1.0,
                                                 stochastic=stochastic, debug=debug)
        self.stochastic = stochastic
        self.debug = debug
        self.test_noise = test_noise
        self.precision = None          # None -> ops default; "fp32" / "tf32" / "bf16"

    def _check_supported(self):
        if self.groups != 1 or tuple(self.dilation) != (1, 1):
            raise NotImplementedError("noisynet_b200.NoisyConv2d: groups/dilation != 1 are not on the hot path")
        if self.stride[0] != self.stride[1] or self.padding[0] != self.padding[1] or isinstance(self.padding, str):
            raise NotImplementedError("noisynet_b200.NoisyConv2d: anisotropic stride/padding not supported")

    def forward(self, input):
        self._check_supported()
        if self.num_bits > 0 and self.num_bits < 8:                            # hm:337-340
            qinput = self.quantize_input(input)
        else:
            qinput = input
        weight, bias, ste = _prepare_weight(self, linear=False)
        a_cs, w_cs = code_scales(qinput, weight)
        raw, lo, hi = ste if ste is not None else (None, 0.0, 0.0)
        return ops.ConvFn.apply(qinput, weight, bias, self.stride[0], self.padding[0], self.precision, raw, lo, hi,
                                a_cs, w_cs)


class NoisyLinear(nn.Linear):
    """hm:369-423."""

    def __init__(self, in_features, out_features, bias=False, num_bits=0, num_bits_weight=0, noise=0, test_noise=0,
                 stochastic=True, debug=False):
        super(NoisyLinear, self).__init__(in_features, out_features, bias)
        self.fc_in = in_features
        self.fc_out = out_features
        self.num_bits = num_bits
        self.num_bits_weight = num_bits_weight
        self.noise = noise
        if num_bits > 0:
            self.quantize_input = QuantMeasure(self.num_bits, stochastic=stochastic, debug=debug)
        if num_bits_weight > 0:
            self.quantize_weights = QuantMeasure(self.num_bits_weight, min_value=-1.0, max_value=1.0,
                                                 stochastic=stochastic, debug=debug)
        self.stochastic = stochastic
        self.debug = debug
        self.test_noise = test_noise
        self.precision = None

    def forward(self, input):
        if self.num_bits > 0 and self.num_bits < 8:                            # hm:394-397
            qinput = self.quantize_input(input)
        else:
            qinput = input
        weight, bias, ste = _prepare_weight(self, linear=True)
        a_cs, w_cs = code_scales(qinput, weight)
        lead = qinput.shape[:-1]
        x4 = qinput.reshape(-1, qinput.shape[-1])
        x4 = x4.view(x4.shape[0], x4.shape[1], 1, 1)
        w4 = weight.view(weight.shape[0], weight.shape[1], 1, 1)
        if ste is None:
            y = ops.ConvFn.apply(x4, w4, bias, 1, 0, self.precision, None, 0.0, 0.0, a_cs, w_cs)
        else:
            raw, lo, hi = ste
            y = ops.ConvFn.apply(x4, w4, bias, 1, 0, self.precision, raw.view(raw.shape[0], raw.shape[1], 1, 1), lo, hi,
                                 a_cs, w_cs)
        return y.view(*lead, weight.shape[0])


def distort_tensor(self, args, input, scale=0, stop=False):
    """hm:426-458: fixed Gaussian offsets (--offset/--offset_input) or uniform multiplicative distortion."""
    with torch.no_grad():
        if args.offset or args.offset_input:
            if self.generate_offsets:
                offs = torch.randn_like(input) * scale
                if '224' in input.shape:          # (sic) always False: a str is never in a torch.Size (hm:434)
                    self.input_offsets = offs
                elif stop:
                    self.act2_offsets = offs
                else:
                    self.act1_offsets = offs
                if stop:
                    self.generate_offsets = False
            if '224' in input.shape:
                out = input + self.input_offsets
            elif stop:
                out = input + self.act2_offsets
            else:
                out = input + self.act1_offsets
        else:
            out = ops.alt_noise(input, "distort_act", args.noise)
    return out
