"""SURVEY.md section 8f.3 (the callers either side of the path): a ResNet BasicBlock built from the drop-in modules
exactly as models/resnet.py:16-62 builds it -- quantize1 -> conv1 3x3 (stride s, pad 1) -> bn1 -> Hardtanh(0, act_max)
-> quantize2 -> conv2 3x3 -> bn2, shortcut conv3 1x1 stride s -> bn3 on the quantized block input, sum (forward order:
models/resnet.py:72-155) -- against the same block evaluated on the CPU with the oracle's functions.

Deterministic configuration (stochastic rounding off, weight noise off, fixed activation ranges) so that the only
differences are arithmetic: fp32 kernels within 2e-5 relative of the oracle; tensor-core kernels exact for the 4-bit
forward contractions (integer codes) and within the bf16 operand tolerance (1.5e-2 of max) for the gradients.
Geometries exercised through the public module API: 3x3 pad 1 stride 1/2, 1x1 stride 2, 16 -> 32 channels.
"""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import noisynet_oracle as O

pytestmark = pytest.mark.gpu

ACT_MAX, QA, QW = 5.0, 4, 4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__ as entry
    entry.build()
    return torch.device("cuda:0")


class Block(nn.Module):
    """models/resnet.py BasicBlock on noisynet_b200's drop-in modules (constructor arguments as resnet.py:40-61)."""

    def __init__(self, inplanes, planes, stride, precision):
        super().__init__()
        from noisynet_b200.hardware_model import NoisyConv2d, QuantMeasure
        kw = dict(bias=False, num_bits=0, num_bits_weight=QW, noise=0.0, test_noise=0.0, stochastic=0.0)
        self.conv1 = NoisyConv2d(inplanes, planes, kernel_size=3, stride=stride, padding=1, **kw)
        self.conv2 = NoisyConv2d(planes, planes, kernel_size=3, stride=1, padding=1, **kw)
        self.conv3 = NoisyConv2d(inplanes, planes, kernel_size=1, stride=stride, **kw)
        self.bn1, self.bn2, self.bn3 = nn.BatchNorm2d(planes), nn.BatchNorm2d(planes), nn.BatchNorm2d(planes)
        self.relu = nn.Hardtanh(0.0, ACT_MAX)
        self.quantize1 = QuantMeasure(QA, stochastic=0.0, max_value=ACT_MAX)
        self.quantize2 = QuantMeasure(QA, stochastic=0.0, max_value=ACT_MAX)
        for c in (self.conv1, self.conv2, self.conv3):
            c.precision = precision

    def forward(self, x):
        x = self.quantize1(x)
        out = self.quantize2(self.relu(self.bn1(self.conv1(x))))
        out = self.bn2(self.conv2(out))
        return out + self.bn3(self.conv3(x))


def oracle_block(x, w, bn, stride):
    """The same block on the CPU: oracle quantizer (hardware_model.py:133-183 restated), torch conv / batch norm."""
    def q_act(t):
        y = O.uniform_quantize_fwd(t.detach(), QA, 0.0, ACT_MAX)
        return _STE.apply(t, y, 0.0, ACT_MAX)

    def q_w(t):
        y = O.uniform_quantize_fwd(t.detach(), QW, -1.0, 1.0)
        return _STE.apply(t, y, -1.0, 1.0)

    xq = q_act(x)
    out = F.conv2d(xq, q_w(w[0]), None, stride, 1)
    out = F.batch_norm(out, None, None, bn[0][0], bn[0][1], True, 0.1, 1e-5)
    out = q_act(F.hardtanh(out, 0.0, ACT_MAX))
    out = F.conv2d(out, q_w(w[1]), None, 1, 1)
    out = F.batch_norm(out, None, None, bn[1][0], bn[1][1], True, 0.1, 1e-5)
    res = F.conv2d(xq, q_w(w[2]), None, stride, 0)
    res = F.batch_norm(res, None, None, bn[2][0], bn[2][1], True, 0.1, 1e-5)
    return out + res


class _STE(torch.autograd.Function):
    """Forward: the given quantized value; backward: the saturated straight-through estimator (hm:176-183)."""

    @staticmethod
    def forward(ctx, t, y, lo, hi):
        ctx.save_for_backward(t)
        ctx.lo, ctx.hi = lo, hi
        return y.clone()

    @staticmethod
    def backward(ctx, g):
        (t,) = ctx.saved_tensors
        return O.uniform_quantize_bwd(t, g, ctx.lo, ctx.hi), None, None, None


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_basic_block_matches_oracle(dev, stride, precision):
    from noisynet_b200 import ops
    gen = torch.Generator().manual_seed(10 * stride + len(precision))
    B, Cin, Cout, H = 6, 16, 32, 16
    x = (torch.rand(B, Cin, H, H, generator=gen) * 6.0 - 0.5)           # some values outside [0, act_max]: STE saturation
    w = [torch.randn(Cout, Cin, 3, 3, generator=gen) * 0.4, torch.randn(Cout, Cout, 3, 3, generator=gen) * 0.4,
         torch.randn(Cout, Cin, 1, 1, generator=gen) * 0.6]              # some |w| > 1: weight STE saturation
    bn = [(torch.rand(Cout, generator=gen) + 0.5, torch.randn(Cout, generator=gen) * 0.2) for _ in range(3)]
    gy = torch.randn(B, Cout, H // stride, H // stride, generator=gen)

    # CPU oracle
    xo = x.clone().requires_grad_(True)
    wo = [t.clone().requires_grad_(True) for t in w]
    bo = [(g.clone().requires_grad_(True), b.clone().requires_grad_(True)) for g, b in bn]
    yo = oracle_block(xo, wo, bo, stride)
    yo.backward(gy)

    blk = Block(Cin, Cout, stride, precision).to(dev).train()
    with torch.no_grad():
        for conv, t in zip((blk.conv1, blk.conv2, blk.conv3), w):
            conv.weight.copy_(t)
        for m, (g, b) in zip((blk.bn1, blk.bn2, blk.bn3), bn):
            m.weight.copy_(g); m.bias.copy_(b)
    xd = x.to(dev).requires_grad_(True)
    yd = blk(xd)
    yd.backward(gy.to(dev))
    assert ops.error_flag() == 0

    def close(a, b, rel, what):
        # Elementwise |err| <= rel * max|ref|, except for the handful of elements downstream of a 4-bit code that
        # flipped in quantize2: its input is a batch-norm output, CUDA and CPU batch norm differ in the last ulp, and
        # a value within an ulp of a rounding boundary lands on the other side (about one in 1e5 elements).  Such a
        # flip changes the affected outputs by a whole code step, so it cannot hide a systematic error.
        a, b = a.detach().cpu(), b.detach()
        lim = rel * b.abs().max().item() + 1e-6
        bad = ((a - b).abs() > lim).float().mean().item()
        assert bad <= 2e-3, (what, bad, (a - b).abs().max().item(), lim)

    # forward: the contractions are exact integer sums in code mode; what remains is fp32 batch-norm arithmetic
    close(yd, yo, 2e-5 if precision == "fp32" else 2e-4, "y")
    rel = 2e-5 if precision == "fp32" else 1.5e-2
    close(xd.grad, xo.grad, rel, "gx")
    for i, conv in enumerate((blk.conv1, blk.conv2, blk.conv3)):
        close(conv.weight.grad, wo[i].grad, rel, "gw%d" % i)
    for i, m in enumerate((blk.bn1, blk.bn2, blk.bn3)):
        close(m.weight.grad, bo[i][0].grad, rel, "dgamma%d" % i)
        close(m.bias.grad, bo[i][1].grad, rel, "dbeta%d" % i)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_batchnorm_folded_into_noisy_conv_inference(dev, precision):
    """main.py:540-654 (merge_batchnorm, the ImageNet drivers' inference mode): the BatchNorm scale gamma / sqrt(var + eps) is
    multiplied into the conv weights through the state_dict (same keys as the reference's modules) and the shift
    beta - mean * scale becomes the conv bias, so that conv'(x) == bn_eval(conv(x)).  Exercises the bias path of
    nn_noisy_conv_fwd on the drop-in NoisyConv2d (3x3 pad 1 and 1x1 stride 2, unquantized weights as in merge mode)."""
    from noisynet_b200 import ops
    from noisynet_b200.hardware_model import NoisyConv2d
    gen = torch.Generator().manual_seed(4)
    for (Cin, Cout, k, s, p) in ((16, 32, 3, 1, 1), (32, 48, 1, 2, 0)):
        kw = dict(num_bits=0, num_bits_weight=0, noise=0.0, test_noise=0.0, stochastic=0.0)
        conv = NoisyConv2d(Cin, Cout, kernel_size=k, stride=s, padding=p, bias=False, **kw).to(dev)
        bn = nn.BatchNorm2d(Cout).to(dev)
        with torch.no_grad():
            conv.weight.copy_(torch.randn(conv.weight.shape, generator=gen) * 0.2)
            bn.weight.copy_(torch.rand(Cout, generator=gen) + 0.5); bn.bias.copy_(torch.randn(Cout, generator=gen) * 0.3)
            bn.running_mean.copy_(torch.randn(Cout, generator=gen) * 0.2); bn.running_var.copy_(torch.rand(Cout, generator=gen) + 0.3)
        conv.precision = precision
        conv.eval(); bn.eval()
        x = torch.randn(4, Cin, 12, 12, generator=gen).to(dev)
        with torch.no_grad():
            ref = bn(conv(x))
            merged = NoisyConv2d(Cin, Cout, kernel_size=k, stride=s, padding=p, bias=True, **kw).to(dev)
            merged.precision = precision
            merged.eval()
            sd = merged.state_dict()
            scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
            sd["weight"].copy_(conv.weight * scale.view(-1, 1, 1, 1))            # main.py:598: param.data *= bn_weight / sqrt(var + eps)
            sd["bias"].copy_(bn.bias - bn.running_mean * scale)
            out = merged(x)
        assert ops.error_flag() == 0
        tol = (2e-5 if precision == "fp32" else 1.5e-2) * ref.abs().max().item()
        assert (out - ref).abs().max().item() <= tol, (precision, k, (out - ref).abs().max().item(), tol)
