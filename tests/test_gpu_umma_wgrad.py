"""Tensor-core wgrad (MN-major operands, split reduction) against torch's fp32 conv2d_weight.
Tolerance: grad_output (and, outside code mode, the activations) are rounded to bf16 before the
tensor-core contraction -> |err| <= 1.5e-2 * max|ref| (errors average down over the pixel reduction)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SHAPES = [  # B, Cin, H, W, Cout, k, stride, pad
    (4, 3, 32, 32, 65, 5, 1, 0),
    (5, 65, 14, 14, 120, 5, 1, 0),
    (9, 3000, 1, 1, 390, 1, 1, 0),
    (33, 390, 1, 1, 10, 1, 1, 0),
    (2, 16, 15, 15, 24, 3, 1, 1),
    (2, 16, 14, 14, 32, 1, 2, 0),
    (1, 3, 33, 33, 16, 7, 2, 3),
    (3, 40, 9, 9, 200, 3, 1, 1),        # Cout > 128: two 128-channel tiles
    (1, 1, 5, 5, 1, 5, 1, 0),
    (3, 64, 12, 12, 64, 3, 1, 1),       # TMA-staged operands: one 64-channel chunk per tap, padding taps
    (2, 128, 9, 9, 96, 3, 1, 1),        # two chunks per tap, 18 atoms = 4.5 column tiles
    (2, 64, 16, 16, 136, 3, 2, 1),      # stride 2, two n-tiles
    (2, 96, 10, 10, 24, 1, 2, 0),       # 1x1 stride 2, 64 + 32 channels (zero-filled second chunk)
    (2, 72, 8, 8, 40, 3, 1, 1),         # 64 + 8 channels, 3 column tiles: the remainder accumulator (9 taps, 80 columns)
    (2, 72, 9, 9, 24, 5, 1, 2),         # 64 + 8 channels, 7 column tiles: the remainder accumulator (8 columns per tap), padding
    (3, 136, 8, 8, 16, 3, 2, 1),        # 128 + 8 channels, stride 2: remainder accumulator at channel 128
    (2, 136, 7, 7, 16, 1, 1, 0),        # 128 + 8 channels, 1x1
]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__ as entry
    entry.build()
    return torch.device("cuda:0")


@pytest.mark.parametrize("shape", SHAPES)
def test_wgrad_bf16(dev, shape):
    from noisynet_b200 import ops
    B, Cin, H, W, Cout, k, s, p = shape
    gen = torch.Generator().manual_seed(77 + sum(shape))
    x = torch.randn(B, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, k, k, generator=gen)
    OH, OW = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    gy = torch.randn(B, Cout, OH, OW, generator=gen)
    ref = torch.nn.grad.conv2d_weight(x, w.shape, gy, s, p)
    gw = ops.conv_wgrad(gy.to(dev), x.to(dev), w.shape, s, p, precision="bf16")
    assert ops.error_flag() == 0
    err = (gw.cpu() - ref).abs().max().item()
    assert err <= 1.5e-2 * ref.abs().max().item() + 1e-6, (err, ref.abs().max().item())
    # deterministic (fixed-order split reduction) and STE mask of the weight quantizer fused
    gw2 = ops.conv_wgrad(gy.to(dev), x.to(dev), w.shape, s, p, precision="bf16")
    assert torch.equal(gw, gw2)
    gwm = ops.conv_wgrad(gy.to(dev), x.to(dev), w.shape, s, p, w_raw=w.to(dev), w_lo=-1.0, w_hi=1.0, precision="bf16")
    keep = ((w >= -1.0) & (w <= 1.0)).float()
    assert torch.equal(gwm.cpu(), gw.cpu() * keep)
    # integer-code activations: the activation operand is exact, only grad_output is rounded
    s_a = 5.0 / 15.0
    ka = torch.randint(0, 16, (B, Cin, H, W), generator=gen).float()
    xq = ka * s_a
    refq = torch.nn.grad.conv2d_weight(xq, w.shape, gy, s, p)
    gwq = ops.conv_wgrad(gy.to(dev), xq.to(dev), w.shape, s, p, precision="bf16", a_code_scale=s_a)
    gyb = gy.bfloat16().float()
    refq_b = torch.nn.grad.conv2d_weight(xq.double(), w.shape, gyb.double(), s, p).float()
    assert ops.error_flag() == 0
    assert (gwq.cpu() - refq_b).abs().max().item() <= 2e-5 * refq_b.abs().max().item() + 1e-5
    assert (gwq.cpu() - refq).abs().max().item() <= 1.5e-2 * refq.abs().max().item() + 1e-6


def test_wgrad_full_size(dev):
    """BASELINE config-2 sizes: conv1 and conv2 at batch 512 -- adjoint identity <gy, conv(x,w)> == <wgrad, w>."""
    from noisynet_b200 import ops
    gen = torch.Generator().manual_seed(1)
    for (Cin, H, Cout) in ((3, 32, 65), (65, 14, 120)):
        x = (torch.randint(0, 16, (512, Cin, H, H), generator=gen).float() / 3.0).to(dev)
        w = (torch.randn(Cout, Cin, 5, 5, generator=gen) * 0.1).to(dev)
        y = ops.noisy_conv_fwd(x, w, precision="fp32")["y"]
        gy = torch.randn_like(y)
        gw = ops.conv_wgrad(gy, x, w.shape, precision="bf16", a_code_scale=1.0 / 3.0)
        assert ops.error_flag() == 0
        a = (gy.bfloat16().float() * y).sum().item()
        b = (gw * w).sum().item()
        assert abs(a - b) <= 2e-3 * abs(a) + 1.0, (a, b)
        g32 = ops.conv_wgrad(gy, x, w.shape, precision="fp32")
        assert (gw - g32).abs().max().item() <= 1.5e-2 * g32.abs().max().item()
