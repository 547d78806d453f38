"""Edge cases of the CTA-pair schedule of the TMA-im2col kernel (csrc/nn_conv_tma.cu): two CTAs walk adjacent m-tiles of
one n-tile and multicast a weight half each; with an odd m-tile count the second CTA of the last pair only serves its
weight half and stores nothing.  Code-mode operands make the main contraction exact, so every output is checked
against float64 (rtol 1e-6 forward, 2e-5 dgrad as in test_gpu_tma.py), the noisy output against the fp32 kernel with
the same Philox stream, and two launches must agree bit for bit.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

S_A, S_W = 5.0 / 15.0, 1.0 / 15.0


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__ as entry
    entry.build()
    return torch.device("cuda:0")


def _operands(shape, seed):
    B, Cin, H, W, Cout, k, s, p = shape
    gen = torch.Generator().manual_seed(seed)
    ka = torch.randint(0, 16, (B, Cin, H, W), generator=gen).float()
    cw = (torch.randint(0, 16, (Cout, Cin, k, k), generator=gen) * 2 - 15).float()
    w_raw = torch.randn(Cout, Cin, k, k, generator=gen) * 0.3
    return gen, ka, cw, w_raw


SHAPES = [  # B, Cin, H, W, Cout, k, stride, pad      forward m-tiles x n-tiles (noisy) / dgrad m-tiles
    (1, 65, 14, 14, 120, 5, 1, 0),      # conv2, one image: 1 x 1 / 2
    (3, 65, 14, 14, 120, 5, 1, 0),      # conv2, three images: 3 x 1 / 5
    (14, 96, 10, 10, 136, 1, 2, 0),     # 1x1 stride 2 (no TMA dgrad): 3 x 2
]


@pytest.mark.parametrize("shape", SHAPES)
def test_cluster_forward_code_mode(dev, shape):
    from noisynet_b200 import ops
    from noisynet_b200._lib import NOISE_EXTERNAL
    B, Cin, H, W, Cout, k, s, p = shape
    _, ka, cw, w_raw = _operands(shape, 17 + B)
    x, wq = ka * S_A, cw * S_W
    xd, wqd, wrd = x.to(dev), wq.to(dev), w_raw.to(dev)
    exact = F.conv2d(ka.double(), cw.double(), None, s, p) * (float(np.float32(S_A)) * float(np.float32(S_W)))
    ys = [ops.noisy_conv_fwd(xd, wqd, None, None, s, p, precision="bf16", a_code_scale=S_A, w_code_scale=S_W)["y"]
          for _ in range(2)]
    assert ops.error_flag() == 0
    assert torch.allclose(ys[0].cpu().double(), exact, rtol=1e-6, atol=1e-9), (ys[0].cpu().double() - exact).abs().max()
    assert torch.equal(ys[0], ys[1])
    scale = ops.tensor_stats(xd)[0:1]
    kw = dict(noise_mode=NOISE_EXTERNAL, current=1.0, scale_dev=scale, want_y=False)
    rs = [ops.noisy_conv_fwd(xd, wqd, wrd, None, s, p, precision="bf16", a_code_scale=S_A, w_code_scale=S_W,
                             rng=ops._fixed_rng(7, 3), **kw)["y_noisy"] for _ in range(2)]
    r32 = ops.noisy_conv_fwd(xd, wqd, wrd, None, s, p, precision="fp32", rng=ops._fixed_rng(7, 3), want_z=True,
                             want_sigma=True, **kw)
    assert ops.error_flag() == 0
    assert torch.equal(rs[0], rs[1])
    noise_max = (r32["z"] * r32["sigma"]).abs().max().item()
    assert (rs[0] - r32["y_noisy"]).abs().max().item() <= 3e-3 * noise_max + 1e-5


@pytest.mark.parametrize("shape", [sh for sh in SHAPES if sh[6] == 1])
def test_cluster_dgrad_code_mode(dev, shape):
    from noisynet_b200 import ops
    B, Cin, H, W, Cout, k, s, p = shape
    gen, ka, cw, _ = _operands(shape, 29 + B)
    OH, OW = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    gy = torch.randn(B, Cout, OH, OW, generator=gen).bfloat16().float()
    wqd = (cw * S_W).to(dev)
    gxs = [ops.conv_dgrad(gy.to(dev), wqd, (B, Cin, H, W), s, p, precision="bf16", w_code_scale=S_W) for _ in range(2)]
    assert ops.error_flag() == 0
    ref = torch.nn.grad.conv2d_input((B, Cin, H, W), cw.double(), gy.double(), s, p) * float(np.float32(S_W))
    assert torch.allclose(gxs[0].cpu().double(), ref, rtol=2e-5, atol=1e-5 * ref.abs().max().item())
    assert torch.equal(gxs[0], gxs[1])
