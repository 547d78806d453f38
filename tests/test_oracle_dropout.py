"""Dropout in the CPU oracle (noisynet.py:375-376, :456-457, :512-513, :565-566) against the unmodified reference, and the
numpy statement of the stage kernels' keep-mask stream.

``OracleNetDropout`` is oracle.noisynet_oracle.OracleNet with the reference's three dropout sites: after ReLU + clamp and
before the next quantizer, after relu1 only with --dropout_conv > 0 (at rate --dropout), after relu2 (before the flatten)
and after relu3.  Without injected masks it calls F.dropout, which draws from torch's CPU generator in the reference's
order (that is how tests/golden/net_step_dropout.npz is matched); with ``rnd`` carrying keep1/keep2/keep3 it applies
``x * (mask / (1 - p))`` -- the arithmetic of torch's dropout on fp32 -- so the CUDA kernels can be matched mask for mask.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import noisynet_oracle as O


def T(a):
    return torch.from_numpy(np.asarray(a))


# --------------------------------------------------------------------------
# Spec of the stage kernels' dropout stream (NOT a restatement of the reference)
# --------------------------------------------------------------------------

def stage_groups(B, C, HW, Cp):
    """Philox group and word of every element (b, c, r) of a stage's BN input [B, C, HW]: the thread of (pixel, 8-channel
    chunk) i = (b*HW + r) * Cp/8 + c//8 draws groups 2i and 2i+1; channel c uses group 2i + (c%8)//4, word c%4."""
    b = np.arange(B, dtype=np.uint64)[:, None, None]
    c = np.arange(C, dtype=np.uint64)[None, :, None]
    r = np.arange(HW, dtype=np.uint64)[None, None, :]
    i = (b * np.uint64(HW) + r) * np.uint64(Cp // 8) + c // np.uint64(8)
    return i * np.uint64(2) + (c % np.uint64(8)) // np.uint64(4), np.broadcast_to((c % np.uint64(4)).astype(np.int64), i.shape)


def _words(B, C, HW, Cp, seed, offset):
    g, w = stage_groups(B, C, HW, Cp)
    r = O.philox4x32_10(g.reshape(-1), seed, offset)
    return np.take_along_axis(r, w.reshape(-1, 1), axis=1).reshape(B, C, HW)


def philox_keep_mask(B, C, HW, Cp, p, seed, offset):
    """The stage kernels' keep mask uint8 [B, C, HW]: keep iff u01(word) >= float32(p), u01 = (r >> 8) * 2^-24."""
    return (O.philox_uniform01(_words(B, C, HW, Cp, seed, offset)) >= np.float32(p)).astype(np.uint8)


def philox_stage_uniform(B, C, HW, Cp, s, seed, offset):
    """The hot stage kernels' stochastic-rounding draws (same thread mapping): U[-s, s) = fl(fl(u * 2s) - s)."""
    u = O.philox_uniform01(_words(B, C, HW, Cp, seed, offset))
    two_s = np.float32(np.float32(2.0) * np.float32(s))
    return ((u * two_s).astype(np.float32) - np.float32(s)).astype(np.float32)


def drop_scale(p):
    """fl(1 / fl(1 - p)): torch's bernoulli_(1 - p).div_(1 - p) on an fp32 tensor."""
    return np.float32(1.0) / np.float32(1.0 - p)


def apply_dropout(h, mask, p):
    """x * (mask / (1 - p)) as torch's CPU dropout forms it; autograd gives g * mask / (1 - p)."""
    return h * mask.to(h.dtype).div(1.0 - p)


class OracleNetDropout(O.OracleNet):
    """OracleNet.forward (noisynet.py:378-594) plus the three dropout sites."""

    def _drop(self, h, rnd, name):
        a = self.args
        if not self.training:
            return h
        if rnd is not None and name in rnd:
            return apply_dropout(h, rnd[name].reshape(h.shape), a.dropout)
        return F.dropout(h, a.dropout, True)

    def forward(self, x, i=0, rnd=None):
        a = self.args
        if a.q_a > 0:
            x = self._q(x, a.q_a, 0.0, 1.0, rnd, "ua1")
        c1 = self._layer(x, self.conv1, 0, "conv", a.merged_dac, i, rnd)
        h = self.bn1(F.max_pool2d(c1, 2, 2))
        h = O.act_clamp(F.relu(h), a.act_max)
        if a.dropout_conv > 0 and a.dropout > 0:
            h = self._drop(h, rnd, "keep1")                                   # :456-457
        if a.q_a > 0:
            h = self._q(h, a.q_a, 0.0, a.quant_max2 if a.quant_max2 > 0 else float(h.max()), rnd, "ua2")
        c2 = self._layer(h, self.conv2, 1, "conv", False, i, rnd)
        h = self.bn2(F.max_pool2d(c2, 2, 2))
        h = O.act_clamp(F.relu(h), a.act_max)
        if a.dropout > 0:
            h = self._drop(h, rnd, "keep2")                                   # :512-513
        h = h.view(h.size(0), -1)
        if a.q_a > 0:
            h = self._q(h, a.q_a, 0.0, a.act_max / (1.0 - a.dropout), rnd, "ua3")
        l1 = self._layer(h, self.linear1, 2, "linear", a.merged_dac, i, rnd)
        h = O.act_clamp(F.relu(self.bn3(l1)), a.act_max)
        if a.dropout > 0:
            h = self._drop(h, rnd, "keep3")                                   # :565-566
        if a.q_a > 0:
            h = self._q(h, a.q_a, 0.0, a.quant_max4 if a.quant_max4 > 0 else float(h.max()), rnd, "ua4")
        l2 = self._layer(h, self.linear2, 3, "linear", False, i, rnd)
        return self.bn4(l2)


def _net_step(golden, tag, q):
    g = golden("net_step_dropout")
    p = float(g["p"])
    a = O.default_args(q_a=q, q_w=q, quant_max2=4.0, quant_max4=4.5, fm1=9, fm2=12, fc=24, dropout=p, dropout_conv=p)
    m = OracleNetDropout(a)
    sd = {k[len(tag) + 5:]: T(v) for k, v in g.items() if k.startswith(f"{tag}_sd0_")}
    sd = {k: v for k, v in sd.items() if k in m.state_dict()}
    m.load_state_dict(sd)
    opt = O.make_optimizer(m, a)
    m.train()
    torch.manual_seed(31337)      # same generator state as the reference run: same draw order, dropout masks included
    loss, logits = O.train_step(m, opt, T(g[f"{tag}_x"]), T(g[f"{tag}_label"]), i=0)
    return g, m, loss, logits


def _check(golden, tag, q):
    g, m, loss, logits = _net_step(golden, tag, q)
    assert torch.allclose(logits, T(g[f"{tag}_logits"]), atol=2e-5, rtol=1e-5)
    assert abs(loss.item() - float(g[f"{tag}_loss"])) < 1e-5
    for k, p in m.named_parameters():
        ref = T(g[f"{tag}_grad_{k}"])
        assert torch.allclose(p.grad, ref, atol=1e-5, rtol=1e-4), k
    for k, v in m.state_dict().items():
        assert torch.allclose(v, T(g[f"{tag}_sd1_{k}"]), atol=1e-5, rtol=1e-4), k


def test_net_step_dropout_fp(golden):
    _check(golden, "fp", 0)


def test_net_step_dropout_q4(golden):
    _check(golden, "q4", 4)


def test_dropout_changes_the_step(golden):
    """The fixture really exercises dropout: the same step with p = 0 gives a different loss."""
    g, _, loss, _ = _net_step(golden, "q4", 4)
    a = O.default_args(q_a=4, q_w=4, quant_max2=4.0, quant_max4=4.5, fm1=9, fm2=12, fc=24)
    m = OracleNetDropout(a)
    sd = {k[len("q4_sd0_"):]: T(v) for k, v in g.items() if k.startswith("q4_sd0_")}
    m.load_state_dict({k: v for k, v in sd.items() if k in m.state_dict()})
    m.train()
    torch.manual_seed(31337)
    loss0, _ = O.train_step(m, O.make_optimizer(m, a), T(g["q4_x"]), T(g["q4_label"]), i=0)
    assert abs(loss0.item() - loss.item()) > 1e-3


def test_injected_masks_reproduce_f_dropout():
    """x * (mask / (1 - p)) with the mask F.dropout drew is bit-identical to F.dropout's output and gradient."""
    g = torch.Generator().manual_seed(4)
    x = (torch.rand(6, 7, 5, 5, generator=g) * 3).requires_grad_(True)
    gy = torch.randn(6, 7, 5, 5, generator=g)
    torch.manual_seed(9)
    y = F.dropout(x, 0.1, True)
    y.backward(gy)
    gx = x.grad.clone()
    mask = (y != 0) | (x == 0)
    x.grad = None
    y2 = apply_dropout(x, mask, 0.1)
    y2.backward(gy)
    assert torch.equal(y, y2) and torch.equal(gx, x.grad)
    k = drop_scale(0.1)
    assert torch.equal(y2.detach(), x.detach() * torch.from_numpy(np.asarray(k)) * mask)


def test_philox_keep_mask_statistics():
    B, C, HW, Cp, p = 16, 13, 25, 16, 0.1
    m = philox_keep_mask(B, C, HW, Cp, p, seed=7, offset=3)
    n = m.size
    frac = m.mean()
    assert abs(frac - (1 - p)) <= 5 * np.sqrt(p * (1 - p) / n), frac
    m2 = philox_keep_mask(B, C, HW, Cp, p, seed=7, offset=3 + (1 << 32))
    assert (m != m2).mean() > 0.1                                           # another offset: another mask
    u = philox_stage_uniform(B, C, HW, Cp, 0.5, seed=7, offset=3)
    assert u.min() >= -0.5 and u.max() < 0.5
    # the keep words are the rounding words' mapping on another stream: same seed/offset -> u01 < p <=> dropped
    u01 = (u + np.float32(0.5)) / np.float32(1.0)
    assert np.array_equal(m, (u01 >= np.float32(p)).astype(np.uint8))
