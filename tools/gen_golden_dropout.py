"""Mint tests/golden/net_step_dropout.npz: one training step of the UNMODIFIED reference noisynet.Net with
--dropout 0.2 --dropout_conv 0.2 (noisynet.py:375-376, :456-457, :512-513, :565-566), fp and 4-bit, narrow widths.

Same structure as the net_step case of oracle/gen_golden.py, written to its own file so that the existing fixtures are
not rewritten:
    NOISYNET_REFERENCE=<checkout> python tools/gen_golden_dropout.py
The dropout masks are drawn by torch's CPU generator inside the reference's forward; the test replays the same seed, so
its F.dropout calls draw the same masks in the same order.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402
from oracle.gen_golden import OUT, net_args, t2n  # noqa: E402

P = 0.2


def gen_net_dropout():
    from oracle import noisynet_oracle as O
    out = {}
    for tag, q in (("fp", 0), ("q4", 4)):
        args = net_args(q_a1=q, q_a2=q, q_a3=q, q_a4=q, q_w1=q, q_w2=q, q_w3=q, q_w4=q,
                        fm1=9, fm2=12, fc=24, dropout=P, dropout_conv=P)
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
        oa = O.default_args(q_a=q, q_w=q, quant_max2=4.0, quant_max4=4.5, fm1=9, fm2=12, fc=24, dropout=P, dropout_conv=P)
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
    out["p"] = np.asarray(P)
    np.savez_compressed(os.path.join(OUT, "net_step_dropout.npz"), **t2n(out))
    print("net_step_dropout.npz", len(out), "arrays")


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gen_net_dropout()
