#!/usr/bin/env python
"""Mints tests/golden/script_trace.npz: the loss curve of the UNMODIFIED reference script
(noisynet.py, module-level training loop :1215-1542) over its first steps, on a deterministic synthetic dataset --
the fixture the GPU test of the drop-in modules compares against (the tests never read the reference itself).
Needs a checkout of the reference (michaelklachko/NoisyNet) named by NOISYNET_REFERENCE:

    NOISYNET_REFERENCE=<checkout> python oracle/gen_script_trace.py            # CPU, a few minutes

Process-level shims only (SURVEY Appendix A): matplotlib / torch._six stubs, .cuda() -> identity, distribution
validation off, np.random seeded (the script seeds `random` and torch but permutes with np.random, noisynet.py:1232),
a step counter on torch.optim.AdamW.step that ends the run, a recorder on nn.CrossEntropyLoss.forward.
"""
import os
import subprocess
import sys
import tempfile
import textwrap

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("NOISYNET_REFERENCE", "")

STEPS = 60
BATCH = 64
ARGV = ["--current", "1", "--act_max", "5", "--w_max1", "0.3", "--LR", "0.005", "--L2_1", "0.0005", "--L2_2", "0.0002",
        "--q_a", "4", "--q_w", "4", "--batch_size", str(BATCH), "--nepochs", "1", "--seed", "0", "--no-augment"]


def synthetic_learnable_cifar(n, seed):
    """4-bit CIFAR-shaped inputs with labels that are a fixed linear function of the pixels (learnable in a few steps):
    label = argmax_c <x, P_c>, P_c in {-1, +1}^3072.  Pure integer arithmetic: identical on every host."""
    rng = np.random.default_rng(seed)
    proj = rng.integers(0, 2, (10, 3072)).astype(np.int64) * 2 - 1
    k = rng.integers(0, 16, (n, 3072)).astype(np.int64)
    labels = np.argmax(k @ proj.T, axis=1).astype(np.int64)
    return (k.astype(np.float32) / np.float32(15.0)).astype(np.float32), labels


RUNNER = textwrap.dedent('''
    import sys, types, runpy, collections.abc, json
    import numpy as np, torch
    sys.path.insert(0, {ref!r})
    six = types.ModuleType('torch._six'); six.container_abcs = collections.abc
    sys.modules['torch._six'] = six
    mpl = types.ModuleType('matplotlib'); mpl.use = lambda *a, **k: None
    plt = types.ModuleType('matplotlib.pyplot'); mpl.pyplot = plt
    sys.modules['matplotlib'] = mpl; sys.modules['matplotlib.pyplot'] = plt
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.distributions.Distribution.set_default_validate_args(False)
    _tensor = torch.tensor
    def tensor_cpu(*a, **k):
        k.pop('device', None)
        return _tensor(*a, **k)
    torch.tensor = tensor_cpu                       # torch.tensor(..., device='cuda:0') at noisynet.py:1258
    np.random.seed(0)
    torch.set_num_threads(8)
    losses = []
    class Stop(Exception):
        pass
    _fwd = torch.nn.CrossEntropyLoss.forward
    def fwd(self, out, lab):
        l = _fwd(self, out, lab)
        if torch.is_grad_enabled():
            losses.append(float(l))
        return l
    torch.nn.CrossEntropyLoss.forward = fwd
    _step = torch.optim.AdamW.step
    count = [0]
    def step(self, *a, **k):
        r = _step(self, *a, **k)
        count[0] += 1
        if count[0] >= {steps}:
            raise Stop()
        return r
    torch.optim.AdamW.step = step
    sys.argv = ['noisynet.py'] + {argv!r}
    try:
        runpy.run_path({script!r}, run_name='__main__')
    except Stop:
        pass
    json.dump(losses, open('losses.json', 'w'))
''')


def main(extra=()):
    import json
    out = os.path.join(ROOT, "tests", "golden", "script_trace.npz")
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "data"))
        x, y = synthetic_learnable_cifar(50000, seed=123)
        xt, yt = synthetic_learnable_cifar(10000, seed=124)
        np.savez(os.path.join(tmp, "data", "cifar_RGB_4bit.npz"), x, y, xt, yt)
        argv = ARGV + list(extra)
        code = RUNNER.format(ref=REF, steps=STEPS, argv=argv, script=os.path.join(REF, "noisynet.py"))
        r = subprocess.run([sys.executable, "-c", code], cwd=tmp, capture_output=True, text=True, timeout=3600)
        if not os.path.isfile(os.path.join(tmp, "losses.json")):
            sys.stderr.write(r.stdout[-2000:] + r.stderr[-4000:])
            raise SystemExit("reference run failed")
        losses = np.asarray(json.load(open(os.path.join(tmp, "losses.json"))), dtype=np.float64)
    print("reference script: %d steps, loss %.4f -> %.4f (mean of first / last 10: %.4f / %.4f)"
          % (len(losses), losses[0], losses[-1], losses[:10].mean(), losses[-10:].mean()))
    np.savez(out, losses=losses, argv=np.asarray(argv), steps=STEPS, batch=BATCH, data_seed=123, np_seed=0)
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv[1:])
