"""Process-level shims that let the UNMODIFIED reference import and run on CPU.

Only usable next to a checkout of the reference (michaelklachko/NoisyNet), named by the environment
variable NOISYNET_REFERENCE; used by ``oracle/gen_golden.py`` to mint the golden fixtures under
tests/golden/.  Never imported by the product package or the tests.

Shims (SURVEY §8c): (1) matplotlib stub (hardware_model.py:9 -> plot_histograms.py:1-4),
(2) torch._six stub (models/conv2d_layers.py:4), (3) .cuda() -> identity on GPU-less hosts
(utils.py:150-153, hardware_model.py:123-125), (4) distribution arg validation off so that
Normal(scale=0) is accepted (hardware_model.py:59).
"""
import collections.abc
import os
import sys
import types

import torch

REFERENCE_ROOT = os.environ.get("NOISYNET_REFERENCE", "")


def reference_available():
    return os.path.isfile(os.path.join(REFERENCE_ROOT, "hardware_model.py"))


def install():
    if not reference_available():
        raise RuntimeError("reference tree not found at %r: set NOISYNET_REFERENCE to a checkout of michaelklachko/NoisyNet"
                           % REFERENCE_ROOT)
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    if "matplotlib" not in sys.modules:
        mpl = types.ModuleType("matplotlib")
        mpl.use = lambda *a, **k: None
        plt = types.ModuleType("matplotlib.pyplot")
        mpl.pyplot = plt
        sys.modules["matplotlib"] = mpl
        sys.modules["matplotlib.pyplot"] = plt
    if "torch._six" not in sys.modules:
        six = types.ModuleType("torch._six")
        six.container_abcs = collections.abc
        sys.modules["torch._six"] = six
    if not torch.cuda.is_available():
        torch.Tensor.cuda = lambda self, *a, **k: self
        torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.distributions.Distribution.set_default_validate_args(False)


def import_reference_ops():
    """Returns the reference's (hardware_model, quant) modules, unmodified."""
    install()
    import importlib
    hm = importlib.import_module("hardware_model")
    q = importlib.import_module("quant")
    assert hm.__file__.startswith(REFERENCE_ROOT), hm.__file__
    assert q.__file__.startswith(REFERENCE_ROOT), q.__file__
    return hm, q


def load_reference_net_class(args):
    """Executes ONLY the ``class Net`` statement of the reference script (noisynet.py:326-695)
    from its original location, in a namespace providing the globals it reads.  The script
    itself cannot be imported because its module level runs the whole training."""
    hm, _ = import_reference_ops()
    import numpy as np
    import torch.nn as nn
    src_path = os.path.join(REFERENCE_ROOT, "noisynet.py")
    with open(src_path) as f:
        lines = f.readlines()
    start = next(i for i, l in enumerate(lines) if l.startswith("class Net(nn.Module):"))
    end = next(i for i in range(start + 1, len(lines))
               if lines[i].strip() and not lines[i].startswith((" ", "\t", "#")))
    ns = dict(torch=torch, nn=nn, np=np, args=args,
              QuantMeasure=hm.QuantMeasure, NoisyConv2d=hm.NoisyConv2d, NoisyLinear=hm.NoisyLinear,
              add_noise_calculate_power=hm.add_noise_calculate_power)
    code = compile("".join(["\n"] * start + lines[start:end]), src_path, "exec")
    exec(code, ns)
    return ns["Net"]
