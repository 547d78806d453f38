#!/usr/bin/env python
"""Per-k-block hand-off timeline of the tiled wgmma kernel (NN_UMMA_KDEBUG=1): for every k-block of every CTA, when
producer thread 0 woke from the empty barrier / arrived on the full barrier, and when the first MMA warpgroup woke / released the stage.
The stamps are compiled in only with -DNN_KDEBUG:  NN_EXTRA_NVCC=-DNN_KDEBUG python __graft_entry__.py --force"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["NN_UMMA_KDEBUG"] = "1"
import numpy as np  # noqa: E402
import torch  # noqa: E402

from noisynet_b200 import _lib, ops  # noqa: E402

dev = torch.device("cuda:0")
lib = _lib.load()
B = 512
wq = ops.quantize_fwd(torch.randn(120, 65, 5, 5, device=dev) * 0.1, 4, -1.0, 1.0, 0.0)
gy = torch.randn(B, 120, 10, 10, device=dev)
for name, fn, ctas, nkb in (("conv2 dgrad", lambda: ops.conv_dgrad(gy, wq, (B, 65, 14, 14), precision="bf16", w_code_scale=1.0 / 15.0), 784, 47),):
    for _ in range(3):
        fn()
    rows = (ctas * nkb * 4 + 7) // 8
    buf = np.zeros((rows, 8), dtype=np.int64)
    n = lib.nn_debug_cta_timeline(buf.ctypes.data_as(C.c_void_p), rows)
    t = buf.reshape(-1)[:ctas * nkb * 4].reshape(ctas, nkb, 4).astype(np.float64)
    us = 1.0 / 1965.0
    ok = (t[:, :, 3] > 0).all(axis=1)
    t = t[ok]
    print("%s: %d CTAs with stamps" % (name, t.shape[0]))
    build = (t[:, :, 1] - t[:, :, 0]) * us
    mma = (t[:, :, 3] - t[:, :, 2]) * us
    p2m = (t[:, :, 2] - t[:, :, 1]) * us                  # producer arrived -> MMA warpgroup woke (same k-block)
    per_p = np.diff(t[:, :, 0], axis=1) * us
    per_m = np.diff(t[:, :, 2], axis=1) * us
    m2p = (t[:, 2:, 0] - t[:, :-2, 3]) * us              # MMA committed k-block kb -> producer woke for kb + 2 (2 stages)
    for lab, a in (("producer: wake -> arrive (issue 8 chunk copies)", build), ("producer arrive -> MMA warpgroup awake", p2m),
                   ("MMA warpgroup: awake -> stage released", mma), ("stage release(kb) -> producer awake for kb+stages", m2p),
                   ("k-block period (producer)", per_p), ("k-block period (MMA)", per_m)):
        print("   %-52s mean %6.3f us  p10 %6.3f  p50 %6.3f  p90 %6.3f" % (lab, a.mean(), np.percentile(a, 10), np.percentile(a, 50), np.percentile(a, 90)))
    print("   CTA main-loop span: mean %.1f us" % ((t[:, -1, 3] - t[:, 0, 0]) * us).mean())
