#!/usr/bin/env python
"""Per-tile timeline of the persistent shift-GEMM kernel k_conv_shift (conv1: 3 -> 65 channels, 5x5, batch 512).

Needs a library built with NN_EXTRA_NVCC=-DNN_KDEBUG; the stamps are taken when NN_UMMA_DEBUG is set (done here).  Per tile
the kernel stamps: MMA warpgroup 0's A stage ready and half 0 stored, MMA warpgroup 1's half 1 stored; epilogue warp 0
(rows 0-63) accumulators seen and done; epilogue warp 2 (rows 64-127) accumulators seen and done.  The clock is the card's
SM clock rate.  The number to watch is the epilogue's wait for accumulators: the time from the end of a warp's epilogue
of one tile to the moment it sees the next tile's half, which MMA warpgroups running ahead would bring to zero.
"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["NN_UMMA_DEBUG"] = "1"
import numpy as np  # noqa: E402
import torch  # noqa: E402

from noisynet_b200 import _lib, ops  # noqa: E402
from noisynet_b200._lib import NOISE_MERGED, NOISE_NONE, PREC_BF16, ConvFwdArgs, ConvGeom  # noqa: E402

STAMPS = 8      # SH_DBG in nn_conv_umma.cu


def pooled_fwd(lib, x, wq, w_raw, scale, s_a):
    """The benchmarked launch: noisy forward with the fused MaxPool and the BatchNorm statistics."""
    dev = x.device
    B, Cout = x.shape[0], wq.shape[0]
    g = ConvGeom(B, 3, 32, 32, Cout, 5, 5, 1, 0)
    a = ConvFwdArgs()
    a.g = g
    a.x, a.w_eff, a.w_raw = x.data_ptr(), wq.data_ptr(), w_raw.data_ptr()
    pooled = torch.empty(B, Cout, 14, 14, device=dev)
    arg = torch.empty(B, Cout, 14, 14, dtype=torch.uint8, device=dev)
    a.pooled_out, a.argmax_out = pooled.data_ptr(), arg.data_ptr()
    a.noise_mode, a.current, a.scale_dev, a.rng = NOISE_MERGED, 1.0, scale.data_ptr(), ops._fixed_rng(3, 9)
    a.precision, a.a_code_scale, a.w_code_scale = PREC_BF16, s_a, 1.0 / 15.0
    ws = torch.empty(int(lib.nn_conv_workspace_bytes(C.byref(g), PREC_BF16)) + 4096, dtype=torch.uint8, device=dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    mean, invstd = torch.empty(Cout, device=dev), torch.empty(Cout, device=dev)
    rm, rv = torch.zeros(Cout, device=dev), torch.ones(Cout, device=dev)
    scratch = torch.zeros(int(lib.nn_conv_bn_scratch_bytes(Cout)), dtype=torch.uint8, device=dev)
    a.bn_mean, a.bn_invstd, a.bn_running_mean, a.bn_running_var = mean.data_ptr(), invstd.data_ptr(), rm.data_ptr(), rv.data_ptr()
    a.bn_eps, a.bn_momentum, a.bn_eval_mode, a.bn_scratch = 1e-5, 0.1, 0, scratch.data_ptr()
    _lib.check(lib.nn_noisy_conv_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream), "nn_noisy_conv_fwd")
    torch.cuda.synchronize()


def main():
    dev = torch.device("cuda:0")
    lib = _lib.load()
    props = torch.cuda.get_device_properties(0)
    us = 1e3 / props.clock_rate             # clock_rate: kHz
    print("card: %s, SM clock %.0f MHz" % (props.name, props.clock_rate / 1e3))
    s_a = 1.0 / 15.0
    x = torch.randint(0, 16, (512, 3, 32, 32), device=dev).float() * s_a
    w_raw = torch.randn(65, 3, 5, 5, device=dev) * 0.1
    wq = ops.quantize_fwd(w_raw, 4, -1.0, 1.0, 0.0)
    scale = ops.tensor_stats(w_raw)[1:2]
    kw = dict(precision="bf16", a_code_scale=s_a, w_code_scale=1.0 / 15.0)
    runs = (("pooled noisy (the benchmarked launch)", lambda: pooled_fwd(lib, x, wq, w_raw, scale, s_a)),
            ("noisy", lambda: ops.noisy_conv_fwd(x, wq, w_raw, None, 1, 0, noise_mode=NOISE_MERGED, current=1.0, scale_dev=scale,
                                                 want_y=False, **kw)),
            ("plain", lambda: ops.noisy_conv_fwd(x, wq, None, None, 1, 0, noise_mode=NOISE_NONE, **kw)))
    max_ctas = props.multi_processor_count
    for name, fn in runs:
        for _ in range(2):
            fn()
        rows = max_ctas * 32 * STAMPS // 8
        buf = np.zeros((rows, 8), dtype=np.int64)
        n = lib.nn_debug_cta_timeline(buf.ctypes.data_as(C.c_void_p), rows)
        if n <= 0:
            raise SystemExit("no stamps: build the library with NN_EXTRA_NVCC=-DNN_KDEBUG")
        t = buf[:n].reshape(-1, 32, STAMPS).astype(np.float64)
        ok = t[:, :, 4] > 0
        print("%s: %d CTAs x %.1f tiles (first 32 tiles of each CTA stamped)" % (name, t.shape[0], ok.sum() / t.shape[0]))
        # the two MMA warpgroups run independently: warpgroup 0 from the A stage it waited for to its store, warpgroup 1
        # from store to store
        rows_out = [("MMA warpgroup 0: A ready -> half 0 stored", t[:, :, 1] - t[:, :, 0], ok),
                    ("MMA warpgroup 1: half 1 stored, tile to tile", np.diff(t[:, :, 2], axis=1), ok[:, 1:])]
        for h, (seen, done) in enumerate(((3, 4), (5, 6))):
            rows_out.append(("epilogue half %d: wait for accumulators" % h, t[:, 1:, seen] - t[:, :-1, done], ok[:, 1:]))
            rows_out.append(("epilogue half %d: accumulators seen -> done" % h, t[:, :, done] - t[:, :, seen], ok))
        rows_out.append(("tile period (half 0 epilogue end to end)", np.diff(t[:, :, 4], axis=1), ok[:, 1:]))
        for lab, a, m in rows_out:
            a = a[m] * us
            print("   %-44s mean %6.2f us  p10 %6.2f  p90 %6.2f" % (lab, a.mean(), np.percentile(a, 10), np.percentile(a, 90)))
        span = (t[:, :, 4].max(axis=1) - t[:, 0, 0]) * us
        print("   CTA span mean %.1f us max %.1f us" % (span.mean(), span.max()))
    assert ops.error_flag() == 0


if __name__ == "__main__":
    main()
