#!/usr/bin/env python
"""Standalone timing of conv2's input gradient at the benchmark's batch: nn_noisy_conv_dgrad (k_conv_tma<2, 72>, one
im2col tile per pixel tile and tap) against nn_conv_dgrad_planes (k_dgrad_planes<72>, each grad_output image loaded once).

    python tools/bench_conv2_dgrad.py [--batch 512] [--launches 100] [--rounds 5]

Both run on the engine's operands: the NN_PACK_TMA dgrad image from nn_prepare_weights and NHWC bf16 grad_output images.
Eight distinct grad_output images (8 x 12.3 MB at batch 512, more than the 50 MB L2) are cycled through, so every launch
reads its operand from HBM as in the training step.  Each round times `--launches` back-to-back launches of one path with
CUDA events, alternating the two paths; prints the card, its power limit and SM clock, then per path the median and the
spread over rounds in microseconds per launch, and whether the two outputs are bit-identical.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv2_dgrad: needs a CUDA device")
    import __graft_entry__ as entry
    entry.build()
    from step_profile import card_info

    from noisynet_b200 import _lib
    from noisynet_b200._lib import PACK_TMA, PREC_BF16, ConvDgradArgs, ConvGeom, Rng, WPrepJob
    lib = _lib.load()
    dev = torch.device("cuda:0")
    B, Cin, H, Cout, k = args.batch, 65, 14, 120, 5
    geom = ConvGeom(B, Cin, H, H, Cout, k, k, 1, 0)
    assert lib.nn_conv_dgrad_pack_layout(C.byref(geom), PREC_BF16) == PACK_TMA and lib.nn_conv_dgrad_planes_ok(C.byref(geom))
    g = torch.Generator().manual_seed(0)
    w_raw = (torch.rand(Cout, Cin, k, k, generator=g) * 2 - 1).to(dev)
    codes = torch.zeros(w_raw.numel() + 16, dtype=torch.int8, device=dev)
    jobs = (WPrepJob * 1)()
    jb = jobs[0]
    jb.w_raw, jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.m_rows, jb.noise_mode, jb.want_wsum = w_raw.data_ptr(), Cout, Cin, k * k, 1, B * H * H, 0, 0
    jb.layout, jb.q_bits, jb.q_hi, jb.stochastic, jb.u_inject, jb.rng = PACK_TMA, 4, 1.0, 0.0, None, Rng(0, 0, None)
    jb.codes = codes.data_ptr()
    wbuf = torch.zeros(int(lib.nn_weight_pack_bytes(C.byref(jb))) + 1024, dtype=torch.uint8, device=dev)
    jb.packed_out = (wbuf.data_ptr() + 1023) // 1024 * 1024
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.nn_prepare_weights(jobs, 1, 0, st), "nn_prepare_weights")
    gyps = [(torch.randn(B, 10, 10, Cout, generator=g) * 1e-3).to(torch.bfloat16).to(dev) for _ in range(8)]
    gx = {p: torch.empty(B, Cin, H, H, device=dev) for p in ("old", "new")}
    ws = torch.empty(int(lib.nn_conv_workspace_bytes(C.byref(geom), PREC_BF16)) + 4096, dtype=torch.uint8, device=dev)
    calls = {}
    for path in ("old", "new"):
        lst = []
        for gyp in gyps:
            a = ConvDgradArgs()
            a.g, a.gy, a.w_eff, a.gx, a.precision, a.w_code_scale = geom, None, None, gx[path].data_ptr(), PREC_BF16, 1.0 / 15.0
            a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
            a.gy_packed, a.w_packed, a.w_packed_layout = gyp.data_ptr(), jb.packed_out, PACK_TMA
            lst.append(a)
        calls[path] = lst
    fn = {"old": lib.nn_noisy_conv_dgrad, "new": lib.nn_conv_dgrad_planes}

    def run(path, n):
        for i in range(n):
            rc = fn[path](C.byref(calls[path][i % len(gyps)]), 0, st)
            if rc:
                _lib.check(rc, path)

    for path in ("old", "new"):          # warm-up: module load, tensor-map encoders, shared-memory opt-in
        run(path, 10)
    torch.cuda.synchronize()
    t = {"old": [], "new": []}
    for _ in range(args.rounds):
        for path in ("old", "new"):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(path, args.launches)
            e1.record()
            e1.synchronize()
            t[path].append(e0.elapsed_time(e1) * 1e3 / args.launches)
    for path in ("old", "new"):          # the same input for both: compare the outputs
        fn[path](C.byref(calls[path][0]), 0, st)
    torch.cuda.synchronize()
    assert _lib.load().nn_debug_error_flag(0, 0) == 0
    card = card_info(0)
    flop = 2.0 * B * 256 * 72 * 128 * 25              # MMA work the planes kernel issues (four m64 blocks, padded K and N)
    out = {"card": card["name"], "power_limit": card["power_limit"], "sm_max_clock": card["sm_max_clock"], "batch": B,
           "launches_per_round": args.launches, "rounds": args.rounds, "bit_identical": bool(torch.equal(gx["old"], gx["new"]))}
    for path, name in (("old", "k_conv_tma<2, 72>"), ("new", "k_dgrad_planes<72>")):
        v = t[path]
        out[path] = {"kernel": name, "median_us": round(statistics.median(v), 2), "min_us": round(min(v), 2), "max_us": round(max(v), 2)}
    out["new"]["mma_tflops"] = round(flop / (out["new"]["median_us"] * 1e-6) / 1e12, 1)
    out["speedup"] = round(out["old"]["median_us"] / out["new"]["median_us"], 3)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
