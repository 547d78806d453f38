#!/usr/bin/env python
"""Per-kernel breakdown of the benchmarked training step (bench.py's flagship workload).

    python tools/step_profile.py [--steps 20] [--batch 512] [--variant q4] [--eager] [--trace FILE]

Builds the model exactly as bench.py does (engine flow, fused AdamW, tensor-core precision), captures the step in a CUDA
graph and replays it under torch.profiler with CUDA activities.  This run is only a profile: tracing slows the host, so
step times come from bench.py, not from here.  If the profiler reports no kernels inside the graph replays, eager engine
steps are profiled instead (--eager forces that).  Prints the card name and power limit, then one row per (kernel,
stream): launches and device time per step, and the share of the summed kernel time.
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402


def card_info(index):
    """Name, power limit and max SM clock of the card, read in the same process as the profile (NVML, then nvidia-smi)."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit": "not reported", "sm_max_clock": "not reported"}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        info["power_limit"] = "%.0f W" % (pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0)
        info["sm_max_clock"] = "%d MHz" % pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception:  # noqa: BLE001
        try:
            out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                 capture_output=True, text=True, timeout=30).stdout.strip()
            info["power_limit"], info["sm_max_clock"] = [v.strip() for v in out.split(",")]
        except Exception:  # noqa: BLE001
            pass
    return info


def kernel_table(trace_file, steps):
    """{(kernel name, stream): [launches, total us]} from a chrome trace written by torch.profiler."""
    with open(trace_file) as f:
        events = json.load(f)["traceEvents"]
    tab = collections.defaultdict(lambda: [0, 0.0])
    for e in events:
        if e.get("cat") == "kernel" and e.get("ph") == "X":
            k = (e["name"], e.get("args", {}).get("stream", -1))
            tab[k][0] += 1
            tab[k][1] += float(e["dur"])
    return {k: (n / steps, us / steps) for k, (n, us) in tab.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--variant", default="q4", choices=["q4", "fp"])
    ap.add_argument("--pool", type=int, default=24)
    ap.add_argument("--eager", action="store_true", help="profile eager engine steps instead of graph replays")
    ap.add_argument("--trace", default=None, help="also keep the chrome trace here")
    ap.add_argument("--json", default=None, help="write the table as JSON here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "step_profile.py needs a CUDA device"
    from noisynet_b200 import ops
    from noisynet_b200.engine import NoisyNetEngine

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = card_info(0)
    # bench.py's model construction (args namespace with the fields build_model reads)
    args = argparse.Namespace(variant=a.variant, flow="engine", optimizer="fused", graph=1, batch=a.batch)
    torch.manual_seed(0)
    precision = bench.pick_precision(argparse.Namespace(precision="auto"), dev)
    if precision != "bf16":
        raise SystemExit("the engine flow needs the tensor-core path (bf16)")
    model, _, opt = bench.build_model(args, dev, precision)
    B = a.batch
    gen = torch.Generator().manual_seed(1234)
    xs = [(torch.randint(0, 16, (B, 3, 32, 32), generator=gen).float() / 15).to(dev) for _ in range(a.pool)]
    ys = [torch.randint(0, 10, (B,), generator=gen).to(dev) for _ in range(a.pool)]
    sx, sy = torch.empty_like(xs[0]), torch.empty_like(ys[0])
    loss_out = torch.zeros((), device=dev)
    engine = NoisyNetEngine(model, B, opt=opt)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for s in range(3):
            loss_out.copy_(engine.train_step(xs[s], ys[s])[0])
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()

    graph = None
    if not a.eager:
        step_ctr = torch.zeros(1, dtype=torch.int64, device=dev)
        graph = torch.cuda.CUDAGraph()
        with ops.graph_rng(step_ctr, seed=0):
            with torch.cuda.graph(graph):
                loss_out.copy_(engine.train_step(sx, sy)[0])
                ops.rng_advance(step_ctr, 1)
        torch.cuda.synchronize()

    def run(i, g):
        if g is not None:
            sx.copy_(xs[i % a.pool], non_blocking=True)
            sy.copy_(ys[i % a.pool], non_blocking=True)
            g.replay()
        else:
            loss_out.copy_(engine.train_step(xs[i % a.pool], ys[i % a.pool])[0])

    def profiled(g):
        for i in range(5):
            run(i, g)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(a.steps):
                run(i, g)
            torch.cuda.synchronize()
        fd, path = tempfile.mkstemp(suffix=".json")
        os.close(fd)
        prof.export_chrome_trace(path)
        tab = kernel_table(path, a.steps)
        if a.trace:
            os.replace(path, a.trace)
        else:
            os.remove(path)
        return tab

    mode = "graph replay"
    tab = profiled(graph)
    if not any(not name.startswith("Memcpy") for name, _ in tab):
        mode = "eager (the profiler reported no kernels inside graph replays)"
        tab = profiled(None)
    elif graph is None:
        mode = "eager"
    assert ops.error_flag() == 0
    total = sum(us for _, us in tab.values())
    rows = sorted(tab.items(), key=lambda kv: -kv[1][1])
    print("card: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["sm_max_clock"]))
    print("workload: engine step, batch %d, %s, %s, %d profiled steps" % (B, a.variant, mode, a.steps))
    print("%-10s %-8s %-7s %-6s %s" % ("us/step", "launches", "share", "stream", "kernel"))
    for (name, stream), (n, us) in rows:
        print("%10.1f %8.2f %6.1f%% %6s %s" % (us, n, 100.0 * us / total, stream, name[:150]))
    print("%10.1f %8.2f %6.1f%%        sum of kernel time per step (streams overlap: not the step time)"
          % (total, sum(n for n, _ in tab.values()), 100.0))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card, "mode": mode, "batch": B, "variant": a.variant, "steps": a.steps,
                       "kernels": [{"name": k[0], "stream": k[1], "launches_per_step": n, "us_per_step": us}
                                   for k, (n, us) in rows]}, f, indent=1)


if __name__ == "__main__":
    main()
