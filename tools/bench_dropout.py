"""Step time of training with dropout (--dropout p, noisynet.py:375-376) on the engine and on the module path.

    python tools/bench_dropout.py [--steps 40] [--warmup 5] [--rounds 3] [--out DIR]

Measures, on one GPU, with the card's name and power limit read in the same run:
  (a) the benchmarked configuration (batch 512, full widths, q_a = q_w = 4, I = 1 nA, act_max 5) on the engine, captured as
      one CUDA graph, at p = 0 and at p = 0.1 with --dropout_conv: what the dropout sites cost;
  (b) the README's noise-free baseline (--L2 0.0005 --dropout 0.1: q = 0, I = 0, act_max = 0) at batch 64 (the script's
      default) and 512, on the engine (CUDA graph) and on NoisyNet(fused=True) with autograd and torch.nn.Dropout (eager).
Each configuration is timed with device events over --steps steps after --warmup steps; the configurations are run in
turn, --rounds times, so drift on a shared card spreads over all of them.  Prints one JSON object (and writes it to
DIR/bench_dropout.json with --out).
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def make(cfg, B, dev):
    from noisynet_b200.engine import NoisyNetEngine
    from noisynet_b200.net import NoisyNet, default_args, init_like_reference, make_fused_optimizer, with_quant
    if cfg["name"].startswith("bench"):
        a = with_quant(default_args(dropout=cfg["p"], dropout_conv=cfg["p"]), 4, 4)
    else:       # README noise-free baseline
        a = default_args(dropout=0.1, act_max=0.0, act_max1=0.0, act_max2=0.0, act_max3=0.0, layer_currents=[0.0] * 4,
                         current1=0.0, current2=0.0, current3=0.0, current4=0.0, L2_1=5e-4, L2_2=5e-4, L2_3=5e-4, L2_4=5e-4)
    torch.manual_seed(0)
    m = init_like_reference(NoisyNet(a, fused=True, precision="bf16")).to(dev)
    if a.q_a2 > 0:
        m.quantize2.running_max = torch.tensor(5.0, device=dev)
        m.quantize4.running_max = torch.tensor(5.0, device=dev)
    m.collect_stats = False
    m.train()
    opt = make_fused_optimizer(m, a)
    gen = torch.Generator().manual_seed(4321)
    xs = [(torch.randint(0, 16, (B, 3, 32, 32), generator=gen).float() / 15).to(dev) for _ in range(4)]
    ys = [torch.randint(0, 10, (B,), generator=gen).to(dev) for _ in range(4)]
    loss_out = torch.zeros((), device=dev)
    keep_alive = [m, opt, xs, ys]       # a captured graph replays into these buffers: they must outlive it
    if cfg["flow"] == "engine":
        from noisynet_b200 import ops
        eng = NoisyNetEngine(m, B, opt=opt)
        sx, sy = torch.empty_like(xs[0]), torch.empty_like(ys[0])
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for s in range(3):
                eng.train_step(xs[s], ys[s])
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        ctr = torch.zeros(1, dtype=torch.int64, device=dev)
        graph = torch.cuda.CUDAGraph()
        with ops.graph_rng(ctr, seed=99):
            with torch.cuda.graph(graph):
                loss_out.copy_(eng.train_step(sx, sy)[0])
                ops.rng_advance(ctr, 1)
        torch.cuda.synchronize()
        keep_alive += [eng, graph, sx, sy, ctr]

        def step(i):
            sx.copy_(xs[i % 4], non_blocking=True)
            sy.copy_(ys[i % 4], non_blocking=True)
            graph.replay()
    else:       # module path: fused noisy layers, torch pool / BN / ReLU / clamp / nn.Dropout, autograd
        from noisynet_b200.net import bind_absmax

        def step(i):
            out = m(xs[i % 4], 0, 100)
            loss = F.cross_entropy(out, ys[i % 4])
            opt.zero_grad()
            loss.backward()
            opt.step()
            bind_absmax(m, opt)
            loss_out.copy_(loss.detach())
    return step, loss_out, keep_alive


def time_steps(step, loss_out, keep_alive, steps, warmup):
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        step(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, loss_out.item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dropout: needs a CUDA device")
    import __graft_entry__ as entry
    entry.build()
    from noisynet_b200 import ops
    dev = torch.device("cuda:0")
    cfgs = [dict(name="bench_q4_I1_p0", flow="engine", B=512, p=0.0),
            dict(name="bench_q4_I1_p0.1_conv", flow="engine", B=512, p=0.1),
            dict(name="readme_baseline_B64_engine", flow="engine", B=64),
            dict(name="readme_baseline_B64_module", flow="module", B=64),
            dict(name="readme_baseline_B512_engine", flow="engine", B=512),
            dict(name="readme_baseline_B512_module", flow="module", B=512)]
    runners = {c["name"]: make(c, c["B"], dev) for c in cfgs}
    res = {c["name"]: [] for c in cfgs}
    loss = {}
    for _ in range(args.rounds):
        for c in cfgs:
            ms, lo = time_steps(*runners[c["name"]], args.steps, args.warmup)
            res[c["name"]].append(round(ms, 4))
            loss[c["name"]] = lo
    assert ops.error_flag() == 0
    out = {"card": card(), "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
           "ms_per_step": res, "ms_per_step_min": {k: min(v) for k, v in res.items()}, "last_loss": loss,
           "method": "device events around --steps steps; engine = one CUDA-graph replay per step, module = eager"}
    b0, b1 = out["ms_per_step_min"]["bench_q4_I1_p0"], out["ms_per_step_min"]["bench_q4_I1_p0.1_conv"]
    out["dropout_cost_bench_config"] = {"ms": round(b1 - b0, 4), "relative": round(b1 / b0 - 1.0, 4)}
    for B in (64, 512):
        e, mo = out["ms_per_step_min"]["readme_baseline_B%d_engine" % B], out["ms_per_step_min"]["readme_baseline_B%d_module" % B]
        out["readme_baseline_B%d_module_over_engine" % B] = round(mo / e, 3)
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_dropout.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
