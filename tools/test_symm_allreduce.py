#!/usr/bin/env python
"""Multi-GPU check of the symmetric-memory gradient all-reduce (csrc/nn_collective.cu), run under torchrun on one node:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 tools/test_symm_allreduce.py

Compares with NCCL's all-reduce on the same data (fp32 sums in a different order: rtol 1e-6), checks that every rank ends
with bit-identical sums, replays the exchange from a CUDA graph, and times both (CUDA events, max over ranks)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from noisynet_b200 import dp  # noqa: E402


class Toy(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Parameter(torch.zeros(390, 3000))
        self.b = torch.nn.Parameter(torch.zeros(120, 65, 5, 5))
        self.c = torch.nn.Parameter(torch.zeros(65, 3, 5, 5))
        self.d = torch.nn.Parameter(torch.zeros(10, 390))
        self.e = torch.nn.Parameter(torch.zeros(65))


def log(rank, msg):
    with open("symm_rank%d.log" % rank, "a") as f:          # per-rank progress log in the working directory
        f.write(msg + "\n")


def main():
    rank, world, local = dp.init_from_env()
    log(rank, "process group up")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    m = Toy().to(dev)
    red = dp.SymmGradAllReduce(m, world, early=[[m.a, m.d], [m.b]])
    log(rank, "reducer built: multicast=%s ranges=%s" % (hex(red._mc), red.ranges))
    ref = torch.empty_like(red.flat)
    ok = True
    for it in range(3):
        g = torch.Generator(device=dev).manual_seed(100 * it + rank)
        red.flat.copy_(torch.randn(red.flat.shape, generator=g, device=dev))
        ref.copy_(red.flat)
        dist.all_reduce(ref)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            red.start_early(0)
            red.start_early(1)
        torch.cuda.current_stream().wait_stream(side)
        red.all_reduce_sum_()
        log(rank, "iter %d launched" % it)
        torch.cuda.synchronize()
        log(rank, "iter %d done" % it)
        err = ((red.flat - ref).abs().max() / ref.abs().max()).item()
        gathered = [torch.empty_like(red.flat) for _ in range(world)]
        dist.all_gather(gathered, red.flat)
        same = all(torch.equal(gathered[0], t) for t in gathered)
        if rank == 0:
            print("iter %d: max rel err vs NCCL %.2e, identical on all ranks: %s, multicast: %s" % (it, err, same, bool(red._mc)))
        ok = ok and err < 1e-5 and same
    # CUDA graph replay + timing
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        red.all_reduce_sum_()
    nccl_graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(nccl_graph):
        dist.all_reduce(ref)
    for name, gr in (("symmetric-memory kernel", graph), ("NCCL all_reduce", nccl_graph)):
        for _ in range(5):
            gr.replay()
        dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            gr.replay()
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / 50], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            print("%-26s %d ranks, %.2f MB: %.1f us per all-reduce" % (name, world, red.nbytes / 1e6, 1e3 * t.item()))
    red.flat.fill_(1.0)
    graph.replay()
    torch.cuda.synchronize()
    ok = ok and bool((red.flat == float(world)).all())
    if rank == 0:
        print("RESULT", "ok" if ok else "FAILED", flush=True)
    dist.barrier()
    torch.cuda.synchronize()
    os._exit(0 if ok else 1)        # (tearing the symmetric-memory handles down with the process group can block at exit)


if __name__ == "__main__":
    main()
