#!/usr/bin/env python
"""Step time of decent with periodic global averaging (--global-avg-period P) with R virtual ranks on ONE GPU.

    python benchmarks/global_avg_step.py [--worlds 4,8] [--period 4] [--cycles 30] [--repeats 2] [--model resnet18]
                                         [--out file]

Every virtual rank runs ResNet-18 `ref` with SGD momentum 0.9 on its own stream, against the other virtual ranks'
windows in the same HBM.  Two variants, alternated, --repeats times each:
  plain  decent on the ring, the fused single-slot + ack step (csrc/gossip.cu), no gated launch;
  pga    the same step kernel with --global-avg-period P, preceded at EVERY step by the gated two-shot all-reduce of
         theta (csrc/allreduce.cu): a no-op launch at gossip steps, the average at every P-th step.
The timed region is one step of all R ranks (CUDA events around the launches, after warm-up).  Reported: the median
step time of plain, and of pga's gossip steps and averaging steps separately, with the bytes one rank sends per step of
each kind.  These are single-GPU, HBM-bound numbers: the pushes and the all-reduce's peer loads and broadcasts land in
the same GPU's memory, so they say what the average costs in kernels, not what NVLink would take.  The header holds
the card's name, power limit and maximum SM clock, read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.config import TrainConfig  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.ops import ext  # noqa: E402
from eventgrad_b200.ops.local_world import LocalWorld  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from topology_step import gpu_info  # noqa: E402


def run(R: int, P: int, model: str, cycles: int, warmup_cycles: int) -> dict:
    cfg = TrainConfig(algo="decent", dataset="cifar10", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                      double_buffer=False, overlap_push=False, global_avg_period=P).validate()
    C = ext()
    w = LocalWorld(cfg, R, lambda: build_model(model), grid_cap=max(1, C.gossip_max_grid(0) // R),
                   timeout_ns=20_000_000_000)
    assert all(be.global_avg_period == P and not be.dbuf and not be.overlap for be in w.backends)
    t = w.arenas[0].table
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(t.n_padded, generator=g, device="cuda") * 1e-3 for _ in range(R)]
    cur = torch.cuda.current_stream()
    period = P or 1
    steps = (warmup_cycles + cycles) * period
    gossip, avg = [], []
    for s in range(1, steps + 1):
        for r in range(R):
            w.arenas[r].grad.copy_(grads[r])
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for st in w.streams:
            st.wait_stream(cur)
        a.record(cur)
        for st in w.streams:
            st.wait_event(a)
        for r in range(R):
            with torch.cuda.stream(w.streams[r]):
                w.backends[r].launch()
            w.backends[r].account_step()
        for st in w.streams:
            cur.wait_stream(st)
        b.record(cur)
        b.synchronize()
        if s > warmup_cycles * period:
            (avg if P and s % P == 0 else gossip).append(a.elapsed_time(b) * 1e3)
    for be in w.backends:
        be.check_status()
    n_avg = steps // P if P else 0
    assert w.backends[0].bytes_sent() == (n_avg + (steps - n_avg) * 2) * 4 * t.n_elems
    res = {"variant": "pga" if P else "plain", "world": R, "period": P, "model": model,
           "grid_per_rank": w.backends[0].grid, "steps_timed": len(gossip) + len(avg),
           "gossip_step_us": round(statistics.median(gossip), 1),
           "average_step_us": round(statistics.median(avg), 1) if avg else None,
           "gossip_bytes_per_rank": 2 * 4 * t.n_elems, "average_bytes_per_rank": 4 * t.n_elems if P else None}
    w.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="4,8")
    ap.add_argument("--period", type=int, default=4)
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--cycles", type=int, default=30)
    ap.add_argument("--warmup-cycles", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    lines = [f"# {info} (name, power limit, maximum SM clock); single GPU, R virtual ranks, HBM-bound (not NVLink); "
             f"ring, momentum 0.9; plain decent alternated with --global-avg-period {a.period}"]
    print(lines[0], flush=True)
    for R in (int(x) for x in a.worlds.split(",")):
        for rep in range(a.repeats):
            for P in (0, a.period):
                # the same number of timed steps for both variants
                res = run(R, P, a.model, a.cycles * (a.period if P == 0 else 1),
                          a.warmup_cycles * (a.period if P == 0 else 1))
                res["repeat"] = rep
                res["gpu"] = info
                lines.append(json.dumps(res))
                print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
