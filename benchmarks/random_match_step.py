#!/usr/bin/env python
"""Step time of random pairwise matchings (--topology random-match) against the ring, exp and onepeer-exp, with R
virtual ranks on ONE GPU.

    python benchmarks/random_match_step.py [--worlds 4,6,8] [--topologies "ring;exp;onepeer-exp;random-match"]
                                           [--model resnet18] [--runs 2] [--out file]

Every virtual rank runs the full decent step (momentum 0.9, the ResNet-18 `ref` arena) on its own stream, against the
other virtual ranks' windows in the same HBM; the ring runs its single-slot + ack protocol, as in topology_step.py.
The timed region is one step of all R ranks (CUDA events, after warm-up); the median over --steps is reported with the
bytes each rank sent per step, as the backend counts them (random-match: an idle rank of an odd R sends nothing, so its
mean is below one copy).  The rows alternate between topologies, --runs times, so a slow phase of a shared host hits
all of them.  The header records the card's name, power limit and maximum SM clock, and every row the SM clock sampled
during its timed steps.  Single-GPU, HBM-bound numbers: not NVLink.
"""
import argparse
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from eventgrad_b200.config import TrainConfig  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.ops import ext  # noqa: E402
from eventgrad_b200.ops.local_world import LocalWorld  # noqa: E402
from topology_step import gpu_info, sm_clock_mhz  # noqa: E402


def run(R: int, topology: str, model: str, steps: int, warmup: int) -> dict:
    cfg = TrainConfig(algo="decent", dataset="mnist", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                      double_buffer=False, topology=topology, topology_seed=1).validate()
    C = ext()
    grid_cap = max(1, min(C.gossip_max_grid(0), C.gossip_graph_max_grid(0), C.gossip_match_max_grid(0)) // R)
    w = LocalWorld(cfg, R, lambda: build_model(model), grid_cap=grid_cap, timeout_ns=20_000_000_000)
    t = w.arenas[0].table
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(t.n_padded, generator=g, device="cuda") * 1e-3 for _ in range(R)]
    cur = torch.cuda.current_stream()
    times, clocks = [], []
    for s in range(warmup + steps):
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
        if s >= warmup:
            times.append(a.elapsed_time(b) * 1e3)
            clk = sm_clock_mhz()
            if clk is not None:
                clocks.append(clk)
    for be in w.backends:
        be.check_status()
    sent = sum(be.bytes_sent() for be in w.backends) / (R * (warmup + steps))
    med = statistics.median(times)
    grid = w.backends[0].grid
    w.close()
    return {"world": R, "topology": topology, "model": model, "grid_per_rank": grid, "median_us": round(med, 1),
            "min_us": round(min(times), 1), "max_us": round(max(times), 1),
            "bytes_per_rank_per_step": int(sent), "copies_per_rank_per_step": round(sent / (4 * t.n_elems), 3),
            "sm_clock_mhz": ({"median": statistics.median(clocks), "min": min(clocks), "max": max(clocks)}
                             if clocks else "not recorded")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="4,6,8")
    ap.add_argument("--topologies", default="ring;exp;onepeer-exp;random-match", help="';'-separated topology names")
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    lines = [f"# {info} (name, power limit, maximum SM clock); single GPU, R virtual ranks, HBM-bound (not NVLink); "
             "decent step of all R ranks"]
    print(lines[0], flush=True)
    for run_i in range(a.runs):
        for R in (int(x) for x in a.worlds.split(",")):
            for topo in a.topologies.split(";"):
                res = run(R, topo, a.model, a.steps, a.warmup)
                res.update({"run": run_i, "gpu": info})
                lines.append(json.dumps(res))
                print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
