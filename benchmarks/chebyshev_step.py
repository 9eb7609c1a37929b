#!/usr/bin/env python
"""Decent step time with Q Chebyshev-accelerated gossip rounds (--gossip-accel chebyshev) against Q power rounds
(--gossip-rounds Q alone), with R virtual ranks on ONE GPU.

    python benchmarks/chebyshev_step.py [--worlds 4,8] [--topologies "ring;exp"] [--rounds 1,2,3] [--runs 2]
                                        [--model resnet18] [--steps 100] [--out file]

power:     the Q - 1 round kernels (csrc/gossip_rounds.cu), then the step kernel with its own push and mix (the
           double-buffered ring step, or the graph step on exp).
chebyshev: Q Chebyshev round kernels (the same handshake, plus the `prev` read / write and the combine), then the
           serial step kernel (no push, no mix, no handshake).
Both with momentum 0.9, each rank on its own stream against the other virtual ranks' windows in the same HBM.  The
timed region is one step of all R ranks (CUDA events around the launches, after warm-up); the median over --steps is
reported.  For every Q the two modes run back to back, and the whole sweep runs --runs times, reversing the order of Q
values and of modes on every other run, so drift of the card's clock over the session shows as a difference between
runs, not between modes.  Bytes per rank are counted here, not read from the backend: Q * slots * 4 * n_elems per step
in both modes.
These are single-GPU, HBM-bound numbers: pushes land in the same GPU's memory, so they say what a round costs the
kernels, not what NVLink would take.  Each row records the SM clock sampled after every timed step, next to the
card's name, power limit and maximum SM clock in the header.
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
from eventgrad_b200.parallel.topology import Graph  # noqa: E402


def gpu_info() -> str:
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:     # noqa: BLE001
        return f"unknown ({e})"


def sm_clock_mhz():
    try:
        return int(torch.cuda.clock_rate())
    except Exception:     # noqa: BLE001
        return None


def run(R: int, topology: str, Q: int, accel: str, model: str, steps: int, warmup: int) -> dict:
    cfg = TrainConfig(algo="decent", dataset="cifar10", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                      overlap_push=False, topology=topology, gossip_rounds=Q, gossip_accel=accel).validate()
    C = ext()
    grid_cap = max(1, min(C.gossip_max_grid(0), C.gossip_dbuf_max_grid(0), C.gossip_graph_max_grid(0),
                          C.gossip_rounds_max_grid(0)) // R)          # all R grids co-resident (both round instances)
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
            times.append(a.elapsed_time(b))
            clk = sm_clock_mhz()
            if clk is not None:
                clocks.append(clk)
    for be in w.backends:
        be.check_status()
    graph = Graph.build(0, R, w.cfg.topology)
    per_rank = Q * graph.fanout * 4 * t.n_elems
    be = w.backends[0]
    kernel = ("serial" if be.cs is not None else "graph" if be.graph is not None else "dbuf" if be.dbuf else "ring")
    med = statistics.median(times)
    w.close()
    return {"world": R, "topology": topology, "offsets": list(graph.offsets), "slots": graph.n_slots, "Q": Q,
            "accel": accel, "step_kernel": kernel, "model": model, "grid_per_rank": grid_cap, "median_ms": round(med, 3),
            "min_ms": round(min(times), 3), "max_ms": round(max(times), 3), "bytes_per_rank_per_step": per_rank,
            "sm_clock_mhz": ({"median": statistics.median(clocks), "min": min(clocks), "max": max(clocks)}
                             if clocks else "not recorded")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="4,8")
    ap.add_argument("--topologies", default="ring;exp", help="';'-separated topology names")
    ap.add_argument("--rounds", default="1,2,3")
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    lines = [f"# {info} (name, power limit, maximum SM clock); single GPU, R virtual ranks, HBM-bound (not NVLink); "
             "decent step of all R ranks: Q power rounds (Q - 1 round kernels + the step's mix) against Q Chebyshev "
             "round kernels + the serial step"]
    print(lines[0], flush=True)
    qs = [int(x) for x in a.rounds.split(",")]
    for R in (int(x) for x in a.worlds.split(",")):
        for topo in a.topologies.split(";"):
            for run_i in range(a.runs):
                fwd = run_i % 2 == 0
                for Q in (qs if fwd else qs[::-1]):
                    for accel in (("none", "chebyshev") if fwd else ("chebyshev", "none")):
                        res = run(R, topo, Q, accel, a.model, a.steps, a.warmup)
                        res["run"] = run_i
                        lines.append(json.dumps(res))
                        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
