#!/usr/bin/env python
"""Step-kernel time of the gossip graphs (parallel/topology.py) with R virtual ranks on ONE GPU.

    python benchmarks/topology_step.py [--worlds 4,8] [--topologies "ring;exp;onepeer-exp;1,2"] [--model resnet18]
                                       [--out file]

Every virtual rank runs the full decent step (push into every slot it feeds -> per-slot flags -> mix -> SGD with
momentum; onepeer-exp: push into the step's one out-slot -> its flags -> (theta + slot) / 2 -> SGD) on its own stream, against the other virtual ranks' windows in the same HBM.  The timed region is one step
of all R ranks (CUDA events around the launches, after warm-up); the median over --steps is reported with the bytes
the R kernels move:
    per rank 4 * n_padded * (7 + 2 * msgs):  theta read twice (push and mix), grad and momentum read, theta and
    momentum written, grad zeroed, one push store and one inbox load per message (msgs = 2|O| slots on a static graph,
    2 on the ring, 1 on onepeer-exp, whose rows average over its period: every step moves the same bytes).
These are single-GPU, HBM-bound numbers: pushes land in the same GPU's memory, so they say what the slot count costs
the kernel, not what NVLink would take.  The ring is run with its single-slot + ack protocol (double_buffer off), the
same protocol the graph kernel uses.  Each row records the SM clock the card reported during the timed steps (NVML,
sampled after every step; a power-limited card runs below its maximum clock), next to the card's name, power limit
and maximum clock in the header.
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
    """SM clock over NVML's last sample period (torch.cuda.clock_rate), or None when NVML is unavailable."""
    try:
        return int(torch.cuda.clock_rate())
    except Exception:     # noqa: BLE001
        return None


def run(R: int, topology: str, model: str, steps: int, warmup: int) -> dict:
    cfg = TrainConfig(algo="decent", dataset="mnist", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                      double_buffer=False, topology=topology).validate()
    C = ext()
    grid_cap = max(1, min(C.gossip_max_grid(0), C.gossip_graph_max_grid(0)) // R)   # all R grids co-resident
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
    graph = Graph.build(0, R, topology)
    msgs = graph.fanout
    nbytes = R * 4 * t.n_padded * (7 + 2 * msgs)
    med = statistics.median(times)
    w.close()
    return {"world": R, "topology": topology, "offsets": list(graph.offsets), "slots": graph.n_slots, "msgs": msgs,
            "model": model, "grid_per_rank": w.backends[0].grid, "median_us": round(med, 1),
            "min_us": round(min(times), 1), "max_us": round(max(times), 1), "bytes": nbytes,
            "GBps": round(nbytes / med / 1e3, 1),
            "sm_clock_mhz": ({"median": statistics.median(clocks), "min": min(clocks), "max": max(clocks)}
                             if clocks else "not recorded")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="4,8")
    ap.add_argument("--topologies", default="ring;exp;onepeer-exp;1,2", help="';'-separated topology names")
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    lines = [f"# {info} (name, power limit, maximum SM clock); single GPU, R virtual ranks, HBM-bound (not NVLink); decent step of all R ranks"]
    print(lines[0], flush=True)
    for R in (int(x) for x in a.worlds.split(",")):
        for topo in a.topologies.split(";"):
            res = run(R, topo, a.model, a.steps, a.warmup)
            res["gpu"] = info
            lines.append(json.dumps(res))
            print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
