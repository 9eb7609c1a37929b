#!/usr/bin/env python
"""Step time of decent with quasi-global momentum (--quasi-global-momentum) with R virtual ranks on ONE GPU.

    python benchmarks/qg_step.py [--steps 60] [--repeats 2] [--model resnet18] [--out file]

Every virtual rank runs ResNet-18 `ref` with momentum 0.9 on its own stream, against the other virtual ranks' windows in
the same HBM, at the persistent grid.  Three kernels: the single-slot ring (csrc/gossip.cu) at R = 4 and 8, the
double-buffered ring (gossip_dbuf) at R = 4 and 8, and `exp` (gossip_graph, offsets 1, 2, 4) at R = 8.  Each is run as
plain heavy-ball decent and with --quasi-global-momentum, alternated, --repeats times each.  The timed region is one step
of all R ranks (CUDA events around the launches, after warm-up); reported are the median step time and the bytes one
rank sends per step.  Single-GPU, HBM-bound numbers: they say what the QG update costs in the step kernel, not what
NVLink would take.  The header holds the card's name, power limit and maximum SM clock, read in the same run.
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

KERNELS = (("ring", 4, "ring", False), ("ring", 8, "ring", False), ("dbuf", 4, "ring", True),
           ("dbuf", 8, "ring", True), ("exp", 8, "exp", False))


def run(kind: str, R: int, topology: str, dbuf: bool, qg: bool, model: str, steps: int, warmup: int) -> dict:
    cfg = TrainConfig(algo="decent", dataset="cifar10", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                      topology=topology, double_buffer=dbuf, overlap_push=False,
                      quasi_global_momentum=qg).validate()
    C = ext()
    grid = {"ring": C.gossip_max_grid, "dbuf": C.gossip_dbuf_max_grid, "exp": C.gossip_graph_max_grid}[kind](0)
    w = LocalWorld(cfg, R, lambda: build_model(model), grid_cap=max(1, grid // R), timeout_ns=20_000_000_000)
    be0 = w.backends[0]
    assert be0.qg == qg and be0.dbuf == dbuf and (be0.graph is not None) == (kind == "exp")
    t = w.arenas[0].table
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(t.n_padded, generator=g, device="cuda") * 1e-3 for _ in range(R)]
    cur = torch.cuda.current_stream()
    times = []
    for s in range(1, warmup + steps + 1):
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
        if s > warmup:
            times.append(a.elapsed_time(b) * 1e3)
    for be in w.backends:
        be.check_status()
    n = warmup + steps
    res = {"kernel": kind, "world": R, "topology": topology, "qg": qg, "model": model, "grid_per_rank": be0.grid,
           "steps_timed": len(times), "step_us": round(statistics.median(times), 1),
           "bytes_per_rank_step": be0.bytes_sent() // n}
    w.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    lines = [f"# {info} (name, power limit, maximum SM clock); single GPU, R virtual ranks, HBM-bound (not NVLink); "
             "decent, momentum 0.9; plain heavy ball alternated with --quasi-global-momentum"]
    print(lines[0], flush=True)
    for kind, R, topology, dbuf in KERNELS:
        for rep in range(a.repeats):
            for qg in (False, True):
                res = run(kind, R, topology, dbuf, qg, a.model, a.steps, a.warmup)
                res["repeat"] = rep
                res["gpu"] = info
                lines.append(json.dumps(res))
                print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
