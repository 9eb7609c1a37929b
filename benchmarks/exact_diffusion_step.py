#!/usr/bin/env python
"""Step-kernel time of the dense decent ring step: plain, with gradient tracking (--gradient-tracking) and with exact
diffusion (--exact-diffusion), with R virtual ranks on ONE GPU.

    python benchmarks/exact_diffusion_step.py [--worlds 4,8] [--modes plain,tracking,ed] [--model resnet18]
                                              [--repeats 2] [--out file]

Every virtual rank runs the fused ring step (ResNet-18 `ref` by default, SGD with momentum 0.9) on its own stream,
against the other virtual ranks' windows in the same HBM, at one persistent grid for all modes (the smallest of the
three kernels' co-resident grids).  `plain` is decent's single-slot + ack step (double_buffer off, the protocol the
tracking and exact-diffusion kernels also use); `tracking` is csrc/gossip_gt.cu; `ed` is csrc/gossip_ed.cu, which runs
the optimizer in the push stage (theta, psi, gradient and momentum in; momentum, psi, theta and two pushes out) and
mixes with a load-only pass (phi, L, R in; theta out).  The timed region is one step of all R ranks (CUDA events around
the launches, after warm-up); the median over --steps is reported with the bytes one rank sends per step (plain and ed:
2 * 4 * numel; tracking: 2 * 2 * 4 * numel).  --repeats alternates the modes (plain, tracking, ed, plain, ...).  These
are single-GPU, HBM-bound numbers: pushes land in the same GPU's memory, so they say what each variant costs the kernel,
not what NVLink would take.  The header holds the card's name, power limit and maximum SM clock; each row the SM clock
sampled after every timed step (NVML), all read in the same run.
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
from topology_step import gpu_info, sm_clock_mhz  # noqa: E402


def run(R: int, mode: str, model: str, steps: int, warmup: int) -> dict:
    tracking, ed = mode == "tracking", mode == "ed"
    cfg = TrainConfig(algo="decent", dataset="cifar10", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                      double_buffer=False, overlap_push=False, gradient_tracking=tracking,
                      exact_diffusion=ed).validate()
    C = ext()
    cap = min(C.gossip_max_grid(0), C.gossip_gt_max_grid(0), C.gossip_ed_max_grid(0))   # one grid for every mode
    w = LocalWorld(cfg, R, lambda: build_model(model), grid_cap=max(1, cap // R), timeout_ns=20_000_000_000)
    assert all(be.gt == tracking and be.ed == ed and not be.dbuf and not be.overlap for be in w.backends)
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
    sent = (2 if tracking else 1) * 2 * 4 * t.n_elems
    assert w.backends[0].bytes_sent() == sent * (warmup + steps)
    med = statistics.median(times)
    res = {"world": R, "mode": mode, "model": model, "grid_per_rank": w.backends[0].grid,
           "median_us": round(med, 1), "min_us": round(min(times), 1), "max_us": round(max(times), 1),
           "bytes_sent_per_rank_step": sent,
           "sm_clock_mhz": ({"median": statistics.median(clocks), "min": min(clocks), "max": max(clocks)}
                            if clocks else "not recorded")}
    w.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="4,8")
    ap.add_argument("--modes", default="plain,tracking,ed")
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    lines = [f"# {info} (name, power limit, maximum SM clock); single GPU, R virtual ranks, HBM-bound (not NVLink); "
             "decent ring step of all R ranks, momentum 0.9"]
    print(lines[0], flush=True)
    for R in (int(x) for x in a.worlds.split(",")):
        for rep in range(a.repeats):
            for mode in a.modes.split(","):
                res = run(R, mode, a.model, a.steps, a.warmup)
                res["repeat"] = rep
                res["gpu"] = info
                lines.append(json.dumps(res))
                print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
