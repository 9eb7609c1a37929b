#!/usr/bin/env python
"""Single-GPU micro-benchmark of the fused step kernel variants (self-loop ring: pushes land in
this GPU's own HBM), device-timed.  Also the command to profile with ncu."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.config import TrainConfig  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.ops.local_world import LocalWorld  # noqa: E402

MODES = {
    "sgd_only": dict(algo="cent"),
    "async_nofire": dict(algo="event", sync_mode="async", thres_type=0, constant=1e30, initial_comm_passes=0),
    "async_allfire": dict(algo="event", sync_mode="async", thres_type=0, constant=0.0),
    "sync_nofire": dict(algo="event", sync_mode="iter", thres_type=0, constant=1e30, initial_comm_passes=0),
    "sync_allfire": dict(algo="decent", sync_mode="iter"),
}


def run(mode, model, iters, grid_cap=0, **kw):
    cfg = TrainConfig(dataset="mnist", model=model, lr=1e-2, momentum=0.9, **MODES[mode]).validate()
    w = LocalWorld(cfg, 1, lambda: build_model(model), grid_cap=grid_cap, **kw)
    be = w.backends[0]
    for _ in range(5):
        be.step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        be.step()
    e1.record()
    torch.cuda.synchronize()
    be.check_status()
    ms = e0.elapsed_time(e1) / iters
    n = w.arenas[0].table.n_padded * 4
    streams = {"sgd_only": 6, "async_nofire": 8, "async_allfire": 10, "sync_nofire": 9, "sync_allfire": 11}[mode]
    out = {"mode": mode, "ms": ms, "grid": be.grid, "algorithmic_GBps": streams * n / ms / 1e6}
    w.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="all")
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    modes = list(MODES) if a.mode == "all" else [a.mode]
    res = []
    for m in modes:
        res.append(run(m, a.model, a.iters))
        print(json.dumps(res[-1]), flush=True)
    # copy baseline for calibration (same bytes as one stream pair)
    x = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
    y = torch.empty_like(x)
    for _ in range(3):
        y.copy_(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        y.copy_(x)
    e1.record()
    torch.cuda.synchronize()
    res.append({"mode": "torch_copy_256MB", "GBps": 2 * x.numel() * 4 * 20 / e0.elapsed_time(e1) / 1e6})
    print(json.dumps(res[-1]))
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
