#!/usr/bin/env python
"""Step time of SlowMo (--slowmo-period tau) against decent and Gossip-PGA with R virtual ranks on ONE GPU.

    python benchmarks/slowmo_step.py [--worlds 4,8] [--period 4] [--cycles 30] [--repeats 2] [--model resnet18]
                                     [--out file]

Every virtual rank runs ResNet-18 `ref` with SGD momentum 0.9 on its own stream, against the other virtual ranks'
windows in the same HBM, on the ring.  Four variants, alternated, --repeats times each:
  decent      the fused single-slot + ack step (csrc/gossip.cu), no gated launch;
  pga         --global-avg-period tau: the gated two-shot all-reduce of theta (csrc/allreduce.cu) before the step kernel;
  slowmo_h1   --slowmo-period tau, gossip base: the gated SlowMo sync kernel (average + outer update of x and u) before
              the same step kernel;
  slowmo_ht   --slowmo-period tau --local-steps tau, local-SGD base: the gated sync kernel before the serial step.
The timed region is one step of all R ranks (CUDA events around the launches, after warm-up).  Reported: the median
time of the base steps and of the sync (or averaging) steps separately, with the bytes one rank sends per step of each
kind.  These are single-GPU, HBM-bound numbers: pushes, peer loads and broadcasts land in the same GPU's memory, so they
say what the sync costs in kernels, not what NVLink would take.  The header holds the card's name, power limit and
maximum SM clock, read in the same run.
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

VARIANTS = ("decent", "pga", "slowmo_h1", "slowmo_ht")


def run(R: int, variant: str, tau: int, model: str, cycles: int, warmup_cycles: int) -> dict:
    kw = {"decent": {}, "pga": dict(global_avg_period=tau), "slowmo_h1": dict(slowmo_period=tau),
          "slowmo_ht": dict(slowmo_period=tau, local_steps=tau)}[variant]
    cfg = TrainConfig(algo="decent", dataset="cifar10", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                      double_buffer=False, overlap_push=False, **kw).validate()
    C = ext()
    w = LocalWorld(cfg, R, lambda: build_model(model), grid_cap=max(1, C.gossip_max_grid(0) // R),
                   timeout_ns=20_000_000_000)
    assert all(not be.dbuf and not be.overlap for be in w.backends)
    t = w.arenas[0].table
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(t.n_padded, generator=g, device="cuda") * 1e-3 for _ in range(R)]
    cur = torch.cuda.current_stream()
    steps = (warmup_cycles + cycles) * tau
    base, sync = [], []
    synced = variant != "decent"
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
        if s > warmup_cycles * tau:
            (sync if synced and s % tau == 0 else base).append(a.elapsed_time(b) * 1e3)
    for be in w.backends:
        be.check_status()
    n_sync = steps // tau if synced else 0
    per_base = 0 if variant == "slowmo_ht" else 2 * 4 * t.n_elems
    assert w.backends[0].bytes_sent() == n_sync * 4 * t.n_elems + (steps - n_sync) * per_base
    assert int(w.backends[0].ar_ctr.item()) == n_sync
    res = {"variant": variant, "world": R, "period": tau, "model": model, "grid_per_rank": w.backends[0].grid,
           "steps_timed": len(base) + len(sync),
           "base_step_us": round(statistics.median(base), 1),
           "sync_step_us": round(statistics.median(sync), 1) if sync else None,
           "base_bytes_per_rank": per_base, "sync_bytes_per_rank": 4 * t.n_elems if synced else None}
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
             f"ring, momentum 0.9; decent, --global-avg-period {a.period}, --slowmo-period {a.period} with "
             f"--local-steps 1 and {a.period}, alternated"]
    print(lines[0], flush=True)
    for R in (int(x) for x in a.worlds.split(",")):
        for rep in range(a.repeats):
            for v in VARIANTS:
                res = run(R, v, a.period, a.model, a.cycles, a.warmup_cycles)
                res["repeat"] = rep
                res["gpu"] = info
                lines.append(json.dumps(res))
                print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
