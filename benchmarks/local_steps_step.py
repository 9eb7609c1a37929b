#!/usr/bin/env python
"""Step-kernel time of decent with periodic gossip (--local-steps H) with R virtual ranks on ONE GPU.

    python benchmarks/local_steps_step.py [--worlds 4,8] [--topologies ring,onepeer-exp] [--hs 2,4,8]
                                          [--cycles 40] [--repeats 2] [--model resnet18] [--out file]

Every virtual rank runs the fused single-slot + ack step (ring: csrc/gossip.cu; onepeer-exp: csrc/gossip_graph.cu) on
ResNet-18 `ref` with SGD momentum 0.9 on its own stream, against the other virtual ranks' windows in the same HBM.  With
--local-steps H only every H-th step pushes, waits and mixes; the others are the serial SGD step.  The timed region is
one step of all R ranks (CUDA events around the launches, after warm-up).  A cycle is H consecutive steps ending with a
gossip step; the reported time is the median over --cycles cycles of the mean step time within the cycle, next to the
bytes one rank sends per step (fanout * 4 * numel / H).  H = 1 (the same single-slot kernel, gossiping at every step) is
run before each other H, so every row has an alternated baseline.  `predicted` is the byte-count model of DESIGN §8:
4 * n_padded * (7 + 2 * msgs) bytes per step, with msgs = fanout at gossip steps and 0 at local steps, as a fraction of
the H = 1 step.  These are single-GPU, HBM-bound numbers: pushes land in the same GPU's memory, so they say what the
schedule saves in the kernel, not what NVLink would take.  The header holds the card's name, power limit and maximum SM
clock; each row the SM clock sampled after every timed step (NVML), all read in the same run.
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


def run(R: int, topology: str, H: int, model: str, cycles: int, warmup_cycles: int) -> dict:
    cfg = TrainConfig(algo="decent", dataset="cifar10", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                      double_buffer=False, overlap_push=False, topology=topology, local_steps=H).validate()
    C = ext()
    cap = min(C.gossip_max_grid(0), C.gossip_graph_max_grid(0))     # the same grid for every H and topology
    w = LocalWorld(cfg, R, lambda: build_model(model), grid_cap=max(1, cap // R), timeout_ns=20_000_000_000)
    assert all(be.local_steps == H and not be.dbuf and not be.overlap for be in w.backends)
    t = w.arenas[0].table
    fanout = getattr(w.backends[0].ring, "fanout", 2)
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(t.n_padded, generator=g, device="cuda") * 1e-3 for _ in range(R)]
    cur = torch.cuda.current_stream()
    times, clocks = [], []
    steps = (warmup_cycles + cycles) * H
    for s in range(steps):
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
        if s >= warmup_cycles * H:
            times.append(a.elapsed_time(b) * 1e3)
            clk = sm_clock_mhz()
            if clk is not None:
                clocks.append(clk)
    for be in w.backends:
        be.check_status()
    assert w.backends[0].bytes_sent() == (steps // H) * fanout * 4 * t.n_elems
    per_cycle = [statistics.fmean(times[i:i + H]) for i in range(0, len(times), H)]
    gossip = [times[i] for i in range(H - 1, len(times), H)]
    local = [x for i, x in enumerate(times) if i % H != H - 1]
    res = {"world": R, "topology": topology, "local_steps": H, "model": model, "grid_per_rank": w.backends[0].grid,
           "cycle_mean_step_us": round(statistics.median(per_cycle), 1),
           "gossip_step_us": round(statistics.median(gossip), 1),
           "local_step_us": round(statistics.median(local), 1) if local else None,
           "bytes_sent_per_rank_step": fanout * 4 * t.n_elems / H,
           "predicted_fraction": round((7 * H + 2 * fanout) / ((7 + 2 * fanout) * H), 4),
           "sm_clock_mhz": ({"median": statistics.median(clocks), "min": min(clocks), "max": max(clocks)}
                            if clocks else "not recorded")}
    w.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="4,8")
    ap.add_argument("--topologies", default="ring,onepeer-exp")
    ap.add_argument("--hs", default="2,4,8", help="periods compared with H = 1")
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--cycles", type=int, default=40)
    ap.add_argument("--warmup-cycles", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    lines = [f"# {info} (name, power limit, maximum SM clock); single GPU, R virtual ranks, HBM-bound (not NVLink); "
             "decent step of all R ranks, momentum 0.9, H = 1 alternated with every other H"]
    print(lines[0], flush=True)
    for R in (int(x) for x in a.worlds.split(",")):
        for topology in a.topologies.split(","):
            for rep in range(a.repeats):
                for H in (int(x) for x in a.hs.split(",")):
                    base = run(R, topology, 1, a.model, a.cycles * H, a.warmup_cycles * H)
                    res = run(R, topology, H, a.model, a.cycles, a.warmup_cycles)
                    res["vs_h1"] = round(res["cycle_mean_step_us"] / base["cycle_mean_step_us"], 4)
                    res["h1_step_us"] = base["cycle_mean_step_us"]
                    for row in (base, res):
                        row["repeat"] = rep
                        row["gpu"] = info
                        lines.append(json.dumps(row))
                        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
