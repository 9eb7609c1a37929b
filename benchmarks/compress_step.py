#!/usr/bin/env python
"""Step-kernel time of the ring without compression and with the int8 and sign codecs (--compress int8|sign), with and
without the CHOCO mix (--choco-gamma), with R virtual ranks on ONE GPU.

    python benchmarks/compress_step.py [--worlds 4,8] [--algos decent,event] [--modes none,int8,sign]
                                       [--choco-gamma 0,0.5] [--model resnet18] [--repeats 2] [--out file]

Every virtual rank runs the fused ring step (ResNet-18 `ref` by default, SGD with momentum) on its own stream, against
the other virtual ranks' windows in the same HBM.  event runs at a zero threshold (constant 0: every tensor fires every
step), so both algorithms send every tensor.  The dense ring runs its single-slot + ack protocol (double_buffer off), the
protocol the int8 kernel also uses.  The timed region is one step of all R ranks (CUDA events around the launches,
after warm-up); the median over --steps is reported with the bytes one rank sends per step, counted from the message
formula (dense: 2 * 4 * numel; int8: 2 * (numel + 4 * ceil(numel / 256)); sign: 2 * (ceil(numel / 8) +
4 * ceil(numel / 256)) per tensor).  Every compressed mode runs once per --choco-gamma value (0: the error-feedback
mix).  --repeats alternates the configurations (none, int8, sign, none, int8, sign, ...).  These are single-GPU, HBM-bound numbers: pushes land in the same GPU's memory, so they
say what the codec costs the kernel, not what NVLink would take.  The header holds the card's name, power limit and
maximum SM clock; each row the SM clock sampled after every timed step (NVML), all read in the same run.
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
from eventgrad_b200.parallel.trigger import codec_of  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from topology_step import gpu_info, sm_clock_mhz  # noqa: E402


def run(R: int, algo: str, compress: str, model: str, steps: int, warmup: int, gamma: float = 0.0) -> dict:
    cfg = TrainConfig(algo=algo, dataset="cifar10", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                      double_buffer=False, overlap_push=False, thres_type=0, constant=0.0, initial_comm_passes=0,
                      compress=compress, choco_gamma=gamma).validate()
    C = ext()
    cap = min(C.gossip_max_grid(0), C.gossip_q8_max_grid(0))
    w = LocalWorld(cfg, R, lambda: build_model(model), grid_cap=max(1, cap // R), timeout_ns=20_000_000_000)
    t = w.arenas[0].table
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(t.n_padded, generator=g, device="cuda") * 1e-3 for _ in range(R)]
    cur = torch.cuda.current_stream()
    times, clocks = [], []
    fired_all = True
    for s in range(warmup + steps):
        for r in range(R):
            w.arenas[r].grad.copy_(grads[r])
        if algo == "event" and s == warmup:
            fired_all = all(bool(be.fire.bool().all()) for be in w.backends)
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
    per_msg = [codec_of(compress)[2](n) if compress != "none" else 4 * n for n in t.numels]
    sent = 2 * sum(per_msg)
    med = statistics.median(times)
    res = {"world": R, "algo": algo, "compress": compress, "choco_gamma": gamma, "model": model, "grid_per_rank": w.backends[0].grid,
           "all_fired": fired_all, "median_us": round(med, 1), "min_us": round(min(times), 1),
           "max_us": round(max(times), 1), "bytes_sent_per_rank_step": sent,
           "sm_clock_mhz": ({"median": statistics.median(clocks), "min": min(clocks), "max": max(clocks)}
                            if clocks else "not recorded")}
    w.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="4,8")
    ap.add_argument("--algos", default="decent,event")
    ap.add_argument("--modes", default="none,int8,sign")
    ap.add_argument("--choco-gamma", default="0", help="comma list; each compressed mode runs once per value")
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    lines = [f"# {info} (name, power limit, maximum SM clock); single GPU, R virtual ranks, HBM-bound (not NVLink); "
             "ring step of all R ranks, every tensor fires"]
    print(lines[0], flush=True)
    for R in (int(x) for x in a.worlds.split(",")):
        for algo in a.algos.split(","):
            for rep in range(a.repeats):
                configs = [(mode, g) for mode in a.modes.split(",")
                           for g in ([0.0] if mode == "none" else [float(x) for x in a.choco_gamma.split(",")])]
                for mode, gamma in configs:
                    res = run(R, algo, mode, a.model, a.steps, a.warmup, gamma)
                    res["repeat"] = rep
                    res["gpu"] = info
                    lines.append(json.dumps(res))
                    print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
