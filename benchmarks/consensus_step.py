#!/usr/bin/env python
"""Step time with the consensus distance measured every N steps (--consensus-every N) against N = 0.

    python benchmarks/consensus_step.py [--worlds 2,4,8] [--every 0,1,100] [--steps 200] [--repeats 2]
                                        [--model resnet18] [--out file]

LocalWorld: every virtual rank runs ResNet-18 `ref` (the arena of the flagship step) with SGD momentum 0.9 on its own
stream, decent on the ring with the fused single-slot step, against the other virtual ranks' windows in the same HBM.
The variants N = 0 (no consensus kernel), N = 1 (a measurement after every step) and N = 100 are alternated, --repeats
times each.  The timed region is one step of all R ranks (CUDA events around the launches, after warm-up).  Reported:
the median and mean step time over all steps, and the median over the measuring steps alone.  These are single-GPU,
HBM-bound numbers: the peer loads of the measurement land in the same GPU's memory, so they say what the kernel costs,
not what NVLink would take.

With two or more GPUs the script then runs itself under torchrun with one rank per GPU (the p2p backend over NVLink)
and times the same variants there.  The header holds the card's name, power limit and maximum SM clock, read in the
same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.config import TrainConfig  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.ops import ext  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from topology_step import gpu_info  # noqa: E402

WARMUP = 20


def _cfg(N: int, model: str) -> TrainConfig:
    return TrainConfig(algo="decent", dataset="cifar10", model=model, lr=1e-3, momentum=0.9, sync_mode="iter",
                       double_buffer=False, overlap_push=False, consensus_every=N).validate()


def _summary(times, measuring, N, R, model, grid, where):
    meas = [t for t, m in zip(times, measuring) if m]
    return {"where": where, "every": N, "world": R, "model": model, "grid_per_rank": grid, "steps_timed": len(times),
            "median_step_us": round(statistics.median(times), 1), "mean_step_us": round(statistics.fmean(times), 1),
            "median_measuring_step_us": round(statistics.median(meas), 1) if meas else None}


def run_local(R: int, N: int, model: str, steps: int) -> dict:
    from eventgrad_b200.ops.local_world import LocalWorld
    C = ext()
    w = LocalWorld(_cfg(N, model), R, lambda: build_model(model), grid_cap=max(1, C.gossip_max_grid(0) // R),
                   timeout_ns=20_000_000_000)
    t = w.arenas[0].table
    for be in w.backends:
        be.set_consensus_capacity(steps + WARMUP)
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(t.n_padded, generator=g, device="cuda") * 1e-3 for _ in range(R)]
    cur = torch.cuda.current_stream()
    times, measuring = [], []
    for s in range(1, WARMUP + steps + 1):
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
        if s > WARMUP:
            times.append(a.elapsed_time(b) * 1e3)
            measuring.append(bool(N) and s % N == 0)
    for be in w.backends:
        be.check_status()
    rows = w.backends[0].drain_consensus()
    assert len(rows) == ((WARMUP + steps) // N if N else 0)
    res = _summary(times, measuring, N, R, model, w.backends[0].grid, "localworld")
    w.close()
    return res


def run_torchrun_rank(a) -> None:
    """One rank per GPU: the p2p backend over peer-mapped memory, the variants alternated in one process group."""
    from eventgrad_b200.parallel import ParamArena, Ring
    from eventgrad_b200.parallel.p2p import P2PBackend, preallocate_arena_buffers
    from eventgrad_b200.utils.dist import init_distributed, shutdown
    env = init_distributed("cuda")
    lines = []
    for rep in range(a.repeats):
        for N in (int(x) for x in a.every.split(",")):
            cfg = _cfg(N, a.model)
            torch.manual_seed(0)
            model = build_model(a.model)
            theta, grad, symm = preallocate_arena_buffers(model, cfg, env)
            arena = ParamArena(model, env.device, theta=theta, grad=grad)
            be = P2PBackend(cfg, arena, Ring(env.rank, env.world), env, symm=symm)
            be.set_consensus_capacity(a.steps + WARMUP)
            grad.copy_(torch.randn_like(grad) * 1e-3)
            cur = torch.cuda.current_stream()
            times, measuring = [], []
            for s in range(1, WARMUP + a.steps + 1):
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record(cur)
                be.launch()
                be.account_step()
                ev1.record(cur)
                ev1.synchronize()
                if s > WARMUP:
                    times.append(ev0.elapsed_time(ev1) * 1e3)
                    measuring.append(bool(N) and s % N == 0)
            be.check_status()
            res = _summary(times, measuring, N, env.world, a.model, be.grid, "torchrun")
            res["repeat"] = rep
            lines.append(json.dumps(res))
            be.close()
            torch.distributed.barrier()
    if env.rank == 0:
        print("\n".join(lines), flush=True)
    shutdown()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="2,4,8")
    ap.add_argument("--every", default="0,1,100")
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default="")
    ap.add_argument("--rank-worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    if a.rank_worker:
        return run_torchrun_rank(a)
    info = gpu_info()
    lines = [f"# {info} (name, power limit, maximum SM clock); decent on the ring, fused single-slot step, momentum "
             f"0.9; --consensus-every {a.every} alternated; LocalWorld rows are single-GPU and HBM-bound"]
    print(lines[0], flush=True)
    for R in (int(x) for x in a.worlds.split(",")):
        for rep in range(a.repeats):
            for N in (int(x) for x in a.every.split(",")):
                res = run_local(R, N, a.model, a.steps)
                res["repeat"] = rep
                res["gpu"] = info
                lines.append(json.dumps(res))
                print(lines[-1], flush=True)
    n = torch.cuda.device_count()
    if n >= 2:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
               "--master-addr", "127.0.0.1", "--master-port", "31877", os.path.abspath(__file__), "--rank-worker",
               "--every", a.every, "--model", a.model, "--steps", str(a.steps), "--repeats", str(a.repeats)]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
        for line in r.stdout.splitlines():
            if line.startswith("{"):
                lines.append(line)
                print(line, flush=True)
        if r.returncode != 0:
            print(r.stderr[-3000:], file=sys.stderr, flush=True)
    else:
        lines.append(f"# torchrun rows skipped: {n} GPU")
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
