#!/usr/bin/env python
"""Consensus under random pairwise matchings (--topology random-match) against the ring and onepeer-exp, on
label-skewed shards, on the CPU (gloo), no timing.

    torchrun --nproc-per-node R benchmarks/random_match_convergence.py [--steps 100] [--lr 0.02] [--out file]

Each rank trains MNIST `cnn2` on its own `--partition label` shard with constant-lr SGD, momentum 0.9, batch 32 per
rank, from the same seed, once per topology.  After --steps steps it reports, per run:
  consensus        sqrt(mean_r ||theta_r - theta_bar||^2) / ||theta_bar||, before the final average (the Trainer's
                   --consensus-every measurement)
  bytes_per_rank   what each rank sent (random-match: an idle rank of an odd R sends nothing that step)
  loss, avg_acc    the last step's loss per rank and the test accuracy of the averaged model
and, from the simulator in float64 with lr = 0 (pure mixing of random zero-mean parameters, 200 steps):
  mix_rate         the mean per-step ratio ||theta_{k+1} - theta_bar||^2 / ||theta_k - theta_bar||^2 (the deviation is
                   rescaled to its starting size after every step, so rounding never enters)
  theory           what theory gives for that ratio: lambda_2(W)^2 on the ring; lambda_2(E[W]) =
                   (R - 2) / (2 (R - 1)) (even R) or 1/2 (odd R) on random-match, where it is the expected ratio;
                   none for onepeer-exp (directed and time-varying)
"""
import argparse
import json
import os
import sys
import tempfile

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.config import preset  # noqa: E402
from eventgrad_b200.data import synthetic_source  # noqa: E402
from eventgrad_b200.engine.simulator import RingSimulator  # noqa: E402
from eventgrad_b200.engine.trainer import Trainer  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.parallel.arena import ParamArena  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

_LOGS = tempfile.TemporaryDirectory(prefix="consensus_logs_")
TOPOLOGIES = ("ring", "onepeer-exp", "random-match")


def train(a, env, topology: str) -> dict:
    n_train = 32 * a.steps * env.world
    cfg = preset("decent", device="cpu", backend="gloo", model="cnn2", batch_mode="per_rank", batch_size=32,
                 sampler="random", lr=a.lr, momentum=0.9, epochs=1, max_steps=a.steps, train_samples=n_train,
                 test_samples=a.test_samples, quiet=True, consensus_every=a.steps, log_dir=_LOGS.name,
                 partition="label", topology=topology, topology_seed=1)
    torch.manual_seed(0)
    tr = Trainer(cfg, env, train_source=synthetic_source("mnist", n_train),
                 test_source=synthetic_source("mnist", a.test_samples, train=False))
    tr.fit()
    sent, losses = [None] * env.world, [None] * env.world
    dist.all_gather_object(losses, float(tr.last_loss) if tr.last_loss is not None else float("nan"))
    dist.all_gather_object(sent, int(tr.backend.bytes_sent()))
    res = tr.finalize(evaluate=True)
    out = {"topology": topology, "world": env.world, "steps": tr.steps_done, "lr": a.lr,
           "consensus": round(res["consensus_before_final_average"], 6), "bytes_per_rank": sent,
           "loss": [round(x, 4) for x in losses],
           "avg_acc": round(float(res.get("test_acc", float("nan"))), 2) if env.rank == 0 else None}
    tr.close()
    return out


def mix_rate(topology: str, R: int, steps: int = 200) -> dict:
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    sim = RingSimulator(R, torch.zeros(t.n_padded, dtype=torch.float64), t, "decent", lr=0.0, serial_skip=False,
                        offsets=topology, topology_seed=1)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(R, t.n_padded, generator=g, dtype=torch.float64)
    sim.theta = [row.clone() for row in x - x.mean(0)]
    dev = lambda: float(sum(((th - torch.stack(sim.theta).mean(0)) ** 2).sum() for th in sim.theta))
    ratios, d = [], dev()
    for _ in range(steps):
        sim.step([torch.zeros(t.n_padded, dtype=torch.float64)] * R)
        d2 = dev()
        ratios.append(d2 / d)
        if d2 == 0.0:          # exact consensus (onepeer-exp at a power-of-two R): nothing left to contract
            break
        # mixing is linear: rescale the deviation back to its starting size, so 200 steps stay far above rounding
        mean = torch.stack(sim.theta).mean(0)
        sim.theta = [mean + (th - mean) * (d / d2) ** 0.5 for th in sim.theta]
    if topology == "ring":
        W = sim.mixing_matrix(1)
        theory = float(torch.linalg.eigvalsh(W).abs().sort().values[-2]) ** 2
    elif topology == "random-match":
        theory = (R - 2) / (2 * (R - 1)) if R % 2 == 0 else 0.5
    else:
        theory = None
    return {"mix_rate": round(sum(ratios) / len(ratios), 4), "theory": None if theory is None else round(theory, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--lr", type=float, default=0.02)
    ap.add_argument("--test-samples", type=int, default=1000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    env = init_distributed("cpu")
    rows = [train(a, env, topo) for topo in TOPOLOGIES]
    if env.rank == 0:
        for r in rows:
            r.update(mix_rate(r["topology"], env.world))
        lines = [json.dumps(r) for r in rows]
        print("\n".join(lines), flush=True)
        if a.out:
            open(a.out, "w").write("\n".join(lines) + "\n")
    shutdown()


if __name__ == "__main__":
    main()
