#!/usr/bin/env python
"""Decent, decent with gradient tracking, decent with exact diffusion and decent with periodic global averaging on
label-sorted shards, on the CPU (gloo), no timing.

    torchrun --nproc-per-node 4 benchmarks/tracking_convergence.py [--steps 300] [--data synthetic|DIR] [--lr 0.05]
                                                                    [--global-avg-periods 4,16] [--out file]

Each rank trains MNIST `cnn2` on its own `--partition label` shard (the samples sorted by class, cut into R equal
blocks: each rank sees two or three of the ten classes) with constant-lr SGD, batch 32 per rank, once with plain
decent, once with --gradient-tracking, once with --exact-diffusion and once per --global-avg-period P in
--global-avg-periods (every P-th step an exact average over all ranks), from the same seed.  After --steps steps it
reports, per run:
  consensus   sqrt(mean_r ||theta_r - theta_bar||^2) / ||theta_bar||, before the final average
              (the Trainer's --consensus-every measurement, consensus_before_final_average)
  local_acc   the test accuracy of every rank's own model, before the final average
  avg_acc     the test accuracy of the averaged model
The default data is the project's synthetic MNIST (class templates plus noise), which may be too easy to separate the
algorithms; pass a dataset root with --data for the real set.
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
from eventgrad_b200.data import load_source, synthetic_source  # noqa: E402
from eventgrad_b200.engine.trainer import Trainer  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

# the Trainer's consensus.csv files: not wanted here, kept out of the working directory
_LOGS = tempfile.TemporaryDirectory(prefix="consensus_logs_")


def run(a, env, tracking: bool, ed: bool = False, P: int = 0) -> dict:
    n_train = 32 * a.steps * env.world          # one epoch of a.steps steps
    cfg = preset("decent", device="cpu", backend="gloo", model="cnn2", batch_mode="per_rank", batch_size=32,
                 sampler="random", partition="label", lr=a.lr, momentum=0.0, epochs=1, max_steps=a.steps,
                 train_samples=n_train, test_samples=a.test_samples, quiet=True, consensus_every=a.steps,
                 log_dir=_LOGS.name, gradient_tracking=tracking, exact_diffusion=ed, global_avg_period=P)
    if a.data == "synthetic":
        train, test = synthetic_source("mnist", n_train), synthetic_source("mnist", a.test_samples, train=False)
    else:
        train = load_source("mnist", a.data, n_train, True)
        test = load_source("mnist", a.data, a.test_samples, False)
    torch.manual_seed(0)
    tr = Trainer(cfg, env, train_source=train, test_source=test)
    classes = sorted(set(train.labels[tr.sampler.indices()].tolist()))
    tr.fit()
    local = float(tr.evaluate()["test_acc"])
    accs = [None] * env.world
    cls = [None] * env.world
    dist.all_gather_object(accs, local)
    dist.all_gather_object(cls, classes)
    res = tr.finalize(evaluate=True)
    consensus = res["consensus_before_final_average"]
    out = {"gradient_tracking": tracking, "exact_diffusion": ed, "global_avg_period": P, "world": env.world,
           "steps": tr.steps_done, "lr": a.lr, "data": a.data,
           "consensus": round(consensus, 6), "local_acc": [round(x, 2) for x in accs],
           "avg_acc": round(float(res.get("test_acc", float("nan"))), 2) if env.rank == 0 else None,
           "classes_per_rank": cls}
    tr.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--lr", type=float, default=0.05)
    ap.add_argument("--data", default="synthetic")
    ap.add_argument("--test-samples", type=int, default=2000)
    ap.add_argument("--global-avg-periods", default="4,16", help="comma-separated P of the global-averaging runs")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    env = init_distributed("cpu")
    runs = [(False, False, 0), (True, False, 0), (False, True, 0)]
    runs += [(False, False, int(P)) for P in a.global_avg_periods.split(",") if P]
    lines = [json.dumps(run(a, env, t, ed, P)) for t, ed, P in runs]
    if env.rank == 0:
        print("\n".join(lines), flush=True)
        if a.out:
            open(a.out, "w").write("\n".join(lines) + "\n")
    shutdown()


if __name__ == "__main__":
    main()
