#!/usr/bin/env python
"""decent with Chebyshev-accelerated gossip rounds (--gossip-accel chebyshev) against power rounds (--gossip-rounds Q) at
matched bytes, on label-skewed shards, on the CPU (gloo), no timing.

    torchrun --nproc-per-node 8 benchmarks/chebyshev_convergence.py [--steps 300] [--lr 0.02]
                                                                    [--data synthetic|DIR] [--out file]

Each rank trains MNIST `cnn2` on its own `--partition label` shard with constant-lr SGD, momentum 0.9, batch 32 per
rank, from the same seed (one seed per row): the ring with Q = 3, power and Chebyshev, and the exp graph (offsets
1, 2, 4 at R = 8) with Q = 1, power and Chebyshev.  At R = 8 all four send the same bytes per step (6 messages of the
whole model).  In theory (||M - 11^T/R||_2 at R = 8) the order is ring Chebyshev 0.177 < exp Chebyshev 0.404 < exp
power 0.429 < ring power 0.521.
After --steps steps it reports, per run:
  loss             the last training step's loss, per rank
  bytes_per_rank   what each rank sent
  consensus        sqrt(mean_r ||theta_r - theta_bar||^2) / ||theta_bar||, before the final average
                   (the Trainer's --consensus-every measurement, consensus_before_final_average)
  local_acc        the test accuracy of every rank's own model, before the final average
  avg_acc          the test accuracy of the averaged model
The default data is the project's synthetic MNIST (class templates plus noise), which is known to be too easy to
separate the algorithms by accuracy; the consensus distance is the quantity the rounds act on.  Pass a dataset root
with --data for the real set.
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


def run(a, env, name: str, **kw) -> dict:
    n_train = 32 * a.steps * env.world          # one epoch of a.steps steps
    cfg = preset("decent", device="cpu", backend="gloo", model="cnn2", batch_mode="per_rank", batch_size=32,
                 sampler="random", lr=a.lr, momentum=0.9, epochs=1, max_steps=a.steps, train_samples=n_train,
                 test_samples=a.test_samples, quiet=True, consensus_every=a.steps, log_dir=_LOGS.name,
                 partition="label", **kw)
    if a.data == "synthetic":
        train, test = synthetic_source("mnist", n_train), synthetic_source("mnist", a.test_samples, train=False)
    else:
        train = load_source("mnist", a.data, n_train, True)
        test = load_source("mnist", a.data, a.test_samples, False)
    torch.manual_seed(0)
    tr = Trainer(cfg, env, train_source=train, test_source=test)
    tr.fit()
    local = float(tr.evaluate()["test_acc"])
    accs = [None] * env.world
    sent = [None] * env.world
    losses = [None] * env.world
    dist.all_gather_object(losses, float(tr.last_loss) if tr.last_loss is not None else float("nan"))
    dist.all_gather_object(accs, local)
    dist.all_gather_object(sent, int(tr.backend.bytes_sent()))
    res = tr.finalize(evaluate=True)
    consensus = res["consensus_before_final_average"]
    out = {"run": name, "world": env.world, "steps": tr.steps_done, "lr": a.lr, "data": a.data,
           "loss": [round(x, 4) for x in losses], "bytes_per_rank": sent,
           "consensus": round(consensus, 6), "local_acc": [round(x, 2) for x in accs],
           "avg_acc": round(float(res.get("test_acc", float("nan"))), 2) if env.rank == 0 else None}
    tr.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--lr", type=float, default=0.02)
    ap.add_argument("--data", default="synthetic")
    ap.add_argument("--test-samples", type=int, default=2000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    env = init_distributed("cpu")
    runs = [("ring_Q3_power", dict(gossip_rounds=3)),
            ("ring_Q3_chebyshev", dict(gossip_rounds=3, gossip_accel="chebyshev")),
            ("exp_Q1_power", dict(topology="exp")),
            ("exp_Q1_chebyshev", dict(topology="exp", gossip_accel="chebyshev"))]
    rows = [run(a, env, name, **kw) for name, kw in runs]
    if env.rank == 0:
        lines = [json.dumps(r) for r in rows]
        print("\n".join(lines), flush=True)
        if a.out:
            open(a.out, "w").write("\n".join(lines) + "\n")
    shutdown()


if __name__ == "__main__":
    main()
