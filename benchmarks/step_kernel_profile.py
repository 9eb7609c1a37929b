#!/usr/bin/env python
"""Per-kernel device times of the exchange step kernels on ONE GPU (self-loop ring: dataset=mnist semantics keep
the communication on at world 1, so every kernel runs with its full protocol against itself).  torch.profiler
(CUPTI) kernel table; use it to see where a step's time goes before reaching for ncu.

    python benchmarks/step_kernel_profile.py [--algo spevent|decent|event|cent] [--topk 1] [--out file]
        [--weight-decay 5e-4] [--nesterov] [--lr-schedule multistep|step|cosine] [--trigger norm|drift]
The optimizer flags run the same kernels with weight decay, Nesterov momentum and a per-step learning-rate table
(engine/lr_schedule.py: two "epochs" spanning the run, so the lr changes inside the profiled window) instead of
the reference's constant-lr heavy-ball SGD.  The threshold is a constant 0, so event fires every tensor at every
step; --trigger drift (event/spevent) adds the `sent` traffic of the drift trigger at that full firing rate.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.config import TrainConfig  # noqa: E402
from eventgrad_b200.engine import lr_schedule  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.parallel import ParamArena, Ring  # noqa: E402
from eventgrad_b200.parallel.p2p import P2PBackend, preallocate_arena_buffers  # noqa: E402
from eventgrad_b200.utils.dist import DistEnv  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--algo", default="spevent")
    ap.add_argument("--topk", type=float, default=1.0)
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default="")
    ap.add_argument("--weight-decay", type=float, default=0.0)
    ap.add_argument("--nesterov", action="store_true")
    ap.add_argument("--lr-schedule", default="constant", choices=["constant", "step", "multistep", "cosine"])
    ap.add_argument("--trigger", default="norm", choices=["norm", "drift"])
    a = ap.parse_args()
    env = DistEnv(0, 1, 0, torch.device("cuda", 0), "none")
    cfg = TrainConfig(algo=a.algo, dataset="mnist", model=a.model, lr=1e-2, momentum=0.9, sync_mode="iter",
                      thres_type=0, constant=0.0, topk_percent=a.topk, weight_decay=a.weight_decay,
                      nesterov=a.nesterov, lr_schedule=a.lr_schedule, lr_milestones=(1,), lr_step_epochs=1,
                      epochs=2, trigger=a.trigger).validate()
    torch.manual_seed(0)
    model = build_model(a.model)
    theta, grad, symm = preallocate_arena_buffers(model, cfg, env)
    arena = ParamArena(model, env.device, theta=theta, grad=grad)
    be = P2PBackend(cfg, arena, Ring(0, 1), env, symm=symm)
    if not lr_schedule.is_constant(cfg):
        be.set_lr_table(lr_schedule.lr_table(cfg, (5 + a.steps) // 2 + 1))
    for _ in range(5):
        arena.grad.normal_(0, 0.01)
        be.step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            arena.grad.normal_(0, 0.01)
            be.step()
        torch.cuda.synchronize()
    be.check_status()
    rows = sorted(((e.key, e.device_time_total / a.steps, e.count / a.steps) for e in prof.key_averages()
                   if e.device_time_total > 0), key=lambda r: -r[1])
    lines = [f"{a.algo} topk={a.topk} model={a.model} wd={a.weight_decay} nesterov={int(a.nesterov)} "
             f"lr_schedule={a.lr_schedule} trigger={a.trigger}: device us per step (calls per step)"]
    lines += [f"{us:10.1f} us  x{n:4.1f}  {k[:110]}" for k, us, n in rows]
    print("\n".join(lines))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write("\n".join(lines) + "\n")
    be.close()


if __name__ == "__main__":
    main()
