"""Learning-rate schedules as one precomputed table: one fp32 learning rate per training step of the run.

Every backend reads the same table -- the fused kernels from device memory, indexed by their device-resident
pass counter (so a captured CUDA graph follows the schedule without being captured again), the collective
backends and the simulator on the host -- so all of them use the same floats.  Step s (1-based) uses
table[min(s-1, len-1)]: a run longer than `epochs` keeps the last value.

Kinds (the epoch e = (s-1) // steps_per_epoch is 0-based, as torch.optim.lr_scheduler counts epochs):
  constant   lr
  step       lr * gamma ** (e // lr_step_epochs)                              (StepLR)
  multistep  lr * gamma ** (number of milestones <= e)                        (MultiStepLR)
  cosine     lr_min + (lr - lr_min) * (1 + cos(pi * e / epochs)) / 2          (CosineAnnealingLR, T_max = epochs)
and an optional linear warm-up over the first W = round(lr_warmup_epochs * steps_per_epoch) steps that multiplies
the value above by (i + 1) / W at step index i = s - 1 (LinearLR(start_factor=1/W, total_iters=W-1), stepped per
step).  Values are computed in float64 and rounded to fp32 once.
"""
from __future__ import annotations

import bisect
import math

import torch

KINDS = ("constant", "step", "multistep", "cosine")


def is_constant(cfg) -> bool:
    """True when every step uses cfg.lr: the kernels then take the scalar lr and no table is needed."""
    return cfg.lr_schedule == "constant" and not cfg.lr_warmup_epochs


def epoch_lr(cfg, e: int) -> float:
    """Learning rate of 0-based epoch `e` before warm-up, in float64."""
    kind, lr = cfg.lr_schedule, float(cfg.lr)
    if kind == "constant":
        return lr
    if kind == "step":
        return lr * float(cfg.lr_gamma) ** (e // int(cfg.lr_step_epochs))
    if kind == "multistep":
        return lr * float(cfg.lr_gamma) ** bisect.bisect_right(sorted(cfg.lr_milestones), e)
    if kind == "cosine":
        lo = float(cfg.lr_min)
        return lo + (lr - lo) * (1.0 + math.cos(math.pi * e / int(cfg.epochs))) / 2.0
    raise ValueError(f"unknown lr_schedule {kind!r}; expected one of {KINDS}")


def warmup_steps(cfg, steps_per_epoch: int) -> int:
    w = float(cfg.lr_warmup_epochs or 0.0)
    return max(1, int(round(w * steps_per_epoch))) if w > 0 else 0


def lr_table(cfg, steps_per_epoch: int) -> torch.Tensor:
    """fp32 tensor [cfg.epochs * steps_per_epoch]: the learning rate of every training step of the run."""
    if steps_per_epoch < 1 or cfg.epochs < 1:
        raise ValueError("lr_table needs steps_per_epoch >= 1 and epochs >= 1")
    W = warmup_steps(cfg, steps_per_epoch)
    vals = []
    for i in range(int(cfg.epochs) * steps_per_epoch):
        v = epoch_lr(cfg, i // steps_per_epoch)
        if i < W:
            v = v * (i + 1) / W
        vals.append(v)
    return torch.tensor(vals, dtype=torch.float64).to(torch.float32)


def lr_at(table, step: int, default: float) -> float:
    """Learning rate of 1-based training step `step` (the scalar default when there is no table)."""
    if table is None:
        return default
    return float(table[min(max(step, 1), len(table)) - 1])
