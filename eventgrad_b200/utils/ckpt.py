"""Checkpoint / resume (a capability the reference lacks entirely -- SURVEY.md section 5:
"no torch::save/load; model lives and dies with the process").

One file per rank: arena (theta + momentum, with its layout), the backend's communication state (trigger FSM,
inboxes / sparse replicas, event counters, pass_num; on a gossip graph every slot's inbox, the offsets and, for
onepeer-exp, the topology name, checked on resume by parallel/base.py; event/spevent: the trigger name, and under
--trigger drift event's `sent` buffer, also checked on resume; decent/event: the `compress` setting, and under
--compress int8 / sign `prev` and the neighbour replicas `rep_l` / `rep_r` instead of the inboxes, checked on resume by
check_compress_state, and `choco_gamma` when --choco-gamma is on (check_choco_state); decent: the
`gradient_tracking` setting, and under --gradient-tracking y, the previous gradient
`g_prev` and the y inboxes `y_in_l` / `y_in_r`, checked on resume by check_tracking_state; decent: the `local_steps`
period, checked on resume by check_local_steps_state; decent: the `exact_diffusion` setting, and under
--exact-diffusion `psi`, checked on resume by check_exact_diffusion_state; decent with --global-avg-period P > 0: the
`global_avg_period`, checked on resume by check_global_avg_state; decent/event/spevent with --quasi-global-momentum:
`quasi_global_momentum`, checked on resume by check_qg_state; decent with --slowmo-period tau > 0: `slowmo_period`,
`slowmo_beta`, `slowmo_lr`, the outer iterate `slowmo_x` and the slow momentum `slowmo_u`, checked on resume by
check_slowmo_state), BN buffers, RNG state
(global + the loader's private augmentation generator), step counter and epoch.  Only tensors / numbers / strings / lists / dicts are stored, so
files are read back with `weights_only=True` (no pickle code execution from a user-supplied --resume path).  The
ranks' models differ between consensus rounds, so a decentralized run can only be resumed
exactly from per-rank state.
"""
from __future__ import annotations

import os
from typing import Any, Dict

import torch


def ckpt_path(ckpt_dir: str, rank: int, tag: str = "last") -> str:
    return os.path.join(ckpt_dir, f"ckpt_{tag}_rank{rank}.pt")


def save_checkpoint(path: str, *, epoch: int, arena, backend, model, loader=None, steps_done: int = 0,
                    extra: Dict[str, Any] | None = None) -> None:
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    backend.synchronize()
    sd = {
        "format": 1,
        "epoch": epoch,
        "arena": arena.state_dict(),
        "backend": backend.state_dict(),
        "buffers": {k: v.detach().cpu().clone() for k, v in model.named_buffers()},
        "rng_cpu": torch.get_rng_state(),
        "steps_done": int(steps_done),
        "extra": extra or {},
    }
    if loader is not None and getattr(loader, "gen", None) is not None:
        sd["loader_gen"] = loader.gen.get_state().cpu()
    if torch.cuda.is_available() and arena.theta.is_cuda:
        sd["rng_cuda"] = torch.cuda.get_rng_state(arena.theta.device)
    tmp = path + ".tmp"
    torch.save(sd, tmp)
    os.replace(tmp, path)


def load_checkpoint(path: str, *, arena, backend, model, loader=None) -> Dict[str, Any]:
    sd = torch.load(path, map_location="cpu", weights_only=True)
    arena.load_state_dict(sd["arena"])
    backend.load_state_dict(sd["backend"])
    bufs = dict(model.named_buffers())
    for k, v in sd["buffers"].items():
        if k in bufs:
            bufs[k].copy_(v.to(bufs[k].device))
    torch.set_rng_state(sd["rng_cpu"])
    if "rng_cuda" in sd and arena.theta.is_cuda:
        torch.cuda.set_rng_state(sd["rng_cuda"], arena.theta.device)
    if loader is not None and "loader_gen" in sd and getattr(loader, "gen", None) is not None:
        loader.gen.set_state(sd["loader_gen"])
    return sd
