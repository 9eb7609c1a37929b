"""Communication-backend interface.

A backend owns everything that happens between backward() and the next forward():
the exchange (all-reduce or neighbour gossip), the consensus average and the optimizer
update.  Three implementations:

  p2p        fused sm_90a kernels over peer-mapped memory (the product)       parallel/p2p.py
  nccl/gloo  torch.distributed collectives + eager elementwise ops (baseline /
             GPU-free plumbing)                                                parallel/collective.py
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

from .topology import is_match


@dataclass
class StepLog:
    """Per-step per-tensor records that back the reference debug files (SURVEY.md A.3)."""
    pass_num: int
    curr_norm: torch.Tensor          # [sz] sender norm
    thres: torch.Tensor              # [sz] threshold used in the test
    fired: torch.Tensor              # [sz] bool
    left_norm: Optional[torch.Tensor] = None
    right_norm: Optional[torch.Tensor] = None
    left_new: Optional[torch.Tensor] = None
    right_new: Optional[torch.Tensor] = None


def check_topology_state(sd: Dict, ring, algo: str) -> None:
    """Refuse to resume gossip state saved under a different graph: the inbox slots would mean other peers.  Ring
    checkpoints carry no `topology_offsets` key (their format predates graphs); static graphs carry no `topology` key,
    time-varying ones store their name (onepeer-exp), whose offsets can equal a static graph's.  random-match also stores
    its `topology_seed`: under another seed the run would continue with another sequence of matchings."""
    if algo not in ("decent", "event"):
        return
    saved = (str(sd.get("topology", "circulant")), tuple(sd.get("topology_offsets", (1,))), sd.get("topology_seed"))
    now = (getattr(ring, "kind", "circulant"), tuple(getattr(ring, "offsets", (1,))),
           ring.seed if is_match(ring) else None)
    if saved != now:
        seed = lambda s: "" if s is None else f" seed {s}"
        raise ValueError(f"checkpoint was written with topology {saved[0]} offsets {saved[1]}{seed(saved[2])}, this run "
                         f"uses {now[0]} offsets {now[1]}{seed(now[2])}; "
                         "resume with the same --topology" + (" and --topology-seed" if saved[2] is not None else ""))


def check_trigger_state(sd: Dict, metric: str, algo: str) -> None:
    """Refuse to resume event / spevent state saved under the other trigger metric: the FSM's thresholds, slopes and
    pending decision were computed from a different quantity.  Checkpoints without a `trigger` key are norm-trigger
    checkpoints (their format predates the drift trigger)."""
    if algo not in ("event", "spevent"):
        return
    saved = str(sd.get("trigger", "norm"))
    if saved != metric:
        raise ValueError(f"checkpoint was written with --trigger {saved}, this run uses --trigger {metric}; "
                         "resume with the same --trigger")


def check_compress_state(sd: Dict, compress: str, algo: str) -> None:
    """Refuse to resume decent / event state saved under the other --compress setting: int8 state is the public copy
    `prev` and the neighbour replicas, dense state the inboxes.  Checkpoints without a `compress` key are dense (their
    format predates compression)."""
    if algo not in ("decent", "event"):
        return
    saved = str(sd.get("compress", "none"))
    if saved != compress:
        raise ValueError(f"checkpoint was written with --compress {saved}, this run uses --compress {compress}; "
                         "resume with the same --compress")


def check_choco_state(sd: Dict, gamma: float, algo: str) -> None:
    """Refuse to resume decent / event state saved under another --choco-gamma: the public copies and replicas were
    built by a different mix, and the run would silently change its fixed point.  Checkpoints without a `choco_gamma`
    key were written with the feature off (0)."""
    if algo not in ("decent", "event"):
        return
    saved = float(sd.get("choco_gamma", 0.0))
    if saved != float(gamma):
        raise ValueError(f"checkpoint was written with --choco-gamma {saved:g}, this run uses --choco-gamma "
                         f"{float(gamma):g}; resume with the same --choco-gamma")


def check_tracking_state(sd: Dict, tracking: bool, algo: str) -> None:
    """Refuse to resume decent state saved under the other --gradient-tracking setting: tracking state is y, the
    previous gradient and the y inboxes, which a plain run neither saves nor restores.  Checkpoints without a
    `gradient_tracking` key are non-tracking (their format predates gradient tracking)."""
    if algo != "decent":
        return
    saved = bool(sd.get("gradient_tracking", False))
    if saved != bool(tracking):
        flag = lambda on: "--gradient-tracking" if on else "no --gradient-tracking"
        raise ValueError(f"checkpoint was written with {flag(saved)}, this run uses {flag(tracking)}; "
                         "resume with the same --gradient-tracking setting")


def check_local_steps_state(sd: Dict, local_steps: int, algo: str) -> None:
    """Refuse to resume decent state saved under another --local-steps: the inboxes hold what the last round of that
    schedule delivered, and the one-peer graph's slot is indexed by its rounds.  Checkpoints without a `local_steps` key
    gossiped at every step (their format predates periodic gossip).  A resume at a step that is not a multiple of H
    continues the cycle by itself: which step gossips is a function of the restored step counter."""
    if algo != "decent":
        return
    saved = int(sd.get("local_steps", 1))
    if saved != int(local_steps):
        raise ValueError(f"checkpoint was written with --local-steps {saved}, this run uses --local-steps "
                         f"{int(local_steps)}; resume with the same --local-steps")


def check_global_avg_state(sd: Dict, period: int, algo: str) -> None:
    """Refuse to resume decent state saved under another --global-avg-period: the inboxes hold what the last gossip step
    of that schedule delivered.  Checkpoints without a `global_avg_period` key never averaged (the key is written only
    when P > 0, so checkpoints of runs without the feature keep their keys).  A resume at any step continues the cycle
    by itself: which step averages is a function of the restored step counter."""
    if algo != "decent":
        return
    saved = int(sd.get("global_avg_period", 0))
    if saved != int(period):
        raise ValueError(f"checkpoint was written with --global-avg-period {saved}, this run uses --global-avg-period "
                         f"{int(period)}; resume with the same --global-avg-period")


def slowmo_state(be) -> Dict:
    """Checkpoint entries of a decent backend under --slowmo-period (none when the feature is off, so other checkpoints
    keep their keys): the settings and the outer iterate x and slow momentum u, on the CPU."""
    if not be.slowmo_period:
        return {}
    return {"slowmo_period": be.slowmo_period, "slowmo_beta": be.slowmo_beta, "slowmo_lr": be.slowmo_lr,
            "slowmo_x": be.slowmo_x.cpu().clone(), "slowmo_u": be.slowmo_u.cpu().clone()}


def check_slowmo_state(sd: Dict, period: int, beta: float, alpha: float, algo: str) -> None:
    """Refuse to resume decent state saved under other --slowmo-period / --slowmo-beta / --slowmo-lr settings, in either
    direction: x and u belong to that schedule.  Checkpoints without a `slowmo_period` key never ran SlowMo.  A resume at
    any step continues the cycle by itself: which step syncs is a function of the restored step counter."""
    if algo != "decent":
        return
    saved = (int(sd.get("slowmo_period", 0)), float(sd.get("slowmo_beta", beta)), float(sd.get("slowmo_lr", alpha)))
    run = (int(period), float(beta), float(alpha))
    if saved[0] != run[0] or (run[0] and saved != run):
        fmt = lambda s: f"--slowmo-period {s[0]}" + (f" --slowmo-beta {s[1]} --slowmo-lr {s[2]}" if s[0] else "")
        raise ValueError(f"checkpoint was written with {fmt(saved)}, this run uses {fmt(run)}; resume with the same "
                         "--slowmo-period, --slowmo-beta and --slowmo-lr")


def check_qg_state(sd: Dict, qg: bool, algo: str) -> None:
    """Refuse to resume gossip state saved under the other --quasi-global-momentum setting: the momentum buffer holds
    m_hat with it and the heavy-ball m without it.  The key is written only when the feature is on, so checkpoints of
    runs without it keep their keys."""
    if algo not in ("decent", "event", "spevent"):
        return
    saved = bool(sd.get("quasi_global_momentum", False))
    if saved != bool(qg):
        have = "with" if saved else "without"
        run = "with" if qg else "without"
        raise ValueError(f"checkpoint was written {have} --quasi-global-momentum, this run is {run} it: its momentum "
                         "buffer holds " + ("m_hat" if saved else "the heavy-ball momentum") +
                         "; resume with the same --quasi-global-momentum setting")

def check_exact_diffusion_state(sd: Dict, ed: bool, algo: str) -> None:
    """Refuse to resume decent state saved under the other --exact-diffusion setting: exact-diffusion state is psi, and
    its inboxes hold the neighbours' phi rather than their theta.  Checkpoints without an `exact_diffusion` key are plain
    (their format predates exact diffusion)."""
    if algo != "decent":
        return
    saved = bool(sd.get("exact_diffusion", False))
    if saved != bool(ed):
        flag = lambda on: "--exact-diffusion" if on else "no --exact-diffusion"
        raise ValueError(f"checkpoint was written with {flag(saved)}, this run uses {flag(ed)}; "
                         "resume with the same --exact-diffusion setting")


class CommBackend:
    name = "base"

    def __init__(self, cfg, arena, ring):
        self.cfg = cfg
        self.arena = arena
        self.ring = ring
        self.pass_num = 0
        self.logs: List[StepLog] = []
        self.want_logs = bool(cfg.file_write)
        self.lr_table: Optional[torch.Tensor] = None

    # -- learning-rate schedule (engine/lr_schedule.py) ------------------------------------
    def set_lr_table(self, table: Optional[torch.Tensor]) -> None:
        """Per-step learning rates of the run (fp32, step s uses table[min(s-1, len-1)]); None = constant cfg.lr.
        The step index is the backend's pass counter, so a restored checkpoint resumes mid-schedule."""
        self.lr_table = None if table is None else table.detach().to("cpu", torch.float32).contiguous()

    def step_lr(self, step: int) -> float:
        """Learning rate of 1-based training step `step`."""
        from ..engine.lr_schedule import lr_at
        return lr_at(self.lr_table, step, self.cfg.lr)

    # -- one training step (after backward) -------------------------------------------
    def step(self) -> None:
        raise NotImplementedError

    # -- end of training ----------------------------------------------------------------
    def final_average(self) -> None:
        raise NotImplementedError

    def num_events(self) -> int:
        return 0

    def total_events(self) -> int:
        return 0

    def bytes_sent(self) -> int:
        return 0

    def set_sparse_init(self, prev, rep_l, rep_r) -> None:
        """spevent only, reference quirk Q8 (spevent.cpp:123-136): start the 'previously sent' copy and the two
        neighbour replicas from the given flat tensors (three more random networks in the reference)
        instead of theta_0.  Must be called before the first step."""
        if self.cfg.algo != "spevent" or not hasattr(self, "prev"):
            raise RuntimeError("set_sparse_init applies to the spevent algorithm only")
        if self.pass_num != 0:
            raise RuntimeError("set_sparse_init must be called before the first step")
        self.prev.copy_(prev.to(self.prev.device))
        self.rep_l.copy_(rep_l.to(self.rep_l.device))
        self.rep_r.copy_(rep_r.to(self.rep_r.device))

    def drain_logs(self) -> List[StepLog]:
        out, self.logs = self.logs, []
        return out

    # -- consensus distance (--consensus-every N) -----------------------------------------
    def set_consensus_capacity(self, cap: int) -> None:
        """Measurements kept between two drains (the p2p backend's device ring); the host-side backends keep all."""

    def drain_consensus(self) -> List:
        """Measurements since the last drain, oldest first: (step, D, A) with D and A float64 CPU tensors [n_tensors]
        (parallel/trigger.py:consensus_stats)."""
        return []

    def measure_consensus(self):
        """(D, A) of the current parameters, measured now whatever the step; every rank must call it."""
        raise NotImplementedError

    def synchronize(self) -> None:
        pass

    def state_dict(self) -> Dict:
        return {"pass_num": self.pass_num}

    def load_state_dict(self, sd: Dict) -> None:
        self.pass_num = int(sd.get("pass_num", 0))

    def close(self) -> None:
        pass

    # helpers ---------------------------------------------------------------------------
    @property
    def comm_enabled(self) -> bool:
        """CIFAR programs skip all communication when R == 1 (event.cpp:281); the MNIST event
        program does not (it Puts to itself).  `serial_skip` carries that distinction."""
        if self.ring.world > 1:
            return True
        return not getattr(self.cfg, "dataset", "cifar10") == "cifar10"
