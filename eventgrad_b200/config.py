"""Configuration: one dataclass + argparse, with a positional-argv compatibility
shim for the reference programs' CLI.

Reference CLI (positional, no validation):
  dmnist/event, dcifar10/event : <file_write> <thres_type> <horizon|constant>
      (/root/reference/dmnist/event/event.cpp:89-100,
       /root/reference/dcifar10/event/event.cpp:46-57)
  dcifar10/spevent             : ... + <topk_percent>
      (/root/reference/dcifar10/spevent/spevent.cpp:47-60)
  dmnist/decent                : <file_write>   (decent.cpp:44)
  dmnist/cent                  : none
Every other knob in the reference is a source constant (SURVEY.md section 2.6);
here they are the *defaults* of the matching preset and can be overridden.
"""
from __future__ import annotations

import argparse
import dataclasses
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

ALGOS = ("cent", "decent", "event", "spevent")
DATASETS = ("mnist", "cifar10")


@dataclass
class TrainConfig:
    # ---- what to run -----------------------------------------------------
    algo: str = "event"              # cent | decent | event | spevent
    dataset: str = "cifar10"         # mnist | cifar10
    model: str = "resnet18"          # mlp | cnn1 | cnn2 | lenet | resnet18/34/50/101/152
    resnet_variant: str = "ref"      # ref (blocks+1 per stage, as shipped) | canonical
    # ---- optimisation ----------------------------------------------------
    epochs: int = 20
    batch_size: int = 256            # meaning depends on batch_mode
    batch_mode: str = "global"       # global (split over ranks) | per_rank | full (whole shard)
    lr: float = 1e-2
    momentum: float = 0.9
    seed: int = 0
    # torch.optim.SGD options and learning-rate schedule, applied inside the fused step kernels (absent in the
    # reference: the defaults reproduce its constant-lr heavy-ball SGD).  See engine/lr_schedule.py.
    weight_decay: float = 0.0        # L2 on every arena tensor (BN included), as SGD without parameter groups
    nesterov: bool = False           # needs momentum > 0
    lr_schedule: str = "constant"    # constant | step | multistep | cosine
    lr_step_epochs: int = 30         # step: multiply by lr_gamma every this many epochs
    lr_milestones: Tuple[int, ...] = ()   # multistep: epochs at which lr is multiplied by lr_gamma
    lr_gamma: float = 0.1
    lr_min: float = 0.0              # cosine: final learning rate
    lr_warmup_epochs: float = 0.0    # linear warm-up, stepped per step (0: none)
    # ---- event trigger (SURVEY.md A.1) -------------------------------------
    thres_type: int = 1              # 1 adaptive (horizon), 0 constant
    horizon: float = 1.0
    constant: float = 0.0
    sent_history: int = 2
    initial_comm_passes: int = 30
    topk_percent: float = 10.0       # spevent only
    trigger: str = "norm"            # norm: | ||theta|| - ||theta at last send|| | >= thres (the reference rule) |
                                     # drift: ||theta - sent|| >= thres, sent = what the receivers hold (event/spevent)
    # ---- communication ---------------------------------------------------
    backend: str = "auto"            # auto | p2p (fused sm_90a kernels) | nccl | gloo | refport (reference-structured)
    sync_mode: str = "iter"          # iter (deterministic handshake) | async (reference RMA semantics)
    final_divide_all: bool = True    # reference divides on rank 0 only (Q5)
    grad_table: bool = True          # p2p gossip: step kernel reads autograd's gradients in place (+ bf16
                                     # shadow weights under dtype=bf16) instead of an fp32 grad arena
    overlap_push: Optional[bool] = None   # p2p: launch the push half of the step on a side stream so it overlaps
                                     # forward/backward (False = single fused kernel).  None = auto: on for
                                     # decent/event on >= 2 GPUs
    spevent_fresh_replicas: bool = False   # reference quirk Q8: prev/left/right replicas of spevent are three
                                     # MORE randomly initialised networks (spevent.cpp:123-136) instead of theta_0
    ce_push: bool = False            # decent + overlap_push: the push half of the split step is copy-engine memcpys
                                     # instead of an SM kernel (csrc/ce_push.cu)
    double_buffer: Optional[bool] = None   # decent, p2p, iter-sync, fused (non-split) step: two inbox slots and no
                                     # WAR ack (csrc/gossip_dbuf.cu).  None = on where it applies
    peer_timeout_s: float = 30.0     # bound of every device-side peer wait (sticky status instead of a hang);
                                     # EGB_PEER_TIMEOUT_S overrides
    topology: str = "ring"           # gossip graph (parallel/topology.py): ring | exp (offsets 1,2,4,...) | "o1,o2,..."
                                     # | onepeer-exp (time-varying: one peer r + 2^((k-1) mod ceil(log2 R)) per step)
                                     # | random-match (a seeded random perfect matching per step, pairwise averaging)
                                     # (circulant offsets, at most 4); decent/event only beyond the ring
    topology_seed: int = 0           # random-match: seed in [0, 2^31) of the per-step matchings (same on every rank)
    compress: str = "none"           # none | int8 | sign: decent/event on the ring send the int8 (sign: 1-bit scaled sign)
                                     # code of theta - prev (one fp32 scale per 256 elements) instead of fp32 theta
    choco_gamma: float = 0.0         # int8/sign: 0 < gamma <= 1 mixes by CHOCO-SGD's consensus step on the public copies,
                                     # theta += gamma * (W prev - prev), which keeps the ranks' average; 0 = off
    gradient_tracking: bool = False  # decent on the ring: also gossip y, which tracks the average gradient, and step
                                     # along y instead of the local gradient (DSGT / DIGing; fused single-slot step)
    local_steps: int = 1             # decent: gossip at every H-th step only (step k iff H divides k); the H - 1 steps
                                     # between are serial SGD steps with no exchange (local / periodic D-PSGD)
    exact_diffusion: bool = False    # decent on the ring: exact diffusion (D^2 on (I + W) / 2): SGD before the push,
                                     # gossip phi = p + theta - psi; no heterogeneity bias at decent's bytes
    global_avg_period: int = 0       # decent on the ring / a static graph: every P-th step (P >= 2) averages theta over
                                     # all ranks exactly in place of the gossip mix (Gossip-PGA); 0 = off
    quasi_global_momentum: bool = False  # decent/event/spevent, momentum > 0: the momentum buffer follows each rank's
                                     # parameter displacement (mix included) instead of its gradient (QG-DSGDm)
    slowmo_period: int = 0           # decent on the ring / a static graph: every tau-th step (tau >= 2) averages theta
                                     # exactly and takes a slow heavy-ball step on the average from where the cycle
                                     # started (SlowMo); base: gossip (local_steps 1) or local SGD (local_steps tau); 0 = off
    slowmo_beta: float = 0.5         # SlowMo slow momentum, 0 <= beta < 1
    slowmo_lr: float = 1.0           # SlowMo slow learning rate, alpha > 0
    consensus_every: int = 0         # gossip algorithms: every N-th step measure the consensus distance
                                     # sqrt(sum_r ||theta_r - theta_bar||^2 / R) per tensor (read-only); 0 = off
    gossip_rounds: int = 1           # decent on the ring / a static graph: Q >= 2 runs Q - 1 mix-only gossip rounds
                                     # before the step's own mix, theta_{k+1} = SGD(W^Q theta_k); Q times the bytes
    gossip_accel: str = "none"       # none | chebyshev: the Q rounds of --gossip-rounds apply the degree-Q Chebyshev
                                     # polynomial P_Q(W) of the graph's spectrum instead of W^Q, at the same bytes
    # ---- data --------------------------------------------------------------
    data: str = "synthetic"          # synthetic | path to dataset root
    sampler: str = "random"          # random | sequential
    partition: str = "iid"           # iid (a block of a random / the identity order) | label (shards cut from the
                                     # samples sorted by class: heterogeneous, still equal-sized)
    augment: bool = True             # pad4 + flip + crop (cifar only)
    native_loader: str = "auto"      # auto (CPU: native C++ prefetcher, CUDA: Python staging) | on | off
    train_samples: int = 50000
    test_samples: int = 10000
    test_batch_size: int = 100
    # ---- execution ---------------------------------------------------------
    device: str = "auto"             # auto | cuda | cpu
    dtype: str = "fp32"              # fp32 | tf32 | bf16 (compute dtype; arena is fp32)
    channels_last: Optional[bool] = None   # None = auto on CUDA: NHWC, except fp32 with conv_tc off (cuDNN's fp32 convs are NCHW)
    conv_tc: Optional[bool] = None         # fp32 only: 3x3 convs on the wgmma tensor cores at fp32 accuracy (csrc/conv_tc.cu);
                                           # None = on for CUDA (EGB_CONV_TC=0 turns it off); False = cuDNN's SIMT fp32 kernels
    cuda_graph: Optional[bool] = None      # None = auto: whole-step CUDA graph on CUDA
    max_steps: int = 0               # >0: stop after this many steps (tests / bench)
    cudnn_benchmark: bool = True     # cuDNN autotune: best steady state, but every new conv shape costs a
                                     # one-time search (seconds; it also hits the partial last batch)
    host_threads: int = 2            # intra-op CPU threads on GPU runs (0 = leave torch's default)
    # ---- observability -------------------------------------------------------
    file_write: int = 0              # reference debug files send/recv/train/values<r>.txt
    log_dir: str = "."
    ckpt_dir: str = ""
    ckpt_every: int = 0              # epochs; 0 = never
    resume: str = ""
    quiet: bool = False
    phase_timers: bool = False       # per-phase device timers (CUDA events + NVTX ranges), printed by rank 0

    def validate(self) -> "TrainConfig":
        if self.algo not in ALGOS:
            raise ValueError(f"algo must be one of {ALGOS}, got {self.algo!r}")
        if self.dataset not in DATASETS:
            raise ValueError(f"dataset must be one of {DATASETS}")
        if self.sync_mode not in ("iter", "async"):
            raise ValueError("sync_mode must be iter|async")
        if self.algo == "decent" and self.sync_mode != "iter":
            raise ValueError("decent (D-PSGD) is lock-step by definition: sync_mode=iter")
        if self.batch_mode not in ("global", "per_rank", "full"):
            raise ValueError("batch_mode must be global|per_rank|full")
        if self.thres_type not in (0, 1):
            raise ValueError("thres_type must be 0 (constant) or 1 (adaptive)")
        if not (0.0 < self.topk_percent <= 100.0):
            raise ValueError("topk_percent must be in (0, 100]")
        if self.dtype not in ("fp32", "tf32", "bf16"):
            raise ValueError("dtype must be fp32|tf32|bf16")
        if not self.weight_decay >= 0.0:
            raise ValueError(f"weight_decay must be >= 0, got {self.weight_decay}")
        if self.nesterov and self.momentum == 0.0:
            raise ValueError("nesterov requires momentum > 0")
        if self.lr_schedule not in ("constant", "step", "multistep", "cosine"):
            raise ValueError(f"lr_schedule must be constant|step|multistep|cosine, got {self.lr_schedule!r}")
        if self.lr_schedule == "step" and self.lr_step_epochs < 1:
            raise ValueError("lr_step_epochs must be >= 1")
        ms = list(self.lr_milestones)
        if any(b <= a for a, b in zip(ms, ms[1:])) or any(m < 0 for m in ms):
            raise ValueError(f"lr_milestones must be non-negative and strictly increasing, got {ms}")
        if not self.lr_warmup_epochs >= 0.0:
            raise ValueError("lr_warmup_epochs must be >= 0")
        if self.trigger not in ("norm", "drift"):
            raise ValueError(f"trigger must be norm|drift, got {self.trigger!r}")
        if self.trigger == "drift":
            if self.algo not in ("event", "spevent"):
                raise ValueError(f"--trigger drift needs algo event or spevent ({self.algo!r} has no trigger)")
            if self.backend == "refport":
                raise ValueError("--trigger drift is not supported by --backend refport (the reference's norm rule only)")
            if self.file_write:
                raise ValueError("--trigger drift does not support file_write: the reference log format's norm column "
                                 "would hold the drift")
        from .parallel.topology import check_topology_name
        check_topology_name(self.topology)
        if not self.ring_topology:
            # a graph beyond the ring runs on the fused single-kernel step (csrc/gossip_graph.cu) and the
            # torch.distributed backends; the split step, the double-buffered inbox, copy-engine pushes, spevent and the
            # reference-structured backend exist for the ring only
            if self.algo not in ("decent", "event"):
                raise ValueError(f"topology {self.topology!r} needs algo decent or event, got {self.algo!r}")
            if self.backend == "refport":
                raise ValueError(f"topology {self.topology!r} is not supported by --backend refport (ring only)")
            for name in ("overlap_push", "double_buffer", "ce_push"):
                if getattr(self, name):
                    raise ValueError(f"topology {self.topology!r} does not support {name} (ring only)")
            if self.file_write:
                raise ValueError(f"topology {self.topology!r} does not support file_write: the reference's log format "
                                 "has exactly one left and one right receive column")
        if self.compress not in ("none", "int8", "sign"):
            raise ValueError(f"compress must be none|int8|sign, got {self.compress!r}")
        g = self.choco_gamma
        if isinstance(g, bool) or not isinstance(g, (int, float)) or not 0.0 <= g <= 1.0:   # NaN fails the range
            raise ValueError(f"--choco-gamma must be a number in [0, 1] (0: off), got {g!r}; aggressive codecs want a "
                             "small gamma (with --compress sign, 1 diverges on 2 ranks and 0.2 converges on 2 to 8)")
        if g > 0.0 and self.compress == "none":
            raise ValueError("--choco-gamma needs --compress int8 or sign: it mixes the compressed public copies")
        if self.compress != "none":
            # the int8 step exists as the iter-sync fused ring step (csrc/gossip_q8.cu) and in the torch.distributed
            # backends.  Explicit offsets other than "1" are never the ring; exp and onepeer-exp are the ring at small
            # world sizes, so for_world() checks them once the world size is known
            s = str(self.topology).strip().lower()
            if not (self.ring_topology or s in ("exp", "onepeer-exp")):
                raise ValueError(f"--compress {self.compress} runs on the ring only, got topology {self.topology!r}")
            if self.algo not in ("decent", "event"):
                raise ValueError(f"--compress {self.compress} needs algo decent or event, got {self.algo!r}"
                                 + (" (spevent is its own compressor)" if self.algo == "spevent" else ""))
            if self.sync_mode != "iter":
                raise ValueError(f"--compress {self.compress} needs --sync-mode iter: a delta applied to a torn or "
                                 "stale inbox is not idempotent")
            if self.backend == "refport":
                raise ValueError(f"--compress {self.compress} is not supported by --backend refport")
            for name in ("overlap_push", "double_buffer", "ce_push"):
                if getattr(self, name):
                    raise ValueError(f"--compress {self.compress} does not support {name} (fused single-kernel step "
                                     "only)")
            if self.file_write:
                raise ValueError(f"--compress {self.compress} does not support file_write: the reference's log "
                                 "format records the received fp32 tensors")
        if self.gradient_tracking:
            # the tracking step exists as the iter-sync fused single-slot ring step (csrc/gossip_gt.cu), in the
            # torch.distributed backends and in the simulator; sum_r y_r = sum_r g_r holds only if every y a rank mixes
            # is its neighbour's current one
            if self.algo in ("event", "spevent"):
                raise ValueError(f"--gradient-tracking needs algo decent, got {self.algo!r}: a held tensor leaves the "
                                 "neighbours mixing a stale y, which breaks sum(y) = sum(g)")
            if self.algo != "decent":
                raise ValueError(f"--gradient-tracking needs algo decent, got {self.algo!r}")
            if not self.ring_topology:
                raise ValueError(f"--gradient-tracking runs on the ring only, got topology {self.topology!r}")
            if self.backend == "refport":
                raise ValueError("--gradient-tracking is not supported by --backend refport")
            for name in ("overlap_push", "double_buffer", "ce_push"):
                if getattr(self, name):
                    raise ValueError(f"--gradient-tracking does not support {name} (fused single-slot step only)")
            if self.compress != "none":
                raise ValueError(f"--gradient-tracking does not support --compress {self.compress}")
            if self.file_write:
                raise ValueError("--gradient-tracking does not support file_write: the reference's log format has no "
                                 "column for y")
        if not isinstance(self.local_steps, int) or self.local_steps < 1:
            raise ValueError(f"--local-steps must be an integer >= 1, got {self.local_steps!r}")
        if self.local_steps > 1:
            # periodic gossip exists for decent in the fused single-kernel ring / graph step (csrc/gossip.cu,
            # csrc/gossip_graph.cu), the torch.distributed backends and the simulator
            h = f"--local-steps {self.local_steps}"
            if self.algo == "cent":
                raise ValueError(f"{h} needs algo decent: local SGD with periodic parameter averaging is a different "
                                 "all-reduce step, and cent's momentum lives outside the peer window")
            if self.algo in ("event", "spevent"):
                raise ValueError(f"{h} needs algo decent, got {self.algo!r}: the trigger already decides when to send, "
                                 "and its slope history and event accounting are indexed by step, not by round")
            if self.gradient_tracking:
                raise ValueError(f"{h} does not support --gradient-tracking")
            if self.compress != "none":
                raise ValueError(f"{h} does not support --compress {self.compress}")
            if self.backend == "refport":
                raise ValueError(f"{h} is not supported by --backend refport")
            for name in ("overlap_push", "double_buffer", "ce_push"):
                if getattr(self, name):
                    raise ValueError(f"{h} does not support {name} (fused single-kernel step only)")
            if self.file_write:
                raise ValueError(f"{h} does not support file_write: the reference's log format records an exchange "
                                 "at every step")
        if self.exact_diffusion:
            # the exact-diffusion step exists as the iter-sync fused single-slot ring step (csrc/gossip_ed.cu), in the
            # torch.distributed backends and in the simulator; sum_r theta_r = sum_r psi_r holds only if every phi a rank
            # mixes is its neighbour's current one
            if self.algo in ("event", "spevent"):
                raise ValueError(f"--exact-diffusion needs algo decent, got {self.algo!r}: a held tensor leaves the "
                                 "neighbours mixing a stale phi, a difference-form message, which breaks "
                                 "sum(theta) = sum(psi)")
            if self.algo != "decent":
                raise ValueError(f"--exact-diffusion needs algo decent, got {self.algo!r}")
            if not self.ring_topology:
                raise ValueError(f"--exact-diffusion runs on the ring only, got topology {self.topology!r}")
            if self.backend == "refport":
                raise ValueError("--exact-diffusion is not supported by --backend refport")
            if self.overlap_push:
                raise ValueError("--exact-diffusion does not support overlap_push: the message phi needs this step's "
                                 "gradient, so it cannot be pushed during backward")
            for name in ("double_buffer", "ce_push"):
                if getattr(self, name):
                    raise ValueError(f"--exact-diffusion does not support {name} (fused single-slot step only)")
            if self.compress != "none":
                raise ValueError(f"--exact-diffusion does not support --compress {self.compress}")
            if self.gradient_tracking:
                raise ValueError("--exact-diffusion does not support --gradient-tracking (both remove the same bias)")
            if self.local_steps > 1:
                raise ValueError(f"--exact-diffusion does not support --local-steps {self.local_steps}")
            if self.file_write:
                raise ValueError("--exact-diffusion does not support file_write: the reference's log format records "
                                 "the received theta, and exact diffusion receives phi")
        P = self.global_avg_period
        if isinstance(P, bool) or not isinstance(P, int) or P < 0:
            raise ValueError(f"--global-avg-period must be an integer >= 0, got {P!r}")
        if P == 1:
            raise ValueError("--global-avg-period 1 averages at every step and leaves no gossip: use algo cent")
        if P:
            # periodic global averaging exists for decent in the fused single-kernel ring / static-graph step (the gated
            # all-reduce of csrc/allreduce.cu before csrc/gossip.cu, csrc/gossip_graph.cu), the torch.distributed
            # backends and the simulator
            h = f"--global-avg-period {P}"
            if self.algo != "decent":
                raise ValueError(f"{h} needs algo decent, got {self.algo!r}")
            if str(self.topology).strip().lower() == "onepeer-exp":
                raise ValueError(f"{h} does not support topology onepeer-exp: it already reaches the exact average "
                                 "every tau steps at power-of-two R, and its per-slot WAR bound has no rule for skipped "
                                 "steps")
            if self.gradient_tracking:
                raise ValueError(f"{h} does not support --gradient-tracking")
            if self.exact_diffusion:
                raise ValueError(f"{h} does not support --exact-diffusion")
            if self.compress != "none":
                raise ValueError(f"{h} does not support --compress {self.compress}")
            if self.local_steps > 1:
                raise ValueError(f"{h} does not support --local-steps {self.local_steps}")
            if self.backend == "refport":
                raise ValueError(f"{h} is not supported by --backend refport")
            for name in ("overlap_push", "double_buffer", "ce_push"):
                if getattr(self, name):
                    raise ValueError(f"{h} does not support {name} (fused single-kernel step only)")
            if self.file_write:
                raise ValueError(f"{h} does not support file_write: the reference's log format records a neighbour "
                                 "exchange at every step")
        if self.quasi_global_momentum:
            # quasi-global momentum exists in the ring, double-buffered and graph step kernels (csrc/gossip.cu), the
            # torch.distributed backends and the simulator
            h = "--quasi-global-momentum"
            if self.algo == "cent":
                raise ValueError(f"{h} needs a gossip algorithm (decent, event or spevent), got algo cent")
            if self.momentum == 0.0:
                raise ValueError(f"{h} needs --momentum > 0")
            if self.sync_mode != "iter":
                raise ValueError(f"{h} needs --sync-mode iter: an async mix of a torn or stale inbox would enter the "
                                 "momentum buffer")
            if self.compress != "none":
                raise ValueError(f"{h} does not support --compress {self.compress}")
            if self.gradient_tracking:
                raise ValueError(f"{h} does not support --gradient-tracking")
            if self.exact_diffusion:
                raise ValueError(f"{h} does not support --exact-diffusion")
            if self.global_avg_period:
                raise ValueError(f"{h} does not support --global-avg-period: the gated all-reduce overwrites theta_k "
                                 "before the step kernel reads it")
            if self.backend == "refport":
                raise ValueError(f"{h} is not supported by --backend refport")
            if self.ce_push:
                raise ValueError(f"{h} does not support ce_push")
        tau = self.slowmo_period
        if isinstance(tau, bool) or not isinstance(tau, int) or tau < 0:
            raise ValueError(f"--slowmo-period must be an integer >= 0, got {tau!r}")
        if tau == 1:
            raise ValueError("--slowmo-period 1 averages at every step and leaves no base step: use algo cent")
        if tau:
            # SlowMo exists for decent in the fused single-kernel ring / static-graph step (the gated sync kernel of
            # csrc/allreduce.cu before csrc/gossip.cu, csrc/gossip_graph.cu), the torch.distributed backends and the
            # simulator
            h = f"--slowmo-period {tau}"
            if not (isinstance(self.slowmo_beta, (int, float)) and 0.0 <= self.slowmo_beta < 1.0):
                raise ValueError(f"--slowmo-beta must be in [0, 1), got {self.slowmo_beta!r}")
            if not (isinstance(self.slowmo_lr, (int, float)) and self.slowmo_lr > 0.0):
                raise ValueError(f"--slowmo-lr must be > 0, got {self.slowmo_lr!r}")
            if not self.lr > 0.0:
                raise ValueError(f"{h} needs --lr > 0: the slow momentum is (x - theta_bar) / lr")
            if self.algo == "cent":
                raise ValueError(f"{h} needs algo decent: cent has its own all-reduce step")
            if self.algo in ("event", "spevent"):
                raise ValueError(f"{h} needs algo decent, got {self.algo!r}: the trigger's last_norm / sent state has no "
                                 "defined meaning across the jump of theta at a sync")
            if str(self.topology).strip().lower() == "onepeer-exp":
                raise ValueError(f"{h} does not support topology onepeer-exp: its per-slot WAR bound has no rule for "
                                 "skipped steps")
            if self.local_steps not in (1, tau):
                raise ValueError(f"{h} needs --local-steps 1 (gossip base) or {tau} (local SGD base), got "
                                 f"--local-steps {self.local_steps}")
            if self.global_avg_period:
                raise ValueError(f"{h} does not support --global-avg-period: both replace the mix at the same steps")
            if self.gradient_tracking:
                raise ValueError(f"{h} does not support --gradient-tracking")
            if self.exact_diffusion:
                raise ValueError(f"{h} does not support --exact-diffusion")
            if self.compress != "none":
                raise ValueError(f"{h} does not support --compress {self.compress}")
            if self.quasi_global_momentum:
                raise ValueError(f"{h} does not support --quasi-global-momentum: the sync overwrites theta_k before the "
                                 "step kernel reads it back")
            if self.backend == "refport":
                raise ValueError(f"{h} is not supported by --backend refport")
            for name in ("overlap_push", "double_buffer", "ce_push"):
                if getattr(self, name):
                    raise ValueError(f"{h} does not support {name} (fused single-kernel step only)")
            if self.file_write:
                raise ValueError(f"{h} does not support file_write: the reference's log format records a neighbour "
                                 "exchange at every step")
        N = self.consensus_every
        if isinstance(N, bool) or not isinstance(N, int) or N < 0:
            raise ValueError(f"--consensus-every must be an integer >= 0, got {N!r}")
        if N:
            h = f"--consensus-every {N}"
            if self.algo == "cent":
                raise ValueError(f"{h} needs a gossip algorithm: cent keeps theta identical on every rank")
            if self.sync_mode != "iter":
                raise ValueError(f"{h} needs --sync-mode iter: a measurement waits for every rank, and async mode "
                                 "promises no cross-rank waits in the step loop")
            if self.backend == "refport":
                raise ValueError(f"{h} is not supported by --backend refport")
        Q = self.gossip_rounds
        if isinstance(Q, bool) or not isinstance(Q, int) or Q < 1:
            raise ValueError(f"--gossip-rounds must be an integer >= 1, got {Q!r}")
        if Q > 1:
            # the mix-only rounds exist for decent in front of the fused single-kernel ring, double-buffered ring and
            # static-graph steps (csrc/gossip_rounds.cu), the torch.distributed backends and the simulator
            self._validate_rounds(f"--gossip-rounds {Q}")
        from .parallel.topology import ACCELS
        if self.gossip_accel not in ACCELS:
            raise ValueError(f"--gossip-accel must be one of {'|'.join(ACCELS)}, got {self.gossip_accel!r}")
        if self.gossip_accel != "none":
            self._validate_gossip_accel()
        from .parallel.topology import check_match_seed, is_match
        check_match_seed(self.topology_seed)
        if is_match(self.topology):
            self._validate_random_match()
        if self.partition not in ("iid", "label"):
            raise ValueError(f"partition must be iid|label, got {self.partition!r}")
        return self

    def _validate_rounds(self, h: str) -> None:
        """The combinations the round kernel ahead of the step does not support, each with its reason; `h` names the
        flag in the message."""
        if self.algo != "decent":
            raise ValueError(f"{h} needs algo decent, got {self.algo!r}"
                             + ("" if self.algo == "cent" else ": the trigger decides what a step sends, and a "
                                "mix-only round would send every tensor"))
        if str(self.topology).strip().lower() == "onepeer-exp":
            raise ValueError(f"{h} does not support topology onepeer-exp: its single active slot per step has no "
                             "rule for extra rounds")
        if self.compress != "none":
            raise ValueError(f"{h} does not support --compress {self.compress}: a mix-only round would have to "
                             "encode and replicate its own deltas")
        if self.gradient_tracking:
            raise ValueError(f"{h} does not support --gradient-tracking: y would need rounds of its own")
        if self.exact_diffusion:
            raise ValueError(f"{h} does not support --exact-diffusion: its step gossips phi, not theta")
        if self.local_steps > 1:
            raise ValueError(f"{h} does not support --local-steps {self.local_steps}")
        if self.global_avg_period:
            raise ValueError(f"{h} does not support --global-avg-period: an averaging step has no mix to repeat")
        if self.slowmo_period:
            raise ValueError(f"{h} does not support --slowmo-period: a sync step has no mix to repeat")
        if self.quasi_global_momentum:
            raise ValueError(f"{h} does not support --quasi-global-momentum: its theta_k is overwritten by the "
                             "rounds before the step kernel reads it")
        if self.backend == "refport":
            raise ValueError(f"{h} is not supported by --backend refport")
        for name in ("overlap_push", "ce_push"):
            if getattr(self, name):
                raise ValueError(f"{h} does not support {name}: the rounds overwrite theta, which the forward "
                                 "reads, so they cannot run under backward")
        if self.file_write:
            raise ValueError(f"{h} does not support file_write: the reference's log format records one exchange "
                             "per step")

    def _validate_gossip_accel(self) -> None:
        """--gossip-accel chebyshev runs the round kernel (csrc/gossip_rounds.cu) for every one of the Q rounds and then
        the serial step kernel, so it takes every restriction of --gossip-rounds > 1, even at Q = 1, and a few of its
        own.  Each rejection says why."""
        h = f"--gossip-accel {self.gossip_accel}"
        topo = str(self.topology).strip().lower()
        if topo in ("onepeer-exp", "random-match"):
            raise ValueError(f"{h} does not support topology {topo}: a time-varying W has no fixed spectrum to fit the "
                             "polynomial to")
        if self.sync_mode != "iter":
            raise ValueError(f"{h} needs --sync-mode iter: every exchange is in the synchronous rounds, there is nothing "
                             "left to relax")
        if self.double_buffer:
            raise ValueError(f"{h} does not support double_buffer: the step after the rounds exchanges nothing, so it "
                             "has no inbox to double")
        if self.gossip_rounds == 1:
            self._validate_rounds(h)            # the rounds path runs at Q = 1 too (Q > 1 was checked already)

    def _validate_random_match(self) -> None:
        """--topology random-match exists for decent in iter-sync mode: the fused single-inbox step (csrc/gossip_match.cu),
        the torch.distributed backends and the simulator.  Each rejection says why."""
        h = "--topology random-match"
        if self.algo in ("event", "spevent"):
            raise ValueError(f"{h} needs algo decent, got {self.algo!r}: a single inbox holds whichever peer wrote last, "
                             "so a tensor that did not fire would mix with another rank's stale copy")
        if self.algo != "decent":
            raise ValueError(f"{h} needs algo decent, got {self.algo!r}: cent averages every gradient, it has no graph")
        if self.sync_mode != "iter":
            raise ValueError(f"{h} needs --sync-mode iter: a single inbox holds whichever peer wrote last, so an async "
                             "mix could read another rank's stale copy")
        if self.local_steps > 1:
            raise ValueError(f"{h} does not support --local-steps {self.local_steps}")
        if self.global_avg_period:
            raise ValueError(f"{h} does not support --global-avg-period")
        if self.slowmo_period:
            raise ValueError(f"{h} does not support --slowmo-period")
        if self.gossip_rounds > 1:
            raise ValueError(f"{h} does not support --gossip-rounds {self.gossip_rounds}: a round would need a "
                             "matching of its own")
        if self.compress != "none":
            raise ValueError(f"{h} does not support --compress {self.compress}: the replicas of a compressed peer "
                             "assume a fixed neighbour")
        if self.choco_gamma:
            raise ValueError(f"{h} does not support --choco-gamma")
        if self.gradient_tracking:
            raise ValueError(f"{h} does not support --gradient-tracking")
        if self.exact_diffusion:
            raise ValueError(f"{h} does not support --exact-diffusion")
        if self.quasi_global_momentum:
            raise ValueError(f"{h} does not support --quasi-global-momentum")
        if self.backend == "refport":
            raise ValueError(f"{h} is not supported by --backend refport (ring only)")
        for name in ("overlap_push", "double_buffer", "ce_push"):
            if getattr(self, name):
                raise ValueError(f"{h} does not support {name} (fused single-kernel step only)")
        if self.file_write:
            raise ValueError(f"{h} does not support file_write: the reference's log format has exactly one left and "
                             "one right receive column")

    @property
    def ring_topology(self) -> bool:
        """True when `topology` names the ring (ring or the single offset 1).  The restrictions of validate() apply by
        this name, independent of the world size; a name that resolves to the ring for the actual world (exp at
        R <= 3) becomes "ring" in resolved() / for_world(), and then gets the ring's code path AND defaults."""
        return str(self.topology).strip().lower() in ("ring", "1")

    def for_world(self, world: int) -> "TrainConfig":
        """This config with `topology` resolved for `world` ranks: a graph whose offsets are {1} is the ring (named
        "ring", so the ring defaults -- double-buffered inbox, overlapped pushes -- apply).  Raises ValueError for
        offsets out of range for `world`."""
        if self.ring_topology:
            return self
        from .parallel.topology import is_match, is_onepeer, parse_topology
        if is_onepeer(self.topology) or is_match(self.topology):   # time-varying: the ring only with no peer at all
            ring = world == 1
        else:
            ring = parse_topology(self.topology, world) == (1,)
        if not ring and self.compress != "none":
            raise ValueError(f"--compress {self.compress} runs on the ring only; topology {self.topology!r} is not "
                             "the ring for "
                             f"{world} ranks")
        return dataclasses.replace(self, topology="ring") if ring else self

    def resolved(self, device_type: str, world: int) -> "TrainConfig":
        """Fill the auto (None) execution switches for the device the job actually runs on: on a GPU the fast path
        (NHWC + fused BN kernels, whole-step CUDA graph, pushes overlapped with backward) IS the default path.
        The topology is resolved for `world` first (for_world): a graph that is the ring there gets the ring defaults."""
        c = self.for_world(world)
        cuda = device_type == "cuda"
        p2p = c.backend == "p2p" or (c.backend == "auto" and cuda)
        kw = {}
        conv_tc = c.conv_tc
        if conv_tc is None:
            import os
            conv_tc = kw["conv_tc"] = bool(cuda and c.dtype == "fp32" and os.environ.get("EGB_CONV_TC", "1") != "0")
        if c.channels_last is None:
            # bf16 / tf32 / fp32 on our tensor-core convolutions: NHWC.  fp32 on cuDNN (conv_tc off): its IEEE-fp32
            # convolutions are NCHW kernels -- fed NHWC they transpose around every conv -- so that path stays NCHW;
            # the fused BN kernels exist for both layouts
            kw["channels_last"] = cuda and (c.dtype != "fp32" or conv_tc)
        if c.cuda_graph is None:
            kw["cuda_graph"] = cuda
        if c.overlap_push is None:
            kw["overlap_push"] = bool(cuda and p2p and world >= 2 and c.algo in ("decent", "event")
                                      and not bool(c.double_buffer) and c.ring_topology and c.compress == "none"
                                      and not c.gradient_tracking and c.local_steps == 1
                                      and not c.exact_diffusion and not c.global_avg_period
                                      and not c.slowmo_period and c.gossip_rounds == 1
                                      and c.gossip_accel == "none")
        return dataclasses.replace(c, **kw) if kw else c

    def replace(self, **kw) -> "TrainConfig":
        return dataclasses.replace(self, **kw)


# Presets = the constants hard-coded in each reference program (SURVEY.md 2.6).
PRESETS = {
    # dmnist/cent/cent.cpp:62-65,75,95  (full batch per rank, lr 1e-2, 250 epochs, random sampler)
    "cent": dict(algo="cent", dataset="mnist", model="mlp", epochs=250, batch_mode="full",
                 lr=1e-2, momentum=0.0, sampler="random", train_samples=60000, augment=False),
    # dmnist/decent/decent.cpp:83-86,121,139 (full batch, lr 1e-2, 50 epochs, sequential)
    "decent": dict(algo="decent", dataset="mnist", model="mlp", epochs=50, batch_mode="full",
                   lr=1e-2, momentum=0.0, sampler="sequential", train_samples=60000,
                   augment=False, sync_mode="iter"),
    # dmnist/event/event.cpp:145,227-230,255 (batch 64 per rank, lr 0.05, 10 epochs, sequential)
    "mnist_event": dict(algo="event", dataset="mnist", model="cnn2", epochs=10, batch_size=64,
                        batch_mode="per_rank", lr=0.05, momentum=0.0, sampler="sequential",
                        train_samples=60000, augment=False),
    # dcifar10/event/event.cpp:29-42,91,196-200
    "cifar_event": dict(algo="event", dataset="cifar10", model="resnet18", epochs=20,
                        batch_size=256, batch_mode="global", lr=1e-2, momentum=0.9,
                        sampler="random", train_samples=50000, augment=True),
    # dcifar10/spevent/spevent.cpp:32-37,60,219-223
    "cifar_spevent": dict(algo="spevent", dataset="cifar10", model="resnet18", epochs=20,
                          batch_size=256, batch_mode="global", lr=1e-2, momentum=0.9,
                          sampler="random", train_samples=50000, augment=True),
}


def preset(name: str, **overrides) -> TrainConfig:
    base = dict(PRESETS[name])
    base.update(overrides)
    return TrainConfig(**base).validate()


def _add_common_flags(p: argparse.ArgumentParser) -> None:
    d = TrainConfig()
    p.add_argument("--model", default=None)
    p.add_argument("--resnet-variant", default=None, choices=["ref", "canonical"])
    p.add_argument("--epochs", type=int, default=None)
    p.add_argument("--batch-size", type=int, default=None)
    p.add_argument("--batch-mode", default=None, choices=["global", "per_rank", "full"])
    p.add_argument("--lr", type=float, default=None)
    p.add_argument("--momentum", type=float, default=None)
    p.add_argument("--weight-decay", type=float, default=None, help="L2 weight decay on every parameter (default 0)")
    p.add_argument("--nesterov", action=argparse.BooleanOptionalAction, default=None,
                   help="Nesterov momentum (needs --momentum > 0)")
    p.add_argument("--lr-schedule", default=None, choices=["constant", "step", "multistep", "cosine"])
    p.add_argument("--lr-step-epochs", type=int, default=None, help="step schedule: period in epochs")
    p.add_argument("--lr-milestones", type=lambda s: tuple(int(x) for x in s.split(",") if x.strip()), default=None,
                   metavar="E1,E2,...", help="multistep schedule: epochs at which lr is multiplied by --lr-gamma")
    p.add_argument("--lr-gamma", type=float, default=None)
    p.add_argument("--lr-min", type=float, default=None, help="cosine schedule: final learning rate")
    p.add_argument("--lr-warmup-epochs", type=float, default=None, help="linear warm-up, stepped per step")
    p.add_argument("--seed", type=int, default=None)
    p.add_argument("--sent-history", type=int, default=None)
    p.add_argument("--initial-comm-passes", type=int, default=None)
    p.add_argument("--trigger", default=None, choices=["norm", "drift"],
                   help="event trigger: norm (default, the reference rule: |norm - norm at last send| >= threshold) or "
                        "drift (||theta - what the neighbours hold|| >= threshold; event/spevent)")
    p.add_argument("--backend", default=None, choices=["auto", "p2p", "nccl", "gloo", "refport"])
    p.add_argument("--sync-mode", default=None, choices=["iter", "async"])
    p.add_argument("--overlap-push", action=argparse.BooleanOptionalAction, default=None,
                   help="default: on for decent/event on >= 2 GPUs")
    p.add_argument("--double-buffer", action=argparse.BooleanOptionalAction, default=None)
    p.add_argument("--peer-timeout-s", type=float, default=None)
    p.add_argument("--ce-push", action="store_true", default=None)
    p.add_argument("--topology", default=None, metavar="ring|exp|onepeer-exp|random-match|O1,O2,...",
                   help="gossip graph: ring (default), exp (offsets 1,2,4,... up to R/2), explicit circulant offsets, "
                        "onepeer-exp (time-varying: at step k push to r + 2^((k-1) mod ceil(log2 R)) only, "
                        "mix (theta + received) / 2), or random-match (decent: a random perfect matching per step, "
                        "seeded by --topology-seed; each rank averages with its partner, one idle rank at odd R)")
    p.add_argument("--topology-seed", type=int, default=None, metavar="S",
                   help="random-match: seed in [0, 2^31) of the per-step matchings, the same on every rank (default 0)")
    p.add_argument("--compress", default=None, choices=["none", "int8", "sign"],
                   help="decent/event on the ring: send the int8 code of theta - (what the neighbours hold) with one "
                        "fp32 scale per 256 elements, about a quarter of the fp32 bytes, or its 1-bit scaled sign, "
                        "about 1/28 (sign; pair it with --choco-gamma) (default none)")
    p.add_argument("--choco-gamma", type=float, default=None, metavar="GAMMA",
                   help="--compress int8/sign: mix by CHOCO-SGD's consensus step theta += GAMMA * (W prev - prev) on "
                        "the public copies, which keeps the ranks' average; 0 < GAMMA <= 1, small for the sign codec "
                        "(default 0: the error-feedback mix)")
    p.add_argument("--gradient-tracking", action="store_true", default=None,
                   help="decent on the ring: also gossip y, a running estimate of the average gradient, and step along "
                        "it (DSGT): removes the bias of constant-lr D-PSGD under heterogeneous data")
    p.add_argument("--local-steps", type=int, default=None, metavar="H",
                   help="decent: gossip only at every H-th step and take plain local SGD steps in between (local "
                        "D-PSGD); sends 1/H of the bytes (default 1: every step)")
    p.add_argument("--exact-diffusion", action="store_true", default=None,
                   help="decent on the ring: exact diffusion (D^2 on (I + W)/2): step before the push and gossip "
                        "phi = p + theta - psi; removes the bias of constant-lr D-PSGD under heterogeneous data at "
                        "decent's bytes")
    p.add_argument("--global-avg-period", type=int, default=None, metavar="P",
                   help="decent on the ring or a static graph: every P-th step (P >= 2) replaces the gossip mix with "
                        "an exact average of the parameters over all ranks (Gossip-PGA; default 0: off)")
    p.add_argument("--quasi-global-momentum", action="store_true", default=None,
                   help="decent/event/spevent with --momentum > 0: build each rank's momentum from its own parameter "
                        "displacement (mix included) instead of its gradient (QG-DSGDm); removes momentum's "
                        "1/(1 - mu) amplification of the heterogeneity bias at unchanged bytes")
    p.add_argument("--slowmo-period", type=int, default=None, metavar="TAU",
                   help="decent on the ring or a static graph: every TAU-th step (TAU >= 2) averages the parameters "
                        "exactly and takes a slow heavy-ball step on the average from where the cycle started (SlowMo); "
                        "the base steps gossip (--local-steps 1) or are local SGD (--local-steps TAU) (default 0: off)")
    p.add_argument("--slowmo-beta", type=float, default=None, metavar="BETA",
                   help="SlowMo slow momentum, 0 <= BETA < 1 (default 0.5; 0 with --slowmo-lr 1 is plain periodic "
                        "averaging)")
    p.add_argument("--slowmo-lr", type=float, default=None, metavar="ALPHA",
                   help="SlowMo slow learning rate, ALPHA > 0 (default 1.0)")
    p.add_argument("--consensus-every", type=int, default=None, metavar="N",
                   help="decent/event/spevent: after every N-th step measure how far the ranks' parameters are from "
                        "their average, per tensor, without changing training; rank 0 prints the relative distance "
                        "per epoch and --log-dir gets consensus.csv and consensus_tensors.csv (default 0: off)")
    p.add_argument("--gossip-rounds", type=int, default=None, metavar="Q",
                   help="decent on the ring or a static graph: mix Q times per step, theta <- W^Q theta, before the "
                        "optimizer step (Q - 1 mix-only rounds, then the step's own); sends Q times the bytes "
                        "(default 1)")
    p.add_argument("--gossip-accel", default=None, choices=["none", "chebyshev"],
                   help="decent on the ring or a static graph: chebyshev runs the --gossip-rounds Q rounds as the "
                        "degree-Q Chebyshev polynomial of the graph's spectrum, P_Q(W) theta, instead of W^Q theta, at "
                        "the same bytes; Q = 1 is the optimally shifted W (default none)")
    p.add_argument("--fresh-replicas", dest="spevent_fresh_replicas", action="store_true", default=None,
                   help="spevent: initialise prev/left/right replicas like the reference (three more random nets)")
    p.add_argument("--no-grad-table", dest="grad_table", action="store_false", default=None)
    p.add_argument("--data", default=None, help="'synthetic' or dataset root directory")
    p.add_argument("--sampler", default=None, choices=["random", "sequential"])
    p.add_argument("--partition", default=None, choices=["iid", "label"],
                   help="data shards: iid (default) or label (cut from the samples sorted by class: each rank sees few "
                        "classes, every shard has the same size)")
    p.add_argument("--no-augment", dest="augment", action="store_false", default=None)
    p.add_argument("--native-loader", default=None, choices=["auto", "on", "off"])
    p.add_argument("--train-samples", type=int, default=None)
    p.add_argument("--test-samples", type=int, default=None)
    p.add_argument("--device", default=None, choices=["auto", "cuda", "cpu"])
    p.add_argument("--dtype", default=None, choices=["fp32", "tf32", "bf16"])
    p.add_argument("--channels-last", action=argparse.BooleanOptionalAction, default=None, help="default: on for CUDA")
    p.add_argument("--cuda-graph", action=argparse.BooleanOptionalAction, default=None, help="default: on for CUDA")
    p.add_argument("--conv-tc", action=argparse.BooleanOptionalAction, default=None,
                   help="fp32: convolutions on the wgmma tensor cores at fp32 accuracy (default: on for CUDA); "
                        "--no-conv-tc = cuDNN's SIMT fp32 kernels")
    p.add_argument("--no-cudnn-benchmark", dest="cudnn_benchmark", action="store_false", default=None)
    p.add_argument("--max-steps", type=int, default=None)
    p.add_argument("--log-dir", default=None)
    p.add_argument("--ckpt-dir", default=None)
    p.add_argument("--ckpt-every", type=int, default=None)
    p.add_argument("--resume", default=None)
    p.add_argument("--quiet", action="store_true", default=None)
    p.add_argument("--phase-timers", action="store_true", default=None)
    del d


def parse_cli(program: str, argv: Optional[Sequence[str]] = None) -> TrainConfig:
    """Parse the CLI of one of the five reference-equivalent programs.

    `program` is one of cent | decent | mnist_event | cifar_event | cifar_spevent.
    Positional arguments follow the reference order; everything else is a flag.
    """
    p = argparse.ArgumentParser(prog=f"eventgrad_b200.cli.{program}",
                                description=f"{program}: reference-compatible positional args + flags")
    if program in ("mnist_event", "cifar_event", "cifar_spevent"):
        p.add_argument("file_write", type=int, nargs="?", default=0)
        p.add_argument("thres_type", type=int, nargs="?", default=1,
                       help="0 constant threshold, 1 adaptive")
        p.add_argument("threshold_arg", type=float, nargs="?", default=1.0,
                       help="horizon if thres_type==1 else the constant threshold")
        if program == "cifar_spevent":
            p.add_argument("topk_percent", type=float, nargs="?", default=10.0)
    elif program == "decent":
        p.add_argument("file_write", type=int, nargs="?", default=0)
    _add_common_flags(p)
    ns = p.parse_args(argv)
    over = {}
    for f in dataclasses.fields(TrainConfig):
        v = getattr(ns, f.name, None)
        if v is not None:
            over[f.name] = v
    if hasattr(ns, "threshold_arg"):
        if over.get("thres_type", 1) == 1:
            over["horizon"] = ns.threshold_arg
        else:
            over["constant"] = ns.threshold_arg
    return preset(program, **over)
