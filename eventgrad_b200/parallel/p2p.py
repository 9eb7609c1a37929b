"""Fused peer-to-peer backend -- the product path.

Per training step, after backward():
  cent     ONE launch: one-/two-shot all-reduce over peer-mapped gradients fused with 1/R and SGD
  decent   ONE launch: push theta to both ring neighbours -> flag handshake -> (t+L+R)/3 -> SGD
           (circulant graph: push into all 2|O| slots I feed -> flags per slot -> (t+s_0+...)/(2|O|+1) -> SGD,
           csrc/gossip_graph.cu; one-peer graph: push into the step's single out-slot m -> slot m's flags ->
           (t+s_m)/2 -> SGD, same kernel)
  event    ONE launch: as decent, but a tensor is pushed only if its device-resident trigger fired;
           the same kernel accumulates the norms and runs the trigger FSM for the next step
           (--compress int8, ring: csrc/gossip_q8.cu pushes the int8 code of theta - prev + block scales, the receivers
           add the delta to their replicas of prev, and the mix reads the replicas; --compress sign sends a 1-bit scaled
           sign instead, and --choco-gamma mixes by CHOCO's theta += gamma * (((prev + rep_l) + rep_r) / 3 - prev))
           (--gradient-tracking, decent on the ring: csrc/gossip_gt.cu also pushes y_{k-1} before the same flag, forms
           y_k = (y + yL + yR)/3 + g_k - g_prev and steps along y_k)
           (--exact-diffusion, decent on the ring: csrc/gossip_ed.cu runs SGD in the push stage, pushes
           phi = p + theta_k - psi, psi <- p, and mixes theta = (phi + (phi + L + R)/3) / 2)
           (--global-avg-period P, decent on the ring / a static graph: TWO launches per step, the two-shot all-reduce
           of theta gated on "P divides the step" (a no-op launch otherwise), then the step kernel, which takes the plain
           SGD step at an averaging step)
           (--slowmo-period tau, decent on the ring / a static graph: TWO launches per step, the SlowMo sync kernel of
           csrc/allreduce.cu gated on "tau divides the step" -- the two-shot average plus the outer update of x and u --
           then the step kernel: the gossip step (local_steps 1, which takes the plain SGD step at a sync step) or the
           serial step (local_steps tau, local SGD))
           (--gossip-rounds Q, decent on the ring / a static graph: Q - 1 mix-only round launches of
           csrc/gossip_rounds.cu before the step kernel, each pushing theta into its own round inboxes and mixing it in
           place with the step's mix)
           (--gossip-accel chebyshev, the same with all Q rounds as Chebyshev round launches, each combining its mix
           with x_{q-1} and x_{q-2}, then the step kernel as the serial step: no push, mix or handshake)
           (--topology random-match, decent: csrc/gossip_match.cu derives this step's partner from the seed, waits for
           the partner's `done` word of the previous step, pushes theta into its single inbox -> flags -> (t+in)/2 ->
           SGD, and publishes `done`; an idle rank of an odd world takes the plain SGD step)
           (--consensus-every N, decent/event/spevent: one more launch per step after the step kernel, the
           consensus kernel of csrc/allreduce.cu gated on "N divides the step that just completed"; it only reads theta
           and writes per-tensor sums into a device ring that drain_consensus() reads at epoch boundaries)
  spevent  batched segmented radix-select top-k + compaction straight into the neighbours'
           inboxes, scatter of arrived records into replicas, then the dense mix+SGD kernel
No NCCL/MPI call, no separate elementwise kernel and no host synchronisation on that path
(BASELINE.json north star).  Kernels: csrc/gossip.cu, csrc/allreduce.cu, csrc/sparse.cu.
"""
from __future__ import annotations

from typing import List

import torch

from .arena import TILE, ParamArena, TensorTable
from .base import (CommBackend, StepLog, check_compress_state, check_exact_diffusion_state, check_global_avg_state,
                   check_choco_state, check_local_steps_state, check_slowmo_state, slowmo_state, check_qg_state, check_topology_state, check_tracking_state,
                   check_trigger_state)
from .topology import Graph, chebyshev_coefficients, is_match
from .trigger import codec_of
from .window import DistBootstrap, Layout, SymmWindow, Window, wants_symm_window

ONE_SHOT_MAX_BYTES = 512 * 1024        # above this the all-reduce switches to two-shot


def default_timeout_ns(cfg=None) -> int:
    """Bound of every device-side peer wait (a wedged / dead peer trips the sticky status word instead of hanging
    the GPU): TrainConfig.peer_timeout_s, overridable with EGB_PEER_TIMEOUT_S."""
    import os
    sec = float(os.environ.get("EGB_PEER_TIMEOUT_S", getattr(cfg, "peer_timeout_s", 30.0) or 30.0))
    return int(sec * 1e9)


def _table_of(model) -> TensorTable:
    return TensorTable.from_named(list(model.named_parameters()), TILE)


def _wants_dbuf(cfg) -> bool:
    """csrc/gossip_dbuf.cu (two inbox slots, no WAR ack) applies to the dense, iter-sync, single-kernel decent step
    only; there it is the default (double_buffer=None), `--no-double-buffer` selects the single-slot + ack protocol."""
    db = getattr(cfg, "double_buffer", None)
    return ((db is None or bool(db)) and cfg.algo == "decent" and cfg.sync_mode == "iter"
            and not getattr(cfg, "overlap_push", False) and getattr(cfg, "ring_topology", True)
            and not _wants_q8(cfg) and not getattr(cfg, "gradient_tracking", False)
            and getattr(cfg, "local_steps", 1) == 1 and not getattr(cfg, "exact_diffusion", False)
            and not getattr(cfg, "global_avg_period", 0) and not getattr(cfg, "slowmo_period", 0)
            and getattr(cfg, "gossip_accel", "none") == "none")


def _wants_q8(cfg) -> bool:
    """--compress int8 / sign: decent/event on the ring run the compressed step of csrc/gossip_q8.cu."""
    return getattr(cfg, "compress", "none") in ("int8", "sign") and cfg.algo in ("decent", "event")


def _wants_gt(cfg, world: int) -> bool:
    """--gradient-tracking: decent on the ring of >= 2 ranks runs the tracking step of csrc/gossip_gt.cu (at R = 1
    tracking is plain SGD on the gradient, the existing path)."""
    return bool(getattr(cfg, "gradient_tracking", False)) and cfg.algo == "decent" and world > 1


def _wants_ed(cfg, world: int) -> bool:
    """--exact-diffusion: decent on the ring of >= 2 ranks runs the exact-diffusion step of csrc/gossip_ed.cu (at R = 1
    it is the plain serial step, the existing path)."""
    return bool(getattr(cfg, "exact_diffusion", False)) and cfg.algo == "decent" and world > 1


def _graph_of(cfg, rank: int, world: int):
    """The circulant graph (or random matching) of a non-ring topology, or None when the topology resolves to the ring."""
    g = Graph.build(rank, world, getattr(cfg, "topology", "ring"), seed=getattr(cfg, "topology_seed", 0))
    return None if g.is_ring else g


def _wants_consensus(cfg, world: int) -> bool:
    """--consensus-every N on a gossip algorithm with peers: the consensus kernel runs, and the window gets its
    partial buffer.  At R = 1 every measurement is zero and nothing is launched."""
    return bool(getattr(cfg, "consensus_every", 0)) and cfg.algo in ("decent", "event", "spevent") and world > 1


def _add_consensus(lay: Layout, table: TensorTable, cfg, world: int) -> Layout:
    """The consensus kernel's partial buffer, last in the window and only with the flag on, so every other window
    keeps its layout: two fp64 sums per (tile, warp), written by the tile's owner into every rank's copy."""
    if _wants_consensus(cfg, world):
        lay.add("cons_part", table.n_tiles * 8 * 2 * 8)
    return lay


def _wants_cheb(cfg) -> bool:
    """--gossip-accel chebyshev: every one of the Q rounds is a Chebyshev round kernel launch, then the serial step."""
    return getattr(cfg, "gossip_accel", "none") == "chebyshev"


def _rounds_per_step(cfg) -> int:
    """Round kernel launches per step: Q - 1 ahead of the step kernel's own mix under --gossip-rounds Q, all Q under
    --gossip-accel chebyshev (whose step kernel then mixes nothing).  The round handshake counter of round q of step k
    is h = n (k - 1) + q with n this number."""
    Q = int(getattr(cfg, "gossip_rounds", 1))
    return Q if _wants_cheb(cfg) else Q - 1


def _wants_rounds(cfg, world: int) -> bool:
    """--gossip-rounds Q >= 2, or --gossip-accel chebyshev at any Q, on decent with peers: the round kernel runs, and
    the window gets its sections.  At R = 1 nothing extra runs."""
    return _rounds_per_step(cfg) >= 1 and cfg.algo == "decent" and world > 1


def _add_rounds(lay: Layout, table: TensorTable, cfg, world: int, n_slots: int) -> Layout:
    """The round kernel's sections, appended last and only with Q > 1, so every other window keeps its layout: one
    inbox, one (tile, warp) flag block and one ack word per slot (csrc/gossip_rounds.cu)."""
    if _wants_rounds(cfg, world):
        for k in range(n_slots):
            lay.add(f"round_inbox_{k}", table.n_padded * 4)
        for k in range(n_slots):
            lay.add(f"round_flag_{k}", (table.n_tiles * 8 + 64) * 4)
            lay.add(f"round_ack_{k}", 256)
    return lay


def build_layout(table: TensorTable, cfg, world: int, max_grid: int, graph=None) -> Layout:
    lay = Layout()
    n = table.n_padded * 4
    lay.add("theta", n)
    lay.add("grad", n)
    nflag = (table.n_tiles * 8 + 64) * 4      # one flag per (tile, warp)
    if is_match(graph):
        # random matchings: ONE inbox, one (tile, warp) flag block and one `done` word, whoever the sender
        # (csrc/gossip_match.cu)
        lay.add("match_inbox", n)
        lay.add("match_flag", nflag)
        lay.add("match_done", 256)
        lay.add("ar_flags", 3 * max_grid * world * 4)
        return _add_consensus(lay, table, cfg, world)
    if graph is not None:
        # circulant graph: one inbox, one flag block and one ack word per slot (csrc/gossip_graph.cu)
        for k in range(graph.n_slots):
            lay.add(f"inbox_{k}", n)
        for k in range(graph.n_slots):
            lay.add(f"flag_from_{k}", nflag)
            lay.add(f"ack_from_{k}", 256)
        lay.add("ar_flags", 3 * max_grid * world * 4)
        return _add_rounds(_add_consensus(lay, table, cfg, world), table, cfg, world, graph.n_slots)
    if _wants_q8(cfg):
        # int8 codes (one byte per arena element) and one fp32 scale per (tile, warp) block from each neighbour
        lay.add("q_from_l", table.n_padded)
        lay.add("q_from_r", table.n_padded)
        lay.add("qs_from_l", table.n_tiles * 8 * 4)
        lay.add("qs_from_r", table.n_tiles * 8 * 4)
    elif cfg.algo in ("decent", "event"):
        slots = 2 if _wants_dbuf(cfg) else 1      # double-buffered decent: slot = step & 1
        lay.add("inbox_l", n * slots)
        lay.add("inbox_r", n * slots)
        if _wants_gt(cfg, world):
            lay.add("y_in_l", n)                  # gradient tracking: y from each neighbour
            lay.add("y_in_r", n)
        if _wants_ed(cfg, world):
            lay.add("psi", n)                     # exact diffusion: the previous optimizer output (this rank only)
    if cfg.algo == "spevent":
        K = sum(table.topk_counts(cfg.topk_percent))
        lay.add("rec_from_l", 2 * K * 4)
        lay.add("rec_from_r", 2 * K * 4)
        lay.add("seq_from_l", table.n_tensors * 4)
        lay.add("seq_from_r", table.n_tensors * 4)
        lay.add("done_from_l", 256)
        lay.add("done_from_r", 256)
    lay.add("flag_from_l", nflag)
    lay.add("flag_from_r", nflag)
    lay.add("ack_from_l", 256)
    lay.add("ack_from_r", 256)
    lay.add("pushed_from_l", 256)
    lay.add("pushed_from_r", 256)
    lay.add("ar_flags", 3 * max_grid * world * 4)
    return _add_rounds(_add_consensus(lay, table, cfg, world), table, cfg, world, 2)


def preallocate_arena_buffers(model, cfg, env, group=None, bootstrap=None):
    """Allocate this rank's window BEFORE the arena exists so that theta and grad live inside
    peer-mapped memory (cent reads peers' gradients; final averaging reads peers' theta)."""
    from ..ops import ext
    C = ext()
    table = _table_of(model)
    max_grid = C.gossip_max_grid(env.device.index or 0)
    graph = _graph_of(cfg, env.rank, env.world) if cfg.algo in ("decent", "event") else None
    if _wants_dbuf(cfg):
        max_grid = min(max_grid, C.gossip_dbuf_max_grid(env.device.index or 0))
    if is_match(graph):
        max_grid = min(max_grid, C.gossip_match_max_grid(env.device.index or 0))
    elif graph is not None:
        max_grid = min(max_grid, C.gossip_graph_max_grid(env.device.index or 0))
    if _wants_q8(cfg):
        max_grid = min(max_grid, C.gossip_q8_max_grid(env.device.index or 0))
    if _wants_gt(cfg, env.world):
        max_grid = min(max_grid, C.gossip_gt_max_grid(env.device.index or 0))
    if _wants_ed(cfg, env.world):
        max_grid = min(max_grid, C.gossip_ed_max_grid(env.device.index or 0))
    if _wants_rounds(cfg, env.world):
        max_grid = min(max_grid, C.gossip_rounds_max_grid(env.device.index or 0))
    if _wants_consensus(cfg, env.world):
        # the query loads the consensus kernel now: enqueued behind spinning step kernels, a lazy load at its first
        # launch could wait for them to finish
        max_grid = min(max_grid, C.consensus_max_grid(env.device.index or 0))
    lay = build_layout(table, cfg, env.world, max_grid, graph)
    symm = wants_symm_window(env) and bootstrap is None      # NVLS path: torch symmetric memory + multicast mapping
    win = (SymmWindow if symm else Window)(lay, env.rank, env.world, env.device)
    theta = win.view("theta", torch.float32)
    grad = win.view("grad", torch.float32)
    return theta, grad, {"window": win, "max_grid": max_grid, "bootstrap": bootstrap}


class P2PBackend(CommBackend):
    name = "p2p"
    zeroes_grad = True     # the fused kernels clear grad after consuming it

    def __init__(self, cfg, arena: ParamArena, ring, env, group=None, symm=None,
                 grid_cap: int = 0, defer_connect: bool = False, group_iters: int = 2,
                 timeout_ns: int = 0, push_grid: int = 0):
        super().__init__(cfg, arena, ring)
        from ..ops import ext
        self.C = ext()
        if symm is None:
            raise ValueError("P2PBackend needs the window that holds the arena (preallocate_arena_buffers)")
        self.env, self.dev = env, arena.theta.device
        self.win: Window = symm["window"]
        self.boot = symm.get("bootstrap") or DistBootstrap(env, group)
        self.table = arena.table
        t = self.table
        if t.n_tensors > 1024:
            raise ValueError("p2p backend supports at most 1024 parameter tensors (EG_MAX_OWN)")
        self.grid = min(t.n_tiles, symm["max_grid"])
        if grid_cap:
            self.grid = min(self.grid, grid_cap)
        # balance: every CTA gets the same number of tiles (+-1 only on the last round)
        rounds = -(-t.n_tiles // self.grid)
        self.grid = -(-t.n_tiles // rounds)
        self.group_iters, self.timeout_ns = group_iters, timeout_ns or default_timeout_ns(cfg)
        self.sync = cfg.sync_mode == "iter"
        self.gossip = cfg.algo in ("decent", "event", "spevent")
        self.sparse = cfg.algo == "spevent"
        self.do_comm = self.comm_enabled and self.gossip
        # circulant graph beyond the ring (parallel/topology.py): the fused single-kernel step of csrc/gossip_graph.cu
        self.graph = None if getattr(ring, "is_ring", True) else ring
        # --topology random-match: the single-inbox step of csrc/gossip_match.cu (decent, iter-sync, fused step only)
        self.match = ring if is_match(ring) else None
        if self.match is not None:
            self.graph = None
            if (cfg.algo != "decent" or not self.sync or getattr(cfg, "overlap_push", False)
                    or getattr(cfg, "ce_push", False) or self.want_logs):
                raise ValueError("p2p backend: random-match runs decent on the fused iter-sync step only")
        if self.graph is not None and (cfg.algo not in ("decent", "event") or getattr(cfg, "overlap_push", False)
                                       or getattr(cfg, "ce_push", False) or self.want_logs):
            raise ValueError("p2p backend: a non-ring topology runs decent/event on the fused step only")
        # split step: everything that depends only on theta_k (pushes / top-k records) is launched on a
        # side stream at the start of the step and overlaps forward+backward
        self.overlap = bool(getattr(cfg, "overlap_push", False)) and self.do_comm
        # --compress int8 / sign: the iter-sync fused ring step of csrc/gossip_q8.cu; --choco-gamma selects its CHOCO mix
        self.q8 = _wants_q8(cfg)
        self.compress = cfg.compress if self.q8 else "none"
        self.choco_gamma = float(getattr(cfg, "choco_gamma", 0.0)) if self.q8 else 0.0
        if self.q8 and (self.graph is not None or self.overlap or getattr(cfg, "ce_push", False) or self.want_logs
                        or not self.sync):
            raise ValueError(f"p2p backend: --compress {self.compress} runs decent/event on the ring's fused iter-sync "
                             "step only")
        # --gradient-tracking: the iter-sync fused single-slot ring step of csrc/gossip_gt.cu
        self.gt = _wants_gt(cfg, ring.world) and self.do_comm
        if self.gt and (self.graph is not None or self.overlap or getattr(cfg, "ce_push", False) or self.want_logs
                        or not self.sync or self.q8):
            raise ValueError("p2p backend: --gradient-tracking runs decent on the ring's fused iter-sync step only")
        # --exact-diffusion: the iter-sync fused single-slot ring step of csrc/gossip_ed.cu
        self.ed = _wants_ed(cfg, ring.world) and self.do_comm
        if self.ed and (self.graph is not None or self.overlap or getattr(cfg, "ce_push", False) or self.want_logs
                        or not self.sync or self.q8 or self.gt):
            raise ValueError("p2p backend: --exact-diffusion runs decent on the ring's fused iter-sync step only")
        # --local-steps H (decent): the fused single-slot ring / graph step gossips at every H-th step only; the
        # kernel takes that choice from its device step counter, so one captured launch serves the whole cycle
        self.local_steps = int(getattr(cfg, "local_steps", 1)) if cfg.algo == "decent" else 1
        if getattr(cfg, "local_steps", 1) > 1 and (cfg.algo != "decent" or self.overlap or self.q8 or self.gt
                                                   or self.ed or getattr(cfg, "ce_push", False) or self.want_logs):
            raise ValueError("p2p backend: --local-steps runs decent on the fused single-kernel step only")
        # --global-avg-period P (decent): the gated all-reduce of theta, then the fused single-slot ring / static-graph
        # step; both take "does P divide this step" from the device pass counter, so one captured pair serves the cycle
        self.global_avg_period = int(getattr(cfg, "global_avg_period", 0)) if cfg.algo == "decent" else 0
        if getattr(cfg, "global_avg_period", 0) and (
                cfg.algo != "decent" or self.overlap or self.q8 or self.gt or self.ed or self.local_steps > 1
                or getattr(cfg, "ce_push", False) or self.want_logs or getattr(self.graph, "period", 0)):
            raise ValueError("p2p backend: --global-avg-period runs decent on the fused single-kernel ring / static "
                             "graph step only")
        # --quasi-global-momentum: the ring, double-buffered and graph step kernels update m_hat from theta_k (re-read
        # after the mix) at every step, gossip, local or serial alike
        self.qg = self.gossip and bool(getattr(cfg, "quasi_global_momentum", False))
        if self.qg and (cfg.momentum == 0 or not self.sync or self.q8 or self.gt or self.ed or self.global_avg_period
                        or getattr(cfg, "ce_push", False)):
            raise ValueError("p2p backend: --quasi-global-momentum runs the ring, double-buffered and graph step "
                             "kernels with momentum and iter-sync, without int8, tracking, exact diffusion, global "
                             "averaging or ce_push")
        # --slowmo-period tau (decent): the gated SlowMo sync kernel, then the fused single-slot ring / static-graph step
        # as the gossip base (local_steps 1) or the serial step as the local-SGD base (local_steps tau, on every
        # topology: that base never exchanges).  x and u live in local device memory, identical on every rank
        self.slowmo_period = int(getattr(cfg, "slowmo_period", 0)) if cfg.algo == "decent" else 0
        self.slowmo_beta = float(getattr(cfg, "slowmo_beta", 0.5))
        self.slowmo_lr = float(getattr(cfg, "slowmo_lr", 1.0))
        self.slowmo_local = bool(self.slowmo_period) and self.local_steps == self.slowmo_period
        if self.slowmo_period and (self.overlap or self.q8 or self.gt or self.ed or self.qg or self.global_avg_period
                                   or self.local_steps not in (1, self.slowmo_period) or getattr(cfg, "ce_push", False)
                                   or self.want_logs or getattr(self.graph, "period", 0)):
            raise ValueError("p2p backend: --slowmo-period runs decent on the fused single-kernel ring / static graph "
                             "step with --local-steps 1 or tau only")
        self.slowmo_x = self.slowmo_u = None
        # --gossip-rounds Q (decent, R >= 2): Q - 1 launches of the round kernel before the unchanged ring,
        # double-buffered ring or static-graph step kernel
        self.gossip_rounds = int(getattr(cfg, "gossip_rounds", 1))
        self.rounds = _wants_rounds(cfg, ring.world) and self.do_comm
        if self.gossip_rounds > 1 and (cfg.algo != "decent" or self.overlap or self.q8 or self.gt or self.ed
                                       or self.local_steps > 1 or self.global_avg_period or self.slowmo_period
                                       or self.qg or getattr(cfg, "ce_push", False) or self.want_logs or not self.sync
                                       or getattr(self.graph, "period", 0)):
            raise ValueError("p2p backend: --gossip-rounds runs decent on the fused single-kernel ring, "
                             "double-buffered ring or static graph step only")
        self.round_ticket = None
        # --gossip-accel chebyshev: all Q rounds are Chebyshev round launches (x_{q-1} kept in `cheb_prev`, local and
        # outside the window), then the step kernel runs as the serial step: no push, no mix, no handshake
        self.cheb = _wants_cheb(cfg) and self.rounds
        if _wants_cheb(cfg) and (cfg.algo != "decent" or self.overlap or getattr(cfg, "double_buffer", None)
                                 or self.q8 or self.gt or self.ed or self.local_steps > 1 or self.global_avg_period
                                 or self.slowmo_period or self.qg or getattr(cfg, "ce_push", False) or self.want_logs
                                 or not self.sync or getattr(self.graph, "period", 0) or self.match is not None):
            raise ValueError("p2p backend: --gossip-accel chebyshev runs decent on the ring or a static graph, with "
                             "the serial step after the rounds, only")
        self.cheb_prev = self.d_cheb_coef = None
        if self.match is not None and (self.q8 or self.gt or self.ed or self.local_steps > 1 or self.global_avg_period
                                       or self.slowmo_period or self.qg or self.gossip_rounds > 1):
            raise ValueError("p2p backend: random-match runs plain decent only (no compression, tracking, exact "
                             "diffusion, local steps, global averaging, slowmo, quasi-global momentum or gossip rounds)")
        # --consensus-every N: the gated consensus kernel after the step kernel (R >= 2); its rows wait in a device
        # ring of `cons_cap` rows until drain_consensus().  At R = 1 account_step() records the zero rows itself
        self.consensus_every = int(getattr(cfg, "consensus_every", 0)) if self.gossip else 0
        if self.consensus_every and not self.sync:
            raise ValueError("p2p backend: --consensus-every needs iter-sync")
        self.cons = _wants_consensus(cfg, ring.world)
        self.cons_cap = 1024
        self._cons_held = []           # rows read from the ring (or recorded at R = 1) and not yet returned
        self._cons_drained = 0         # ring rows read so far
        self.cp = self.cp_now = None
        self.dbuf = _wants_dbuf(cfg) and self.do_comm
        self.ce_push = bool(getattr(cfg, "ce_push", False)) and self.overlap and cfg.algo == "decent" and self.sync
        self.nvls = self.nvls_step = False      # set in connect() when the window has a multicast mapping
        self.wire_dedup = False
        self.push_grid = push_grid
        self.recv_rms = cfg.dataset == "mnist"
        dev = self.dev
        i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=dev)
        zf = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        zi = lambda *s: torch.zeros(*s, dtype=torch.int32, device=dev)
        # ---- device tables ---------------------------------------------------------------
        self.d_tile_tensor = t.tile_to_tensor().to(dev)
        self.d_tile_start, self.d_tile_count, self.d_numel = i32(t.tile_start), i32(t.tile_count), i32(t.numels)
        if self.sparse:
            self.k = t.topk_counts(cfg.topk_percent)
            msg = [2 * k * 4 for k in self.k]
            rec_off, acc = [], 0
            for k in self.k:
                rec_off.append(acc)
                acc += 2 * k
            self.K = sum(self.k)
            self.d_k, self.d_rec_off = i32(self.k), i32(rec_off)
        elif self.q8:
            msg = [codec_of(self.compress)[2](n) for n in t.numels]   # codes of the real elements + the blocks' scales
        else:
            msg = [n * 4 for n in t.numels]
        self.msg_bytes = msg
        self.d_msg = i32(msg)
        # ---- state -----------------------------------------------------------------------
        H = max(1, cfg.sent_history)
        self.thres, self.last_norm, self.last_iter = zf(t.n_tensors), zf(t.n_tensors), zf(t.n_tensors)
        self.slopes = zf(t.n_tensors * H)
        self.fire = torch.ones(t.n_tensors, dtype=torch.int32, device=dev)
        self.cur_norm = zf(t.n_tensors)
        self.counters = torch.zeros(4, dtype=torch.int64, device=dev)
        self.d_pass = zi(1)
        self.ticket = zi(8)      # [0] step tail, [1] push phase, [4] sparse, [6] all-reduce
        self.status = zi(1)
        self.tile_ss = zf(t.n_tiles * 8)
        self.tensor_done = zi(t.n_tensors)
        self.log_cap = 0
        self.log_ring = None
        self.tile_ss_l = self.tile_ss_r = None
        if self.want_logs and cfg.algo in ("event", "spevent"):
            self.log_cap = 4096
            self.log_ring = zf(self.log_cap * t.n_tensors * 5)
            self.tile_ss_l, self.tile_ss_r = zf(t.n_tiles * 8), zf(t.n_tiles * 8)
            self._drained = 0
            self._last_recv_l = torch.zeros(t.n_tensors)
            self._last_recv_r = torch.zeros(t.n_tensors)
        if self.sparse:
            # Q8: prev / replicas start from theta_0 (identical on all ranks)
            self.prev = arena.theta.clone()
            self.rep_l = arena.theta.clone()
            self.rep_r = arena.theta.clone()
            self.hist = torch.zeros(t.n_tensors * 2048, dtype=torch.int32, device=dev)
            self.sel_prefix, self.sel_remain = zi(t.n_tensors), zi(t.n_tensors)
            self.cand = torch.empty(t.n_padded, dtype=torch.int32, device=dev)      # candidate keys (worst case: all)
            self.cand_cnt, self.done1, self.done2 = zi(t.n_tensors), zi(t.n_tensors), zi(t.n_tensors)
            self.desc = torch.zeros(t.n_tiles, dtype=torch.int64, device=dev)       # look-back descriptors
            self.sp_bar = zi(4)
            self.applied_l, self.applied_r = zi(t.n_tensors), zi(t.n_tensors)
        if self.q8:
            # the public copy of my theta and my replicas of the neighbours' copies, all theta_0 (identical on all
            # ranks, so the receivers hold it without a message)
            self.prev = arena.theta.clone()
            self.rep_l = arena.theta.clone()
            self.rep_r = arena.theta.clone()
        if self.gt:
            # y, the previous gradient (fp32 whatever the gradient dtype) and the y inboxes start at zero on every rank
            self.y, self.g_prev = zf(t.n_padded), zf(t.n_padded)
        self.psi = None
        if self.ed:
            # psi starts at theta_0, which is identical on every rank
            self.psi = self.win.view("psi", torch.float32)
            self.psi.copy_(arena.theta)
        # drift trigger (--trigger drift): the FSM reads ||theta - sent||.  event: `sent` is an arena-sized buffer,
        # zero like the receivers' inboxes, that the step kernel's pushes keep equal to what was last pushed; spevent:
        # `prev` already is what the receivers hold, element by element
        self.metric = getattr(cfg, "trigger", "norm")
        self.drift = self.metric == "drift" and cfg.algo in ("event", "spevent")
        self.sent = None
        if self.drift:
            self.sent = self.prev if (self.sparse or self.q8) else zf(t.n_padded)
        self.ar_ctr = zi(1)
        if self.rounds:
            self.round_ticket = zi(1)
        if self.cheb:
            # x_{q-1} of the rounds (rewritten by round q < Q before round q + 1 reads it) and the fp32
            # (alpha_q, omega_q)
            Q = self.gossip_rounds
            self.cheb_prev = zf(t.n_padded)
            self.d_cheb_coef = torch.tensor(chebyshev_coefficients(ring.offsets, ring.world, Q), dtype=torch.float32,
                                            device=dev).reshape(Q * 2)
        if self.cons:
            self.cons_ring = torch.zeros(self.cons_cap * t.n_tensors * 2, dtype=torch.float64, device=dev)
            self.cons_step, self.cons_ctr = zi(self.cons_cap), zi(1)
            self.d_tile_count = i32(t.tile_count)
        if self.slowmo_period:
            self.slowmo_x, self.slowmo_u = arena.theta.clone(), zf(t.n_padded)
        # gradient pointer table (table mode): device arrays + rotating pinned staging
        self.table_mode = bool(getattr(arena, "table_mode", False)) and cfg.algo != "cent"
        self.d_gptr = torch.zeros(t.n_tensors, dtype=torch.int64, device=dev)
        self.d_gbf16 = zi(t.n_tensors)
        self._stage = []
        self._stage_i = 0
        self._grads_alive = None
        self.host_bytes = 0
        self._connected = False
        self.gp = self.ap = self.ap_avg = self.ap_pga = self.sm = self.sp = self.gs = self.qs = self.ts = self.es = None
        self.rp = self.cs = None
        self.ms = self.d_match_peers = None
        self.d_lr = None
        if hasattr(self.boot, "publish"):
            self.boot.publish("window_ptr", self.win.ptr)
            self.boot.publish("grid", self.grid)
            if self.match is not None:
                self.boot.publish("topology_seed", self.match.seed)
        if not defer_connect:
            self.connect()

    # ------------------------------------------------------------------ wiring
    def connect(self) -> None:
        if self._connected:
            return
        boot, win, ring = self.boot, self.win, self.ring
        if hasattr(boot, "collect"):
            grids = boot.collect("grid")
        else:
            grids = boot.all_gather_object(self.grid)
        self.grid = int(min(grids))          # identical persistent grid on every rank
        if self.match is not None:
            # every rank derives the matchings from the seed: a rank with another seed would wait for a partner that
            # never pushes, and end in a timeout.  Refuse it here instead
            seeds = boot.collect("topology_seed") if hasattr(boot, "collect") else \
                boot.all_gather_object(self.match.seed)
            if len(set(int(x) for x in seeds)) != 1:
                raise ValueError(f"p2p backend: random-match needs the same --topology-seed on every rank, got "
                                 f"{list(seeds)}")
        boot.connect(win)
        L, R = (ring.left, ring.right) if (self.graph is None and self.match is None) else (None, None)
        C, t, cfg = self.C, self.table, self.cfg
        a = self.arena
        P = lambda x: 0 if x is None else x.data_ptr()
        tab = {"tab.tile_tensor": P(self.d_tile_tensor), "tab.t_tile_start": P(self.d_tile_start),
               "tab.t_tile_count": P(self.d_tile_count), "tab.t_numel": P(self.d_numel),
               "tab.t_msg_bytes": P(self.d_msg), "tab.n_tiles": t.n_tiles, "tab.n_tensors": t.n_tensors}
        if True:   # the step kernel is also the plain fused-SGD path of cent / serial runs
            gp = C.GossipParams()
            dense = cfg.algo in ("decent", "event")
            gp.update(tab)
            gp.update({
                "theta": P(a.theta), "grad": P(a.grad), "mom": P(a.mom) if cfg.momentum != 0 else 0,
                "tile_ss": P(self.tile_ss), "tile_ss_l": P(self.tile_ss_l), "tile_ss_r": P(self.tile_ss_r),
                "shadow": P(getattr(a, "shadow", None)) if self.table_mode else 0,
                "t_grad_ptr": P(self.d_gptr) if self.table_mode else 0,
                "t_grad_bf16": P(self.d_gbf16) if self.table_mode else 0,
                "ticket": P(self.ticket), "tensor_done": P(self.tensor_done), "status": P(self.status),
                "timeout_ns": int(self.timeout_ns),
                "lr": float(cfg.lr), "mu": float(cfg.momentum),
                "wd": float(cfg.weight_decay), "nesterov": 1 if cfg.nesterov else 0,
                "need_norm": 1 if (cfg.algo in ("event", "spevent") or self.log_ring is not None) else 0,
                "do_mix": 1 if self.do_comm else 0,
                "do_push": 1 if (self.do_comm and dense) else 0,
                "sync": 1 if self.sync else 0,
                "send_ack": 1 if dense else 0,
                "zero_grad": 1, "group_iters": int(self.group_iters),
                "phase": 0,
                "fsm.thres": P(self.thres), "fsm.last_norm": P(self.last_norm),
                "fsm.last_iter": P(self.last_iter), "fsm.slopes": P(self.slopes),
                "fsm.fire": P(self.fire), "fsm.cur_norm": P(self.cur_norm),
                "fsm.counters": P(self.counters), "fsm.pass_num": P(self.d_pass),
                "fsm.log_ring": P(self.log_ring), "fsm.log_cap": int(self.log_cap),
                "fsm.horizon": float(cfg.horizon), "fsm.constant": float(cfg.constant),
                "fsm.thres_type": int(cfg.thres_type), "fsm.history": max(1, int(cfg.sent_history)),
                "fsm.initial_comm_passes": int(cfg.initial_comm_passes),
                "fsm.enabled": 1 if (cfg.algo in ("event", "spevent") and self.do_comm) else 0,
                "fsm.metric": 1 if self.drift else 0,
                "sent": P(self.sent) if (self.drift and self.do_comm) else 0,
                "local_steps": self.local_steps,
                "global_avg_period": (self.global_avg_period or (0 if self.slowmo_local else self.slowmo_period))
                                     if self.do_comm else 0,
                "quasi_global": 1 if self.qg else 0,
            })
            if self.slowmo_local or self.cheb:
                # local-SGD base / after the Chebyshev rounds: every step the step kernel runs is the serial step -- no
                # push, mix, flag or ack
                gp.update({"do_mix": 0, "do_push": 0, "send_ack": 0, "local_steps": 1})
            if self.match is not None:
                # one inbox, one flag block and one `done` word per rank; every rank's three addresses in a device
                # array (MatchPeer: inbox, flags, done), indexed by this step's partner
                W = ring.world
                self.d_match_peers = torch.tensor(
                    [[win.addr("match_inbox", q), win.addr("match_flag", q), win.addr("match_done", q)] for q in range(W)],
                    dtype=torch.int64, device=self.dev)
                assert self.d_match_peers.numel() * 8 == W * C.MATCH_PEER_BYTES
                ms = C.MatchSlots()
                ms.update({"world": W, "rank": ring.rank, "seed": int(self.match.seed),
                           "peers": P(self.d_match_peers), "inbox": win.addr("match_inbox"),
                           "flag_from": win.addr("match_flag"), "done": win.addr("match_done")})
                self.ms = ms
            elif self.graph is None:
                gp.update({
                    "flag_from_l": win.addr("flag_from_l"), "flag_from_r": win.addr("flag_from_r"),
                    "flag_to_l": win.addr("flag_from_r", L), "flag_to_r": win.addr("flag_from_l", R),
                    "ack_from_l": win.addr("ack_from_l"), "ack_from_r": win.addr("ack_from_r"),
                    "ack_to_l": win.addr("ack_from_r", L), "ack_to_r": win.addr("ack_from_l", R),
                    "pushed_from_l": win.addr("pushed_from_l"), "pushed_from_r": win.addr("pushed_from_r"),
                    "pushed_to_l": win.addr("pushed_from_r", L), "pushed_to_r": win.addr("pushed_from_l", R),
                })
            else:
                # slot s receives from g.slots()[s]; out-slot j writes slot j of its peer (inbox, flags) and the
                # receiver acks slot s into its sender's ack word of the same index.  One-peer graph (period > 0): the
                # same wiring, the kernel picks the active slot from its step counter
                g, n = self.graph, self.graph.n_slots
                outs, ins = g.out_slots(), g.slots()
                gs = C.GraphSlots()
                gs.update({
                    "n_slots": n, "period": int(g.period),
                    "inbox": [win.addr(f"inbox_{s}") for s in range(n)],
                    "push": [win.addr(f"inbox_{k}", p) for p, k in outs],
                    "flag_from": [win.addr(f"flag_from_{s}") for s in range(n)],
                    "flag_to": [win.addr(f"flag_from_{k}", p) for p, k in outs],
                    "ack_from": [win.addr(f"ack_from_{j}") for j in range(n)],
                    "ack_to": [win.addr(f"ack_from_{s}", ins[s]) for s in range(n)],
                })
                self.gs = gs
            if self.q8:
                # I am my left neighbour's right and my right neighbour's left.  R = 2: the one neighbour gets two
                # copies in two inboxes and keeps two replicas (no wire dedup)
                qs = C.Q8Slots()
                qs.update({
                    "q_from_l": win.addr("q_from_l"), "q_from_r": win.addr("q_from_r"),
                    "s_from_l": win.addr("qs_from_l"), "s_from_r": win.addr("qs_from_r"),
                    "q_to_l": win.addr("q_from_r", L), "q_to_r": win.addr("q_from_l", R),
                    "s_to_l": win.addr("qs_from_r", L), "s_to_r": win.addr("qs_from_l", R),
                    "prev": P(self.prev), "rep_l": P(self.rep_l), "rep_r": P(self.rep_r),
                    "codec": 1 if self.compress == "sign" else 0, "gamma": self.choco_gamma,
                })
                self.qs = qs
            elif dense and self.graph is None and self.match is None:
                gp.update({"inbox_l": win.addr("inbox_l"), "inbox_r": win.addr("inbox_r"),
                           "push_l": win.addr("inbox_r", L), "push_r": win.addr("inbox_l", R)})
                # 2-rank ring: left == right.  Push theta ONCE (into the peer's inbox_r) and let the peer read that
                # copy as both L and R: (theta + 2 theta')/3 is unchanged bit for bit, the link carries 69.8 MB per
                # step instead of 139.6 MB.  Event/byte counters keep the reference's logical count (2 messages).
                self.wire_dedup = self.ring.world == 2 and L == R
                if self.wire_dedup:
                    gp.update({"inbox_l": win.addr("inbox_r"), "push_r": 0})
                if self.gt:
                    # y travels exactly as theta does, the single-copy dedup of the 2-rank ring included
                    ts = C.TrackSlots()
                    ts.update({"y": P(self.y), "g_prev": P(self.g_prev),
                               "y_in_l": win.addr("y_in_r" if self.wire_dedup else "y_in_l"),
                               "y_in_r": win.addr("y_in_r"),
                               "y_to_l": win.addr("y_in_r", L),
                               "y_to_r": 0 if self.wire_dedup else win.addr("y_in_l", R)})
                    self.ts = ts
                if self.ed:
                    # phi travels in theta's inboxes, the single-copy dedup of the 2-rank ring included
                    es = C.EdSlots()
                    es.update({"psi": P(self.psi)})
                    self.es = es
            elif self.sparse:
                gp.update({"inbox_l": P(self.rep_l), "inbox_r": P(self.rep_r)})
            self.gp = gp
        if self.sparse:
            sp = C.SparseParams()
            sp.update(tab)
            sp.update({
                "theta": P(a.theta), "prev": P(self.prev), "rep_l": P(self.rep_l), "rep_r": P(self.rep_r),
                "rec_from_l": win.addr("rec_from_l"), "rec_from_r": win.addr("rec_from_r"),
                "rec_to_l": win.addr("rec_from_r", L), "rec_to_r": win.addr("rec_from_l", R),
                "seq_from_l": win.addr("seq_from_l"), "seq_from_r": win.addr("seq_from_r"),
                "seq_to_l": win.addr("seq_from_r", L), "seq_to_r": win.addr("seq_from_l", R),
                "applied_l": P(self.applied_l), "applied_r": P(self.applied_r),
                "done_from_l": win.addr("done_from_l"), "done_from_r": win.addr("done_from_r"),
                "done_to_l": win.addr("done_from_r", L), "done_to_r": win.addr("done_from_l", R),
                "ack_from_l": win.addr("ack_from_l"), "ack_from_r": win.addr("ack_from_r"),
                "ack_to_l": win.addr("ack_from_r", L), "ack_to_r": win.addr("ack_from_l", R),
                "t_k": P(self.d_k), "t_rec_off": P(self.d_rec_off), "hist": P(self.hist),
                "sel_prefix": P(self.sel_prefix), "sel_remain": P(self.sel_remain),
                "cand": P(self.cand), "cand_cnt": P(self.cand_cnt), "done1": P(self.done1), "done2": P(self.done2),
                "desc": P(self.desc), "bar": P(self.sp_bar),
                "fire": P(self.fire), "pass_num": P(self.d_pass), "ticket": P(self.ticket[4:]),
                "status": P(self.status), "timeout_ns": int(self.timeout_ns), "sync": 1 if self.sync else 0,
            })
            # 2-rank ring: the one neighbour is both left and right -> write each record (and its seq / done flags)
            # ONCE, into the peer's from-right inbox, and let the peer read that copy for both replicas
            self.wire_dedup = self.ring.world == 2 and L == R
            if self.wire_dedup:
                sp.update({"rec_to_r": 0, "seq_to_r": 0, "done_to_r": 0,
                           "rec_from_l": win.addr("rec_from_r"), "seq_from_l": win.addr("seq_from_r"),
                           "done_from_l": win.addr("done_from_r")})
            self.sp = sp
            # the mix+SGD kernel runs the receive side (scatter into the replicas) as its prologue
            self.d_sp = torch.zeros((C.SPARSE_PARAMS_BYTES + 7) // 8, dtype=torch.int64, device=self.dev)
            C.sparse_params_to_device(sp, self.d_sp.data_ptr())
            if self.do_comm:
                self.gp.update({"sparse": self.d_sp.data_ptr()})
        if self.rounds:
            # the ring's slots and the graph's share one wiring: slot s receives from ring.slots()[s], out-slot j writes
            # slot j of its peer, and the receiver acks slot s into its sender's round ack word of the same index.
            # 2-rank ring: one copy on the wire, into the peer's slot 1, read for both slots (as the ring step does)
            g, n = self.ring, self.ring.n_slots
            outs, ins = g.out_slots(), g.slots()
            dedup = self.graph is None and self.ring.world == 2
            rp = C.RoundParams()
            rp.update({
                "theta": P(a.theta), "pass_num": P(self.d_pass), "ticket": P(self.round_ticket),
                "status": P(self.status), "timeout_ns": int(self.timeout_ns), "n_tiles": t.n_tiles,
                "group_iters": int(self.group_iters), "rounds": _rounds_per_step(cfg), "n_slots": n,
                "inbox": [win.addr("round_inbox_1" if dedup else f"round_inbox_{s}") for s in range(n)],
                "push": [0 if (dedup and j == 0) else win.addr(f"round_inbox_{k}", p) for j, (p, k) in enumerate(outs)],
                "flag_from": [win.addr(f"round_flag_{s}") for s in range(n)],
                "flag_to": [win.addr(f"round_flag_{k}", p) for p, k in outs],
                "ack_from": [win.addr(f"round_ack_{j}") for j in range(n)],
                "ack_to": [win.addr(f"round_ack_{s}", ins[s]) for s in range(n)],
            })
            self.rp = rp
            if self.cheb:
                cs = C.ChebParams()
                cs.update({"prev": P(self.cheb_prev), "coef": P(self.d_cheb_coef)})
                self.cs = cs
        # ---- all-reduce parameter blocks (cent step; final averaging for every algorithm) ----
        W = self.ring.world
        self.d_peer_grad = torch.tensor([win.addr("grad", r) for r in range(W)], dtype=torch.int64, device=self.dev)
        self.d_peer_theta = torch.tensor([win.addr("theta", r) for r in range(W)], dtype=torch.int64, device=self.dev)
        self.d_peer_flags = torch.tensor([win.addr("ar_flags", r) for r in range(W)], dtype=torch.int64, device=self.dev)
        common = {"peer_flags": P(self.d_peer_flags), "flags": win.addr("ar_flags"),
                  "ticket": P(self.ticket[6:]), "status": P(self.status), "step_ctr": P(self.ar_ctr),
                  "timeout_ns": int(self.timeout_ns), "n_tiles": t.n_tiles, "rank": self.ring.rank,
                  "world": W, "lr": float(cfg.lr), "mu": float(cfg.momentum)}
        ap = C.AllReduceParams()
        ap.update(common)
        ap.update({"peer_bufs": P(self.d_peer_grad), "local": P(a.grad), "theta": P(a.theta),
                   "mom": P(a.mom) if cfg.momentum != 0 else 0, "mode": 1, "zero_after": 1,
                   "wd": float(cfg.weight_decay), "nesterov": 1 if cfg.nesterov else 0,
                   "pass_num": P(self.d_pass),      # cent's device step index: the all-reduce advances it
                   "two_shot": 1 if t.n_padded * 4 > ONE_SHOT_MAX_BYTES else 0})
        self.ap = ap
        av = C.AllReduceParams()
        av.update(common)
        av.update({"peer_bufs": P(self.d_peer_theta), "local": P(a.theta), "mode": 0, "zero_after": 0,
                   "two_shot": 1})
        self.ap_avg = av
        # --global-avg-period: the same average, gated on the gossip pass counter (the step kernel that follows it in
        # the stream advances that counter).  It shares the launch counter, the ticket and ar_flags with the final
        # average: a gated-off launch leaves all three untouched, so they stay equal on every rank
        self.ap_pga = None
        if self.global_avg_period and self.do_comm and W > 1:
            pga = C.AllReduceParams()
            pga.update(common)
            pga.update({"peer_bufs": P(self.d_peer_theta), "local": P(a.theta), "mode": 0, "zero_after": 0,
                        "two_shot": 1, "gate_pass": P(self.d_pass), "gate_period": self.global_avg_period})
            self.ap_pga = pga
        # --slowmo-period: the SlowMo sync kernel, gated on the gossip pass counter like ap_pga, sharing the launch
        # counter, the ticket and ar_flags with the final average.  It runs at R = 1 too (a world of one)
        self.sm = None
        if self.slowmo_period:
            sm = C.SlowMoParams()
            sm.update(common)
            sm.update({"peer_bufs": P(self.d_peer_theta), "local": P(a.theta), "mode": 0, "zero_after": 0,
                       "two_shot": 1, "gate_pass": P(self.d_pass), "gate_period": self.slowmo_period,
                       "shadow": P(getattr(a, "shadow", None)) if self.table_mode else 0,
                       "x": P(self.slowmo_x), "u": P(self.slowmo_u), "beta": self.slowmo_beta,
                       "alpha": self.slowmo_lr})
            self.sm = sm
        # --consensus-every: the consensus kernel, gated on the gossip pass counter after the step kernel that advanced
        # it, sharing the launch counter, the ticket and ar_flags with the final average.  cp_now is the same block with
        # N = 1 (every launch measures): the ungated measurement of measure_consensus()
        if self.cons:
            self.d_peer_part = torch.tensor([win.addr("cons_part", r) for r in range(W)], dtype=torch.int64,
                                            device=self.dev)
            f = {"peer_bufs": P(self.d_peer_theta), "local": P(a.theta), "mode": 0, "zero_after": 0, "two_shot": 1,
                 "gate_pass": P(self.d_pass), "peer_part": P(self.d_peer_part), "part": win.addr("cons_part"),
                 "tile_tensor": P(self.d_tile_tensor), "t_tile_start": P(self.d_tile_start),
                 "t_tile_count": P(self.d_tile_count), "t_numel": P(self.d_numel), "n_tensors": t.n_tensors}
            self.cp, self.cp_now = C.ConsensusParams(), C.ConsensusParams()
            for blk, n in ((self.cp, self.consensus_every), (self.cp_now, 1)):
                blk.update(common)
                blk.update(f)
                blk.update({"gate_period": n})
            self._set_cons_ring()
        # EXPERIMENTAL NVLS: multicast mappings of the same buffers (0 unless the window is a SymmWindow on
        # a fabric with multicast support) -> csrc/allreduce_nvls.cu for the two-shot launches
        mc_grad = win.mc_addr("grad") if hasattr(win, "mc_addr") else 0
        mc_theta = win.mc_addr("theta") if hasattr(win, "mc_addr") else 0
        self.nvls = bool(mc_grad) and W > 1
        if self.nvls:
            ap.update({"mc_local": mc_grad})
            av.update({"mc_local": mc_theta})
            if self.ap_pga is not None:
                self.ap_pga.update({"mc_local": mc_theta})
        self.nvls_step = self.nvls and t.n_padded * 4 > ONE_SHOT_MAX_BYTES
        self._connected = True
        self._apply_lr_table()
        if self.gossip or self.table_mode:
            self._init_norms(run_fsm=self.gossip)
        boot.barrier()

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.dev).cuda_stream

    # ------------------------------------------------------------------ consensus distance
    def _set_cons_ring(self) -> None:
        ring = {"ring": self.cons_ring.data_ptr(), "ring_step": self.cons_step.data_ptr(),
                "ring_ctr": self.cons_ctr.data_ptr(), "cap": self.cons_cap}
        self.cp.update(ring)
        self.cp_now.update(ring)

    def set_consensus_capacity(self, cap: int) -> None:
        """Rows the device ring holds between two drain_consensus() calls (default 1024).  Call before the first step
        (a graph captured earlier keeps the ring it was captured with)."""
        cap = int(cap)
        if cap < 1:
            raise ValueError(f"consensus ring capacity must be >= 1, got {cap}")
        if not self.cons or cap == self.cons_cap:
            return
        if self.pass_num or self._cons_drained:
            raise RuntimeError("set_consensus_capacity must be called before the first step")
        self.cons_cap = cap
        self.cons_ring = torch.zeros(cap * self.table.n_tensors * 2, dtype=torch.float64, device=self.dev)
        self.cons_step = torch.zeros(cap, dtype=torch.int32, device=self.dev)
        if self._connected:
            self._set_cons_ring()

    def launch_consensus_now(self) -> None:
        """Enqueue one ungated measurement of the current theta on the current stream (every rank must)."""
        if self.cons:
            with torch.cuda.device(self.dev):
                self.C.consensus(self.cp_now, self.grid, self._stream())

    def drain_consensus(self):
        """The measurements since the last drain, oldest first: a list of (step, D, A), D and A float64 CPU tensors
        [n_tensors] (parallel/trigger.py:consensus_stats).  One host synchronisation.  Raises when the ring overwrote
        rows that were never drained."""
        out, self._cons_held = self._cons_held, []
        if not self.cons:
            return out
        torch.cuda.synchronize(self.dev)
        ctr = int(self.cons_ctr.item())
        n = ctr - self._cons_drained
        if n > self.cons_cap:
            raise RuntimeError(f"consensus ring overwrote {n - self.cons_cap} undrained measurements: drain at least "
                               f"every {self.cons_cap} measurements (set_consensus_capacity)")
        nt = self.table.n_tensors
        ring = self.cons_ring.view(self.cons_cap, nt, 2).cpu()
        steps = self.cons_step.cpu()
        for j in range(self._cons_drained, ctr):
            row = j % self.cons_cap
            out.append((int(steps[row]), ring[row, :, 0].clone(), ring[row, :, 1].clone()))
        self._cons_drained = ctr
        return out

    def measure_consensus(self):
        """(D, A) of the current theta, measured now whatever the step: the kernel with N = 1 (zeros at R = 1).
        Earlier undrained rows stay for the next drain_consensus()."""
        if not self.cons:
            z = torch.zeros(self.table.n_tensors, dtype=torch.float64)
            return z, z.clone()
        self.launch_consensus_now()
        rows = self.drain_consensus()
        self._cons_held = rows[:-1]
        return rows[-1][1], rows[-1][2]

    # ------------------------------------------------------------------ learning-rate schedule
    def set_lr_table(self, table) -> None:
        """Upload the per-step learning rates once; the step kernels index them with the device pass counter
        (d_pass), so eager steps and every replay of a captured graph read the lr of their own step.  Call before
        the first step (a graph captured earlier keeps the parameters it was captured with)."""
        super().set_lr_table(table)
        self.d_lr = None if self.lr_table is None else self.lr_table.to(self.dev)
        if self._connected:
            self._apply_lr_table()

    def _apply_lr_table(self) -> None:
        upd = {"lr_table": 0 if self.d_lr is None else self.d_lr.data_ptr(),
               "lr_len": 0 if self.d_lr is None else int(self.d_lr.numel())}
        self.gp.update(upd)
        self.ap.update(upd)
        if self.sm is not None:
            self.sm.update(upd)

    def set_sparse_init(self, prev, rep_l, rep_r) -> None:
        super().set_sparse_init(prev, rep_l, rep_r)
        if self.drift and self._connected and self.do_comm:
            # the first decision was taken at connect() from theta_0 - prev: take it again from the new prev, from
            # the FSM's initial state (no step has run yet)
            for x in (self.thres, self.last_norm, self.last_iter, self.slopes, self.cur_norm):
                x.zero_()
            self.fire.fill_(1)
            self._init_norms(run_fsm=True)

    def _init_norms(self, run_fsm: bool) -> None:
        with torch.cuda.device(self.dev):
            self.C.gossip_init(self.gp, self.grid, 1 if run_fsm else 0, self._stream())

    # ------------------------------------------------------------------ gradient table
    def update_grad_table(self, compute, persistent: bool = False):
        """Point the step kernel at this backward's gradient tensors (one pointer + dtype flag per
        arena tensor).  Eager mode: every step, through rotating pinned staging buffers.  Graph
        capture: once -- the captured backward writes its gradients to fixed addresses; pass
        persistent=True and keep the returned staging buffers alive with the graph."""
        if not self.table_mode:
            return None
        n = self.table.n_tensors
        if persistent:
            hp, hf = torch.empty(n, dtype=torch.int64).pin_memory(), torch.empty(n, dtype=torch.int32).pin_memory()
            ev = None
        else:
            if len(self._stage) < 4:
                self._stage.append((torch.empty(n, dtype=torch.int64).pin_memory(),
                                    torch.empty(n, dtype=torch.int32).pin_memory(), torch.cuda.Event()))
                hp, hf, ev = self._stage[-1]
            else:
                hp, hf, ev = self._stage[self._stage_i % 4]
                ev.synchronize()                  # the copy that last used this slot has executed
            self._stage_i += 1
        alive = []
        for i, c in enumerate(compute):
            g = c.grad
            if g is None:
                raise RuntimeError(f"tensor {self.table.names[i]} received no gradient")
            if g.stride() != c.stride() or g.dtype not in (torch.float32, torch.bfloat16):
                g = torch.empty_like(c, dtype=g.dtype if g.dtype in (torch.float32, torch.bfloat16)
                                     else torch.float32).copy_(g)
            hp[i] = g.data_ptr()
            hf[i] = 1 if g.dtype == torch.bfloat16 else 0
            alive.append(g)
        self.d_gptr.copy_(hp, non_blocking=True)
        self.d_gbf16.copy_(hf, non_blocking=True)
        if ev is not None:
            ev.record()
        self._grads_alive = alive                 # keep them until the next table replaces them
        return hp, hf, alive

    # ------------------------------------------------------------------ step
    graph_safe = True      # launch() only enqueues kernels whose per-step state lives on the device

    def launch_pre(self) -> None:
        """Split step, first half (side stream, concurrent with forward/backward): push theta_k to
        the neighbours / select + push the top-k records.  Depends only on theta_k and fire[]."""
        if not self.overlap:
            return
        C, s = self.C, self._stream()
        with torch.cuda.device(self.dev):
            if self.sparse:
                C.sparse_select_push(self.sp, self.grid, s)
            elif self.ce_push:
                C.ce_push(self.gp, s)                       # experimental: DMA engines instead of an SM kernel
            else:
                g = self.push_grid or max(1, min(self.grid, 128))
                C.gossip_step_phase(self.gp, 1, g, s)

    def launch(self) -> None:
        """Enqueue this step's kernels on the current stream (CUDA-graph capturable: the step
        counter, trigger state and handshake sequence numbers are all device resident)."""
        C, s = self.C, self._stream()
        with torch.cuda.device(self.dev):
            if self.cfg.algo == "cent":
                if self.ring.world > 1:
                    (C.allreduce_nvls if self.nvls_step else C.allreduce)(self.ap, self.grid, s)
                else:
                    C.gossip_step(self.gp, self.grid, s)       # plain fused SGD
                return
            if self.ap_pga is not None:
                # the average comes first: the step kernel of an averaging step runs SGD on the averaged theta
                (C.allreduce_nvls if self.nvls else C.allreduce)(self.ap_pga, self.grid, s)
            if self.sm is not None:
                # the sync comes first: the step kernel of a sync step runs SGD on theta <- x
                C.slowmo_sync(self.sm, self.grid, s)
            if self.cs is not None:
                # theta <- P_Q(W) theta, then the step kernel as the serial step (gp: no push, mix or ack)
                C.gossip_rounds_cheb(self.rp, self.cs, self.grid, s)
            elif self.rp is not None:
                # theta <- W^(Q-1) theta, then the step kernel's own push, mix and optimizer step
                C.gossip_rounds(self.rp, self.grid, s)
            if self.sparse and self.do_comm:
                if not self.overlap:
                    C.sparse_select_push(self.sp, self.grid, s)        # 3 launches: hist, candidates, compaction
                C.gossip_step(self.gp, self.grid, s)                   # receive prologue + mix + SGD + trigger
            elif self.q8 and self.do_comm:
                C.gossip_step_q8(self.gp, self.qs, self.grid, s)
            elif self.gt:
                C.gossip_step_gt(self.gp, self.ts, self.grid, s)
            elif self.ed:
                C.gossip_step_ed(self.gp, self.es, self.grid, s)
            elif self.match is not None and self.do_comm:
                C.gossip_step_match(self.gp, self.ms, self.grid, s)
            elif self.overlap:
                C.gossip_step_phase(self.gp, 2, self.grid, s)
            elif self.dbuf:
                C.gossip_step_dbuf(self.gp, self.grid, s)
            elif self.graph is not None and self.do_comm and not self.slowmo_local and not self.cheb:
                C.gossip_step_graph(self.gp, self.gs, self.grid, s)
            else:
                C.gossip_step(self.gp, self.grid, s)
            if self.cp is not None:
                # after the step kernel that completed the step: it measures theta_{k} when N divides k
                C.consensus(self.cp, self.grid, s)

    def account_step(self) -> None:
        """Host-side bookkeeping of one executed step (after launch() or a graph replay)."""
        self.pass_num += 1
        if self.consensus_every and not self.cons and self.pass_num % self.consensus_every == 0:
            z = torch.zeros(self.table.n_tensors, dtype=torch.float64)     # R = 1: no launch, the distance is 0
            self._cons_held.append((self.pass_num, z, z.clone()))
        if self.cfg.algo == "cent" and self.ring.world > 1:
            self.host_bytes += self.table.n_elems * 4
        elif self.cfg.algo == "decent" and self.do_comm and self.q8:
            self.host_bytes += 2 * sum(self.msg_bytes)
        elif self.gt:
            self.host_bytes += 2 * 2 * self.table.n_elems * 4      # theta and y, to both neighbours
        elif self.slowmo_period and self.pass_num % self.slowmo_period == 0:
            # --slowmo-period tau: a sync step counts one all-reduce of theta (cent's convention)
            self.host_bytes += self.table.n_elems * 4 if self.ring.world > 1 else 0
        elif self.slowmo_local:
            pass                                                  # local-SGD base: no exchange
        elif self.global_avg_period and self.do_comm and self.pass_num % self.global_avg_period == 0:
            # --global-avg-period P: an averaging step counts one all-reduce of theta (cent's convention)
            self.host_bytes += self.table.n_elems * 4 if self.ring.world > 1 else 0
        elif self.match is not None and self.do_comm:
            # random-match: one copy to this step's partner, nothing on an idle step
            if self.match.partner(self.pass_num) is not None:
                self.host_bytes += self.table.n_elems * 4
        elif self.cfg.algo == "decent" and self.do_comm and self.pass_num % self.local_steps == 0:
            # --local-steps H: only every H-th step sends; --gossip-rounds Q: every step sends Q times
            q = self.gossip_rounds if self.rounds else 1
            self.host_bytes += q * getattr(self.ring, "fanout", 2) * self.table.n_elems * 4

    def step(self) -> None:
        if self.overlap:        # no compute to hide behind when called stand-alone: run both halves in order
            self.launch_pre()
        self.launch()
        self.account_step()

    # ------------------------------------------------------------------ end of training
    def check_status(self) -> None:
        st = int(self.status.item())
        if st != 0:
            raise RuntimeError(f"p2p backend: device status {st} (1 = peer wait timed out) on rank {self.ring.rank}")

    def final_average_nocheck(self) -> None:
        if self.ring.world == 1:
            return
        with torch.cuda.device(self.dev):
            (self.C.allreduce_nvls if self.nvls else self.C.allreduce)(self.ap_avg, self.grid, self._stream())
        if not self.cfg.final_divide_all and self.ring.rank != 0:
            self.arena.theta.mul_(float(self.ring.world))     # reference quirk Q5: only rank 0 divides
        if self.table_mode and getattr(self.arena, "shadow", None) is not None:
            self._init_norms(run_fsm=False)                   # refresh the bf16 shadow of the averaged model

    def final_average(self) -> None:
        self.final_average_nocheck()
        self.check_status()

    def num_events(self) -> int:
        return int(self.counters[0].item())

    def total_events(self) -> int:
        ev = self.num_events()
        if self.ring.world == 1 or not hasattr(self.boot, "all_gather_object"):
            return ev
        return int(sum(self.boot.all_gather_object(ev)))

    def bytes_sent(self) -> int:
        return int(self.counters[1].item()) + self.host_bytes

    def synchronize(self) -> None:
        torch.cuda.synchronize(self.dev)

    # ------------------------------------------------------------------ logs
    def drain_logs(self) -> List[StepLog]:
        if self.log_ring is None:
            return []
        torch.cuda.synchronize(self.dev)
        t = self.table
        ring = self.log_ring.view(self.log_cap, t.n_tensors, 5).cpu()
        out = []
        numel = torch.tensor(t.numels, dtype=torch.float32)
        for s in range(self._drained + 1, self.pass_num + 1):
            row = ring[(s - 1) % self.log_cap]
            ln, rn = row[:, 3].clone(), row[:, 4].clone()
            if self.recv_rms:
                ln, rn = ln / numel.sqrt(), rn / numel.sqrt()
            lnew = (ln - self._last_recv_l).abs() > 0
            rnew = (rn - self._last_recv_r).abs() > 0
            self._last_recv_l = torch.where(lnew, ln, self._last_recv_l)
            self._last_recv_r = torch.where(rnew, rn, self._last_recv_r)
            out.append(StepLog(s, row[:, 0].clone(), row[:, 1].clone(), row[:, 2] > 0.5, ln, rn, lnew, rnew))
        self._drained = self.pass_num
        return out

    # ------------------------------------------------------------------ checkpoint
    def state_dict(self):
        torch.cuda.synchronize(self.dev)
        sd = {"pass_num": self.pass_num, "host_bytes": self.host_bytes}
        if self.qg:
            sd["quasi_global_momentum"] = True     # the arena's momentum holds m_hat
        for k in ("thres", "last_norm", "last_iter", "slopes", "fire", "cur_norm", "counters", "d_pass"):
            sd[k] = getattr(self, k).cpu().clone()
        if self.cfg.algo in ("decent", "event") and self.graph is not None:
            sd["topology_offsets"] = list(self.graph.offsets)
            if self.graph.period:
                sd["topology"] = self.graph.kind
            for k in range(self.graph.n_slots):
                sd[f"inbox_{k}"] = self.win.view(f"inbox_{k}", torch.float32).cpu().clone()
        elif self.match is not None:
            # the matching is a function of (seed, R, step): the name and the seed, and no inbox (every step's partner
            # rewrites it before it is read)
            sd["topology"], sd["topology_seed"], sd["topology_offsets"] = self.match.kind, int(self.match.seed), []
        elif self.cfg.algo in ("decent", "event") and not self.q8:
            sd["inbox_l"] = self.win.view("inbox_l", torch.float32).cpu().clone()
            sd["inbox_r"] = self.win.view("inbox_r", torch.float32).cpu().clone()
        if self.cfg.algo in ("decent", "event"):
            sd["compress"] = self.compress
            if self.choco_gamma:
                sd["choco_gamma"] = self.choco_gamma
        if self.cfg.algo == "decent":
            sd["gradient_tracking"] = self.gt
            sd["local_steps"] = self.local_steps
            sd["exact_diffusion"] = self.ed
            if self.global_avg_period:
                sd["global_avg_period"] = self.global_avg_period
            sd.update(slowmo_state(self))
            if self.ed:
                sd["psi"] = self.psi.cpu().clone()
            if self.gt:
                sd["y"], sd["g_prev"] = self.y.cpu().clone(), self.g_prev.cpu().clone()
                sd["y_in_l"] = self.win.view("y_in_l", torch.float32).cpu().clone()
                sd["y_in_r"] = self.win.view("y_in_r", torch.float32).cpu().clone()
        if self.sparse or self.q8:
            for k in ("prev", "rep_l", "rep_r"):
                sd[k] = getattr(self, k).cpu().clone()
        if self.cfg.algo in ("event", "spevent"):
            sd["trigger"] = self.metric
            if self.drift and not self.sparse and not self.q8:
                sd["sent"] = self.sent.cpu().clone()
        return sd

    def load_state_dict(self, sd):
        check_topology_state(sd, self.ring, self.cfg.algo)
        check_trigger_state(sd, self.metric, self.cfg.algo)
        check_compress_state(sd, self.compress, self.cfg.algo)
        check_choco_state(sd, self.choco_gamma, self.cfg.algo)
        check_tracking_state(sd, self.gt, self.cfg.algo)
        check_local_steps_state(sd, self.local_steps, self.cfg.algo)
        check_exact_diffusion_state(sd, self.ed, self.cfg.algo)
        check_global_avg_state(sd, self.global_avg_period, self.cfg.algo)
        check_qg_state(sd, self.qg, self.cfg.algo)
        check_slowmo_state(sd, self.slowmo_period, self.slowmo_beta, self.slowmo_lr, self.cfg.algo)
        self.pass_num = int(sd["pass_num"])
        self.host_bytes = int(sd.get("host_bytes", 0))
        for k in ("thres", "last_norm", "last_iter", "slopes", "fire", "cur_norm", "counters", "d_pass"):
            getattr(self, k).copy_(sd[k].to(self.dev))
        if self.graph is not None:
            for k in range(self.graph.n_slots):
                self.win.view(f"inbox_{k}", torch.float32).copy_(sd[f"inbox_{k}"].to(self.dev))
        elif "inbox_l" in sd and self.cfg.algo in ("decent", "event"):
            self.win.view("inbox_l", torch.float32).copy_(sd["inbox_l"].to(self.dev))
            self.win.view("inbox_r", torch.float32).copy_(sd["inbox_r"].to(self.dev))
        if self.sparse or self.q8:
            for k in ("prev", "rep_l", "rep_r"):
                getattr(self, k).copy_(sd[k].to(self.dev))
        if self.drift and not self.sparse and not self.q8:
            self.sent.copy_(sd["sent"].to(self.dev))
        if self.gt:
            self.y.copy_(sd["y"].to(self.dev))
            self.g_prev.copy_(sd["g_prev"].to(self.dev))
            self.win.view("y_in_l", torch.float32).copy_(sd["y_in_l"].to(self.dev))
            self.win.view("y_in_r", torch.float32).copy_(sd["y_in_r"].to(self.dev))
        if self.ed:
            self.psi.copy_(sd["psi"].to(self.dev))
        if self.slowmo_period:
            self.slowmo_x.copy_(sd["slowmo_x"].to(self.dev))
            self.slowmo_u.copy_(sd["slowmo_u"].to(self.dev))
        if self.log_ring is not None:
            self._drained = self.pass_num          # log rows of the steps before the checkpoint are not replayed
        if self.cons:
            self._cons_drained = int(self.cons_ctr.item())     # nor are consensus rows
        self._cons_held = []
        # NOTE: handshake counters (flags / acks) restart from pass_num on every rank.  Under --local-steps H the next
        # gossip step k is the first multiple of H above pass_num, so the WAR bound k - H (one-peer: k - tau * H) is at
        # most pass_num, and only that round's pushes reach the flag value k.  Under --global-avg-period P the next gossip
        # step k waits for the ack of k - 1 or k - 2, both <= pass_num; so does a gossip step under --slowmo-period with
        # --local-steps 1, whose step kernel sees tau as its averaging period.  The all-reduce launch counter (ar_ctr) and the
        # ar_flags block are not part of the checkpoint: a new process starts both at zero on every rank, and a backend
        # that keeps running keeps them equal on every rank, since every rank ran the same averages
        if self.gossip:
            self._init_norms(run_fsm=False)
            self._reset_handshake(self.pass_num)
        torch.cuda.synchronize(self.dev)

    def _reset_handshake(self, step: int) -> None:
        if self.match is not None:
            # flags and `done` restart at the resumed step s: step s + 1 waits for fresh flags and for partners that have
            # finished step s, which every rank has
            self.win.view("match_flag", torch.int32).fill_(step)
            self.win.view("match_done", torch.int32).fill_(step)
            return
        if self.graph is not None:
            for k in range(self.graph.n_slots):
                self.win.view(f"flag_from_{k}", torch.int32).fill_(step)
                self.win.view(f"ack_from_{k}", torch.int32).fill_(step)
            self._reset_rounds(step)
            return
        self._reset_rounds(step)
        for name in ("flag_from_l", "flag_from_r", "ack_from_l", "ack_from_r", "pushed_from_l", "pushed_from_r"):
            self.win.view(name, torch.int32).fill_(step)
        if self.q8:
            # the q8 kernel's (tile, warp) flags carry 2 * step + fired (PROTOCOL.md 1.7)
            for name in ("flag_from_l", "flag_from_r"):
                self.win.view(name, torch.int32).fill_(2 * step)
        if self.sparse:
            for name in ("done_from_l", "done_from_r"):
                self.win.view(name, torch.int32).fill_(step)

    def _reset_rounds(self, step: int) -> None:
        """--gossip-rounds: the round flags and acks restart at n * step (n = _rounds_per_step: Q - 1, or Q under
        Chebyshev), the counter of the last round of step `step`, so the next step's first round waits for fresh flags
        and for no ack.  The round inboxes and the Chebyshev `prev` are not restored: every round rewrites them before
        they are read."""
        if self.rounds:
            n = _rounds_per_step(self.cfg)
            for k in range(self.ring.n_slots):
                self.win.view(f"round_flag_{k}", torch.int32).fill_(n * step)
                self.win.view(f"round_ack_{k}", torch.int32).fill_(n * step)

    def close(self) -> None:
        try:
            torch.cuda.synchronize(self.dev)
        except Exception:
            pass
        self.win.close()
