"""Single-process, R-virtual-rank simulator of the four algorithms -- the golden model.

Written from the behavioural specification (SURVEY.md Appendix A), independent of the
distributed backends: all R ranks' arenas live in one process and "communication" is a
tensor copy, executed with iteration-synchronous semantics.  The CPU/gloo backend, the NCCL
baseline and the fused CUDA kernels are all tested against this.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch

from ..parallel.arena import TensorTable
from ..parallel.topology import ACCELS, Graph, chebyshev_coefficients, is_match, match_pairs
from ..parallel.trigger import (COMPRESS, TriggerConfig, TriggerState, cheb_combine_, choco_mix_, codec_of,
                                consensus_stats, drift_norms, mix2_, mix3_, mixk_, qg_sgd_, rank_mean, sgd_, slowmo_sync_,
                                topk_select, trigger_step)
from .lr_schedule import lr_at


class RingSimulator:
    def __init__(self, world: int, theta0: torch.Tensor, table: TensorTable, algo: str,
                 tcfg: Optional[TriggerConfig] = None, lr: float = 1e-2, momentum: float = 0.0,
                 topk_percent: float = 10.0, serial_skip: bool = True, sparse_init=None,
                 weight_decay: float = 0.0, nesterov: bool = False, lr_table: Optional[torch.Tensor] = None,
                 offsets=(1,), compress: str = "none", gradient_tracking: bool = False, local_steps: int = 1,
                 exact_diffusion: bool = False, global_avg_period: int = 0, quasi_global: bool = False,
                 slowmo_period: int = 0, slowmo_beta: float = 0.5, slowmo_lr: float = 1.0,
                 consensus_every: int = 0, choco_gamma: float = 0.0, gossip_rounds: int = 1,
                 topology_seed: int = 0, gossip_accel: str = "none"):
        """`lr_table` (engine/lr_schedule.py): per-step learning rates, step s uses lr_table[min(s-1, len-1)];
        None = the constant `lr`.  `offsets`: circulant gossip graph (parallel/topology.py; a name such as "exp" is
        resolved for `world`), or "onepeer-exp" for the time-varying one-peer exponential graph; the default (1,) is
        the ring.  `tcfg.metric == "drift"`: the trigger reads ||theta - sent|| per tensor, where sent[r] is what rank r's
        receivers hold (event: zero at start, theta_k of every fired tensor at its push; spevent: prev).
        `compress="int8"` (decent/event on the ring): a fired tensor sends the int8 code of theta - prev (q8_encode)
        instead of theta; sender and receivers add the same dequantized delta to prev and to their replica of it, the
        mix reads the replicas, and under drift `sent` is prev.  `compress="sign"`: the same with the 1-bit scaled-sign
        codec (sign_encode / sign_decode).
        `choco_gamma=gamma` in (0, 1] (compress int8 or sign; CHOCO-SGD): the mix becomes choco_mix_, theta <- theta +
        gamma * (((prev + rep_l) + rep_r) / 3 - prev) with prev and the replicas after this step's deltas; pushes, prev,
        replicas, events and bytes are unchanged.  0: the mix above.
        `gradient_tracking=True` (decent on the ring, DSGT): every rank also keeps y (tracking the average gradient),
        the previous gradient g_prev and y inboxes, all zero at start; at step k it pushes theta_k and y_{k-1}, then
        y_k = mix3_(y, yL, yR) + (g_k - g_prev), g_prev <- g_k, and the SGD step reads y_k instead of g_k.  At R = 1 the
        plain serial step runs.  Any dtype works (float64 for convergence studies).
        `local_steps=H` (decent, periodic gossip): step k (1-based) communicates iff H divides k, as round n = k / H --
        exactly the decent step above, with the one-peer graph's active slot (n - 1) mod tau taken from the round.  Every
        other step is the serial step theta <- sgd(theta, g_k): no push, no mix, the inboxes keep what the last round
        delivered, momentum stays local and the lr table stays indexed by step.  Bytes count at communicating steps only.
        `exact_diffusion=True` (decent on the ring; Yuan et al. 2019, D^2 on W_bar = (I + W) / 2): every rank also keeps
        psi, theta_0 at start.  Step k runs the unchanged optimizer on theta_k first, p = sgd(theta_k, g_k), then
        phi = p + (theta_k - psi), psi <- p, pushes phi (decent's bytes) and mixes
        theta_{k+1} = (phi + mix3_(phi, L, R)) / 2 on the received phi's.  sum_r theta_r = sum_r psi_r after every step.
        At R = 1 the plain serial step runs.  Any dtype works (float64 for convergence studies).
        `global_avg_period=P` (decent on the ring or a static circulant graph, P >= 2; Gossip-PGA): at step k with P
        dividing k every rank takes theta' = ((theta_0 + theta_1) + ... + theta_{R-1}) / R (rank_mean) in place of the
        mix and then its own SGD step with its own gradient and momentum; no push, the inboxes keep what the last gossip
        step delivered.  Such a step counts n_elems * 4 bytes per rank (cent's convention for one all-reduce).  Every
        other step is the decent step above.  0: off.
        `quasi_global=True` (decent, event, spevent; momentum > 0; QG-DSGDm): the momentum buffers hold m_hat.  Every
        step of a rank -- gossip, local or serial -- snapshots theta_k first and runs qg_sgd_(theta', theta_k, ...) where
        the other steps run sgd_, so m_hat follows the parameter displacement theta_k - theta_{k+1} instead of the
        gradient.  Bytes and events are unchanged.
        `slowmo_period=tau` (decent on the ring or a static circulant graph, tau >= 2; SlowMo, Wang et al. 2020): every
        rank also keeps the outer iterate x (theta_0 at start) and the slow momentum u (zero at start), identical on every
        rank.  At step k with tau dividing k every rank forms avg = rank_mean(theta), runs slowmo_sync_(x, u, avg, lr_k,
        `slowmo_beta`, `slowmo_lr`), sets theta <- x and takes its own SGD step; such a step counts n_elems * 4 bytes per
        rank (0 at R = 1, where the outer update still runs on the rank's own theta).  The other steps are the base:
        decent's gossip step with local_steps = 1, the serial SGD step with local_steps = tau (local SGD).  0: off.
        `consensus_every=N` (decent, event, spevent): after step k with N dividing k, append (k, D, A) of
        consensus_stats(theta, table) to `self.consensus` -- D_i = sum_r ||theta_r,i - theta_bar_i||^2 and
        A_i = ||theta_bar_i||^2 in float64, theta_bar = rank_mean(theta).  Read-only: training is unchanged.  At R = 1
        every measurement is zero.  0: off.
        `gossip_rounds=Q` (decent on the ring or a static circulant graph, Q >= 2; multi-consensus D-PSGD): a gossip step
        first runs Q - 1 mix-only rounds -- every rank pushes its current theta into every slot it feeds, then mixes
        its inboxes into theta with the step's own mix (mix3_ on the ring, mixk_ on a static graph) -- and then the
        unchanged step on the result, so theta_{k+1} = sgd(W^Q theta_k, g_k).  Bytes are Q times the step's.  At R = 1
        nothing extra runs.  1: off.
        `gossip_accel="chebyshev"` (decent on the ring or a static circulant graph, any Q >= 1): the Q rounds are
        Chebyshev-accelerated -- round q pushes and mixes x_{q-1} into w exactly as a mix-only round, then
        x_q = cheb_combine_(w, x_{q-1}, x_{q-2}, alpha_q, omega_q) with the fp32 coefficients of
        parallel/topology.py chebyshev_coefficients (no omega term at q = 1) -- and every rank takes its SGD step on x_Q
        with no further push or mix: theta_{k+1} = sgd(P_Q(W) theta_k, g_k).  Bytes are those of gossip_rounds=Q.  At
        R = 1 nothing extra runs.  "none": off.
        `offsets="random-match"` with `topology_seed=S` (decent; randomized pairwise gossip): at step k the ranks are
        paired by match_pairs(S, R, k) (parallel/topology.py); every matched rank pushes its whole theta_k into its
        partner's single inbox and mixes theta <- (theta + inbox) / 2 (mix2_), then takes its SGD step; the idle rank of
        an odd R takes its SGD step only.  A matched rank counts n_elems * 4 bytes per step, an idle rank none.  No
        compression, tracking, exact diffusion, local steps, global averaging, quasi-global momentum, slowmo or extra
        gossip rounds.  At R = 1 the name is the ring."""
        assert algo in ("cent", "decent", "event", "spevent")
        if compress not in COMPRESS:
            raise ValueError(f"compress must be one of {COMPRESS}, got {compress!r}")
        self.q8 = compress in ("int8", "sign")
        self.compress = compress
        g = choco_gamma
        if isinstance(g, bool) or not isinstance(g, (int, float)) or not 0.0 <= g <= 1.0:
            raise ValueError(f"choco_gamma must be a number in [0, 1], got {g!r}")
        if g and not self.q8:
            raise ValueError("choco_gamma: compress int8 or sign only")
        self.choco_gamma = float(g)
        self.graphs = [Graph.build(r, world, offsets, seed=topology_seed) for r in range(world)]
        self.match = is_match(self.graphs[0])         # random pairwise matchings: one inbox, partner from the seed
        self.topology_seed = int(topology_seed)
        self.offsets = self.graphs[0].offsets
        self.n_slots = self.graphs[0].n_slots
        self.period = self.graphs[0].period          # 0: static graph; tau: one-peer graph, one active slot per step
        self.fanout = self.graphs[0].fanout          # messages per fired tensor
        if not self.graphs[0].is_ring and algo not in ("decent", "event"):
            raise ValueError(f"topology {offsets!r}: only decent and event gossip beyond the ring")
        if self.q8 and (algo not in ("decent", "event") or not self.graphs[0].is_ring):
            raise ValueError(f"compress {compress}: decent or event on the ring only")
        if gradient_tracking and (algo != "decent" or not self.graphs[0].is_ring or self.q8):
            raise ValueError("gradient tracking: decent on the ring, without compression, only")
        self.gt = bool(gradient_tracking) and world > 1
        if int(local_steps) != local_steps or local_steps < 1:
            raise ValueError(f"local_steps must be an integer >= 1, got {local_steps!r}")
        if local_steps > 1 and (algo != "decent" or self.q8 or gradient_tracking):
            raise ValueError("local steps: decent without compression or gradient tracking only")
        self.local_steps = int(local_steps)
        if exact_diffusion and (algo != "decent" or not self.graphs[0].is_ring or self.q8 or gradient_tracking
                                or local_steps > 1):
            raise ValueError("exact diffusion: decent on the ring, without compression, gradient tracking or local "
                             "steps, only")
        self.ed = bool(exact_diffusion) and world > 1
        if isinstance(global_avg_period, bool) or int(global_avg_period) != global_avg_period or global_avg_period < 0:
            raise ValueError(f"global_avg_period must be an integer >= 0, got {global_avg_period!r}")
        if global_avg_period == 1:
            raise ValueError("global_avg_period 1 averages at every step: that is algo cent")
        if global_avg_period and (algo != "decent" or self.period or self.q8 or gradient_tracking or local_steps > 1
                                  or exact_diffusion):
            raise ValueError("global averaging: decent on the ring or a static graph, without compression, gradient "
                             "tracking, local steps or exact diffusion, only")
        self.global_avg_period = int(global_avg_period)
        if quasi_global and (algo == "cent" or momentum == 0.0 or self.q8 or gradient_tracking or exact_diffusion
                             or global_avg_period):
            raise ValueError("quasi-global momentum: decent, event or spevent with momentum > 0, without compression, "
                             "gradient tracking, exact diffusion or global averaging, only")
        self.qg = bool(quasi_global)
        tau = slowmo_period
        if isinstance(tau, bool) or int(tau) != tau or tau < 0 or tau == 1:
            raise ValueError(f"slowmo_period must be 0 or an integer >= 2, got {tau!r}")
        if tau:
            if not (0.0 <= slowmo_beta < 1.0) or not slowmo_lr > 0.0 or not lr > 0.0:
                raise ValueError("slowmo: slowmo_beta in [0, 1), slowmo_lr > 0 and lr > 0 only")
            if (algo != "decent" or self.period or self.q8 or gradient_tracking or exact_diffusion or global_avg_period
                    or quasi_global or local_steps not in (1, tau)):
                raise ValueError("slowmo: decent on the ring or a static graph with local_steps 1 or slowmo_period, "
                                 "without compression, gradient tracking, exact diffusion, global averaging or "
                                 "quasi-global momentum, only")
        self.slowmo_period, self.slowmo_beta, self.slowmo_lr = int(tau), float(slowmo_beta), float(slowmo_lr)
        if self.slowmo_period:
            self.slowmo_x = [theta0.clone() for _ in range(world)]
            self.slowmo_u = [torch.zeros_like(theta0) for _ in range(world)]
        if isinstance(consensus_every, bool) or int(consensus_every) != consensus_every or consensus_every < 0:
            raise ValueError(f"consensus_every must be an integer >= 0, got {consensus_every!r}")
        if consensus_every and algo == "cent":
            raise ValueError("consensus distance: cent keeps theta identical on every rank")
        self.consensus_every = int(consensus_every)
        Q = gossip_rounds
        if isinstance(Q, bool) or int(Q) != Q or Q < 1:
            raise ValueError(f"gossip_rounds must be an integer >= 1, got {Q!r}")
        if Q > 1 and (algo != "decent" or self.period or self.q8 or gradient_tracking or exact_diffusion
                      or local_steps > 1 or global_avg_period or quasi_global or tau):
            raise ValueError("gossip rounds: decent on the ring or a static graph, without compression, gradient "
                             "tracking, exact diffusion, local steps, global averaging, quasi-global momentum or "
                             "slowmo, only")
        self.gossip_rounds = int(Q)
        if gossip_accel not in ACCELS:
            raise ValueError(f"gossip_accel must be one of {ACCELS}, got {gossip_accel!r}")
        self.cheb_coef = None
        if gossip_accel == "chebyshev":
            if (algo != "decent" or self.period or self.match or self.q8 or gradient_tracking or exact_diffusion
                    or local_steps > 1 or global_avg_period or quasi_global or tau):
                raise ValueError("chebyshev gossip: decent on the ring or a static graph, without compression, gradient "
                                 "tracking, exact diffusion, local steps, global averaging, quasi-global momentum or "
                                 "slowmo, only")
            if world > 1:
                self.cheb_coef = chebyshev_coefficients(self.graphs[0].offsets, world, self.gossip_rounds)
        if self.match and (algo != "decent" or self.q8 or gradient_tracking or exact_diffusion or local_steps > 1
                           or global_avg_period or quasi_global or tau or Q > 1):
            raise ValueError("random-match: decent without compression, gradient tracking, exact diffusion, local "
                             "steps, global averaging, quasi-global momentum, slowmo or gossip rounds, only")
        self.consensus: List[Tuple[int, torch.Tensor, torch.Tensor]] = []
        self.R, self.table, self.algo = world, table, algo
        self.tcfg = tcfg or TriggerConfig()
        self.lr, self.mu = lr, momentum
        self.wd, self.nesterov, self.lr_table = weight_decay, nesterov, lr_table
        self.serial_skip = serial_skip
        self.theta = [theta0.clone() for _ in range(world)]
        self.mom = [torch.zeros_like(theta0) for _ in range(world)]
        self.state = [TriggerState(table.n_tensors, self.tcfg.sent_history) for _ in range(world)]
        self.events = [0] * world
        self.bytes = [0] * world
        self.pass_num = 0
        self.fire_history: List[List[torch.Tensor]] = []
        if algo == "spevent":
            self.k = table.topk_counts(topk_percent)
            # default: everything starts from theta_0; sparse_init=(prev, left, right) mirrors the reference's
            # three extra randomly initialised networks (quirk Q8, identical on every rank: same seed)
            p0, l0, r0 = sparse_init if sparse_init is not None else (theta0, theta0, theta0)
            self.prev = [p0.clone() for _ in range(world)]
            self.rep_l = [l0.clone() for _ in range(world)]
            self.rep_r = [r0.clone() for _ in range(world)]
        elif self.q8:
            # prev[r]: what r's neighbours hold of theta_r; rep_l / rep_r: r's replicas of its neighbours' prev.  theta_0
            # is identical on every rank, so the receivers hold it without a message
            self.prev = [theta0.clone() for _ in range(world)]
            self.rep_l = [theta0.clone() for _ in range(world)]
            self.rep_r = [theta0.clone() for _ in range(world)]
        elif algo in ("decent", "event"):
            # inbox[r][s]: what rank r last received in slot s (zero-initialised RMA window, event.cpp:144-147)
            self.inbox = [[torch.zeros_like(theta0) for _ in range(self.n_slots)] for _ in range(world)]
            if self.n_slots == 2 and not self.period:
                self.inbox_l = [ib[0] for ib in self.inbox]       # ring: slot 0 = from left, slot 1 = from right
                self.inbox_r = [ib[1] for ib in self.inbox]
        if self.gt:
            self.y = [torch.zeros_like(theta0) for _ in range(world)]
            self.g_prev = [torch.zeros_like(theta0) for _ in range(world)]
            self.y_in_l = [torch.zeros_like(theta0) for _ in range(world)]
            self.y_in_r = [torch.zeros_like(theta0) for _ in range(world)]
        if self.ed:
            self.psi = [theta0.clone() for _ in range(world)]
        self.drift = self.tcfg.metric == "drift" and algo in ("event", "spevent")
        if self.drift:
            # what each rank's receivers hold: event -- zero like the inboxes; spevent -- prev itself (same tensors)
            self.sent = self.prev if (algo == "spevent" or self.q8) else [torch.zeros_like(theta0) for _ in range(world)]

    # ------------------------------------------------------------------
    def _flat(self, buf, i):
        t = self.table
        return buf[t.offsets[i]: t.offsets[i] + t.numels[i]]

    def _padded(self, buf, i):
        """Tensor i's whole tiles (its elements and the zero padding after them): the blocks of the int8 codec."""
        t = self.table
        return buf[t.offsets[i]: t.offsets[i] + t.tile_count[i] * t.tile]

    def _norms(self, buf):
        return torch.stack([torch.linalg.vector_norm(self._flat(buf, i))
                            for i in range(self.table.n_tensors)]).float()

    def trigger_norms(self, r):
        """The trigger's per-tensor input for rank r's next decision: ||theta|| (norm) or ||theta - sent|| (drift)."""
        if self.drift:
            return drift_norms(self.theta[r], self.sent[r], self.table.offsets, self.table.numels)
        return self._norms(self.theta[r])

    def _sgd(self, r, grad):
        lr = lr_at(self.lr_table, self.pass_num, self.lr)
        if self.qg:
            qg_sgd_(self.theta[r], self.theta_k[r], grad, self.mom[r], lr, self.mu, self.wd, self.nesterov)
            return
        sgd_(self.theta[r], grad, self.mom[r], lr, self.mu, self.wd, self.nesterov)

    def communicates(self, step: int) -> bool:
        """Does 1-based step `step` gossip (local_steps H: iff H divides it)?"""
        return step % self.local_steps == 0

    def global_avg_step(self, step: int) -> bool:
        """Is 1-based step `step` a global-averaging step (global_avg_period P: iff P divides it)?"""
        return self.global_avg_period > 0 and step % self.global_avg_period == 0

    def slowmo_step(self, step: int) -> bool:
        """Is 1-based step `step` a SlowMo sync step (slowmo_period tau: iff tau divides it)?"""
        return self.slowmo_period > 0 and step % self.slowmo_period == 0

    def round_of(self, step: int) -> int:
        """Gossip round of a communicating step: the one-peer graph's active slot is indexed by it."""
        return step // self.local_steps

    def left(self, r):
        return (r - 1) % self.R

    def right(self, r):
        return (r + 1) % self.R

    @torch.no_grad()
    def step(self, grads: Sequence[torch.Tensor], fires: Optional[Sequence[torch.Tensor]] = None,
             norms: Optional[Sequence[torch.Tensor]] = None) -> None:
        """One training step of every rank (_step), then the consensus measurement when N divides the step."""
        self._step(grads, fires, norms)
        if self.consensus_every and self.pass_num % self.consensus_every == 0:
            self.consensus.append((self.pass_num, *self.consensus_stats()))

    def consensus_stats(self):
        """(D, A) of the ranks' current theta (parallel/trigger.py:consensus_stats); zeros at R = 1."""
        if self.R == 1:
            z = torch.zeros(self.table.n_tensors, dtype=torch.float64)
            return z, z.clone()
        return consensus_stats(self.theta, self.table)

    def _step(self, grads: Sequence[torch.Tensor], fires: Optional[Sequence[torch.Tensor]] = None,
              norms: Optional[Sequence[torch.Tensor]] = None) -> None:
        """`fires` (optional, one bool mask per rank) overrides the trigger decisions -- used to
        compare the data path of a kernel bit-for-bit under the kernel's own decisions; `norms`
        (optional, one [sz] tensor per rank) replaces the oracle's own norm computation (trigger_norms: the drift
        under the drift metric) so the FSM logic can be compared exactly while norm accuracy is tested separately."""
        R, t = self.R, self.table
        self.pass_num += 1
        if self.qg:
            self.theta_k = [th.clone() for th in self.theta]      # before any mix of this step
        if self.algo == "cent":
            g = torch.stack(list(grads)).sum(0) / R if R > 1 else grads[0]
            for r in range(R):
                self._sgd(r, g)
                self.bytes[r] += t.n_elems * 4 if R > 1 else 0
            return
        if self.slowmo_step(self.pass_num):
            return self._step_slowmo(grads)
        if (R == 1 and self.serial_skip) or not self.communicates(self.pass_num):
            for r in range(R):                                 # serial step / local step of --local-steps
                self._sgd(r, grads[r])
            return
        if self.global_avg_step(self.pass_num):
            return self._step_global_avg(grads)
        if self.ed:
            return self._step_ed(grads)
        if self.match:
            return self._step_match(grads)
        if self.cheb_coef is not None:
            return self._step_cheb(grads)
        for _ in range(self.gossip_rounds - 1 if R > 1 else 0):
            self._mix_round()
        rnd = self.round_of(self.pass_num)
        # ---- phase 1: every rank decides and "Puts" (uses pre-mix theta_k) --------------
        if self.algo == "decent":
            fires = [torch.ones(t.n_tensors, dtype=torch.bool) for _ in range(R)]
        elif fires is not None:
            fires = [f.clone().bool().cpu() for f in fires]
        else:
            fires = [trigger_step(self.state[r],
                                  self.trigger_norms(r) if norms is None else norms[r].float().cpu(),
                                  self.pass_num, self.tcfg)
                     for r in range(R)]
        self.fire_history.append([f.clone() for f in fires])
        snap = [th.clone() for th in self.theta]
        n = self.fanout
        for r in range(R):
            L, Rn = self.left(r), self.right(r)
            for i in range(t.n_tensors):
                if not fires[r][i]:
                    continue
                if self.algo != "decent":
                    self.events[r] += n
                src = self._flat(snap[r], i)
                if self.algo == "spevent":
                    pv = self._flat(self.prev[r], i)
                    v, ix = topk_select(src, pv, self.k[i])
                    pv[ix] = v
                    self._flat(self.rep_r[L], i)[ix] = v     # I am my left neighbour's right
                    self._flat(self.rep_l[Rn], i)[ix] = v    # and my right neighbour's left
                    self.bytes[r] += 2 * 2 * self.k[i] * 4
                elif self.q8:
                    enc, dec, msg = codec_of(self.compress)
                    pv = self._padded(self.prev[r], i)
                    deq = dec(*enc(self._padded(snap[r], i) - pv), t.numels[i])
                    pv.add_(deq)
                    self._padded(self.rep_r[L], i).add_(deq)    # I am my left neighbour's right
                    self._padded(self.rep_l[Rn], i).add_(deq)   # and my right neighbour's left
                    self.bytes[r] += 2 * msg(t.numels[i])
                else:
                    outs = self.graphs[r].out_slots()
                    if self.period:                            # one-peer graph: only this round's out-slot
                        outs = [outs[self.graphs[r].active(rnd)]]
                    for p, j in outs:                          # a fired tensor goes into every slot I feed
                        self._flat(self.inbox[p][j], i).copy_(src)
                    if self.drift:                             # one-peer graph: the last value pushed to any peer
                        self._flat(self.sent[r], i).copy_(src)
                    self.bytes[r] += n * t.numels[i] * 4
        if self.gt:
            # y_{k-1} travels with theta_k to both neighbours (every tensor: decent), and doubles the bytes
            for r in range(R):
                self.y_in_r[self.left(r)].copy_(self.y[r])
                self.y_in_l[self.right(r)].copy_(self.y[r])
                self.bytes[r] += 2 * t.n_elems * 4
        # ---- phase 2: mix with whatever the inboxes hold, then SGD -----------------------
        for r in range(R):
            if self.choco_gamma:
                choco_mix_(self.theta[r], self.prev[r], self.rep_l[r], self.rep_r[r], self.choco_gamma)
            elif self.algo == "spevent" or self.q8:
                mix3_(self.theta[r], self.rep_l[r], self.rep_r[r])
            elif self.period:
                mix2_(self.theta[r], self.inbox[r][self.graphs[r].active(rnd)])
            elif self.n_slots == 2:
                mix3_(self.theta[r], self.inbox[r][0], self.inbox[r][1])
            else:
                mixk_(self.theta[r], self.inbox[r])
            if self.gt:
                g = grads[r].to(self.y[r].dtype)
                mix3_(self.y[r], self.y_in_l[r], self.y_in_r[r]).add_(g.sub(self.g_prev[r]))
                self.g_prev[r].copy_(g)
                self._sgd(r, self.y[r])
                continue
            self._sgd(r, grads[r])

    def _mix_round(self) -> None:
        """One mix-only round of --gossip-rounds: every rank pushes its whole theta into every slot it feeds, then every
        rank mixes its inboxes into theta exactly as the step does.  No optimizer, no trigger, no events."""
        R, t = self.R, self.table
        snap = [th.clone() for th in self.theta]
        for r in range(R):
            for p, j in self.graphs[r].out_slots():
                self.inbox[p][j].copy_(snap[r])
            self.bytes[r] += self.fanout * t.n_elems * 4
        for r in range(R):
            if self.n_slots == 2:
                mix3_(self.theta[r], self.inbox[r][0], self.inbox[r][1])
            else:
                mixk_(self.theta[r], self.inbox[r])

    def _step_cheb(self, grads) -> None:
        """Chebyshev-accelerated rounds: Q rounds of push + the step's mix of x_{q-1} (w), each followed by
        cheb_combine_ with (alpha_q, omega_q), then every rank's SGD step on x_Q with no further push or mix."""
        R, t = self.R, self.table
        self.fire_history.append([torch.ones(t.n_tensors, dtype=torch.bool) for _ in range(R)])
        x_prev = [None] * R
        for alpha, omega in self.cheb_coef:
            x = [th.clone() for th in self.theta]
            self._mix_round()
            a = torch.tensor(alpha, dtype=torch.float32)
            o = torch.tensor(omega, dtype=torch.float32)
            for r in range(R):
                cheb_combine_(self.theta[r], x[r], x_prev[r], a, o)
            x_prev = x
        for r in range(R):
            self._sgd(r, grads[r])

    def partners(self, step: int) -> List[Optional[int]]:
        """random-match: the partner of every rank at 1-based step `step` (None: idle)."""
        out: List[Optional[int]] = [None] * self.R
        for a, b in match_pairs(self.topology_seed, self.R, step):
            out[a], out[b] = b, a
        return out

    def _step_match(self, grads) -> None:
        """random-match step: matched ranks swap theta_k through their single inbox and mix (theta + inbox) / 2, then
        every rank takes its SGD step."""
        R, t = self.R, self.table
        part = self.partners(self.pass_num)
        self.fire_history.append([torch.ones(t.n_tensors, dtype=torch.bool) for _ in range(R)])
        snap = [th.clone() for th in self.theta]
        for r in range(R):
            if part[r] is not None:
                self.inbox[part[r]][0].copy_(snap[r])
                self.bytes[r] += t.n_elems * 4
        for r in range(R):
            if part[r] is not None:
                mix2_(self.theta[r], self.inbox[r][0])
            self._sgd(r, grads[r])

    def _step_ed(self, grads) -> None:
        """Exact diffusion: p = sgd(theta_k, g_k), phi = p + (theta_k - psi), psi <- p; phi goes to both neighbours (the
        ring's inboxes, decent's bytes); theta_{k+1} = (phi + ((phi + L) + R) / 3) / 2."""
        R, t = self.R, self.table
        phis = []
        for r in range(R):
            th = self.theta[r].clone()
            self._sgd(r, grads[r])                             # theta[r] <- p
            phis.append(self.theta[r].add(th.sub_(self.psi[r])))
            self.psi[r].copy_(self.theta[r])
        self.fire_history.append([torch.ones(t.n_tensors, dtype=torch.bool) for _ in range(R)])
        for r in range(R):
            self.inbox_r[self.left(r)].copy_(phis[r])         # I am my left neighbour's right
            self.inbox_l[self.right(r)].copy_(phis[r])        # and my right neighbour's left
            self.bytes[r] += 2 * t.n_elems * 4
        for r in range(R):
            tmix = mix3_(phis[r].clone(), self.inbox_l[r], self.inbox_r[r])
            self.theta[r].copy_(phis[r].add(tmix).div_(2))

    def _step_global_avg(self, grads) -> None:
        """Global-averaging step: theta_r <- sgd(rank_mean(theta), g_r) on every rank r."""
        R, t = self.R, self.table
        avg = rank_mean(self.theta)
        for r in range(R):
            self.theta[r].copy_(avg)
            self._sgd(r, grads[r])
            self.bytes[r] += t.n_elems * 4 if R > 1 else 0

    def _step_slowmo(self, grads) -> None:
        """SlowMo sync step: avg = rank_mean(theta); on every rank r the outer update of x_r, u_r, theta_r <- x_r, then
        sgd(theta_r, g_r).  Every rank runs the update on the same inputs, so x and u stay identical across ranks."""
        R, t = self.R, self.table
        avg = rank_mean(self.theta)
        lr = lr_at(self.lr_table, self.pass_num, self.lr)
        for r in range(R):
            slowmo_sync_(self.slowmo_x[r], self.slowmo_u[r], avg, lr, self.slowmo_beta, self.slowmo_lr)
            self.theta[r].copy_(self.slowmo_x[r])
            self._sgd(r, grads[r])
            self.bytes[r] += t.n_elems * 4 if R > 1 else 0

    def final_average(self) -> torch.Tensor:
        return torch.stack(self.theta).sum(0) / self.R

    def total_events(self) -> int:
        return int(sum(self.events))

    def dense_messages(self) -> int:
        """Denominator of 'messages saved': fanout * sz * passes * R (BASELINE.md; 2 on the ring, 2|O| on a static
        graph, 1 on the one-peer graph), times gossip_rounds."""
        return self.gossip_rounds * self.fanout * self.table.n_tensors * self.pass_num * self.R

    def mixing_matrix(self, step: Optional[int] = None) -> torch.Tensor:
        """W [R, R] (float64) of the graph: theta' = W theta for decent without SGD.  It depends on the 1-based step
        (default: the next one) on the one-peer graph, whose slot is that of the step's round, and under local_steps,
        where a step that does not communicate has W = I.  A global-averaging step has W = 11^T / R, and so does the
        average of a SlowMo sync step (before its outer update).  With gossip_rounds Q a gossip step has W^Q.  On
        random-match, W_k pairs the matched ranks with weights 1/2 and leaves the idle rank's row e_r."""
        k = self.pass_num + 1 if step is None else step
        if self.global_avg_step(k) or self.slowmo_step(k):
            return torch.full((self.R, self.R), 1.0 / self.R, dtype=torch.float64)
        if not self.communicates(k):
            return torch.eye(self.R, dtype=torch.float64)
        if self.match or self.period:     # random-match: round_of(k) == k (it refuses local steps)
            return torch.tensor([g.mixing_row(self.round_of(k)) for g in self.graphs], dtype=torch.float64)
        W = torch.tensor([g.mixing_row() for g in self.graphs], dtype=torch.float64)
        if self.cheb_coef is not None:
            # x_q = x_{q-1} + alpha_q (W x_{q-1} - x_{q-1}) + omega_q (x_{q-1} - x_{q-2}), from the fp32 coefficients
            I = torch.eye(self.R, dtype=torch.float64)
            prev, cur = None, I
            for alpha, omega in self.cheb_coef:
                nxt = cur + alpha * (W @ cur - cur)
                if prev is not None:
                    nxt = nxt + omega * (cur - prev)
                prev, cur = cur, nxt
            return cur
        return torch.linalg.matrix_power(W, self.gossip_rounds)
