"""torch.distributed backend (gloo on CPU, NCCL on GPU): the BASELINE path.

It reproduces the reference algorithms with library collectives / point-to-point calls
plus eager elementwise ops -- i.e. what a straightforward port would look like:

  cent    all_reduce(grad)/R + SGD           (/root/reference/dmnist/cent/cent.cpp:130-145)
  decent  isend/irecv theta with both ring neighbours, (t+L+R)/3, SGD
                                            (/root/reference/dmnist/decent/decent.cpp:172-246)
  event   norm trigger -> send only fired tensors -> persistent inboxes -> mix -> SGD
                                            (/root/reference/dcifar10/event/event.cpp:282-479)
  spevent fired tensors travel as (top-k values, indices) records; receiver scatters into
          persistent neighbour replicas      (/root/reference/dcifar10/spevent/spevent.cpp:342-542)
  --compress int8 (decent / event, ring): fired tensors travel as int8 codes of theta - prev plus block scales;
          both ends add the dequantized delta to prev / their replica of it, and the mix reads the replicas;
          --compress sign sends 1-bit scaled signs packed 8 to a byte, and --choco-gamma mixes by choco_mix_
  --gradient-tracking (decent, ring): theta and y travel in one batched exchange; y_k = (y + yL + yR)/3 + g_k - g_prev,
          and SGD steps along y_k
  --local-steps H (decent): only every H-th step runs the exchange and mix; the others are the SGD update alone
  --global-avg-period P (decent): every P-th step all_gathers theta, averages it in rank order and takes the SGD step
  --slowmo-period tau (decent): every tau-th step all_gathers theta, averages it in rank order, applies slowmo_sync_ to
          the outer iterate x and slow momentum u, sets theta <- x and takes the SGD step
  --exact-diffusion (decent, ring): p = SGD(theta), phi = p + (theta - psi), psi <- p; phi travels in the ring exchange,
          and theta <- (phi + (phi + L + R)/3) / 2
  --consensus-every N (decent/event/spevent): after every N-th step all_gathers theta and records consensus_stats
  --quasi-global-momentum (decent/event/spevent): theta_k is snapshotted before the exchange and every SGD update is
          qg_sgd_, whose momentum follows theta_k - theta_{k+1}
  --topology random-match (decent): at step k each matched rank swaps theta with its partner of match_pairs(seed, R, k)
          (one batch_isend_irecv) and mixes add_ then div_(2); the idle rank of an odd R takes its SGD step only
  --gossip-rounds Q (decent, ring / static graph): Q - 1 exchanges of theta, each followed by the step's own mix, then
          the unchanged decent step
  --gossip-accel chebyshev (decent, ring / static graph): Q exchanges of theta, each followed by the step's own mix and
          cheb_combine_ with x_{q-1} and x_{q-2}, then the optimizer alone

torch.distributed has no one-sided RMA, so the "window" is emulated with an iteration-
synchronous exchange: first the fire masks, then a payload holding only the fired tensors.
Bytes on the wire therefore scale with events exactly as with MPI_Put, but every step is
a rendezvous (sync_mode=iter semantics).  This is the number the fused P2P backend beats;
on gloo it doubles as the GPU-free plumbing for BASELINE config 1.
"""
from __future__ import annotations

from typing import List

import torch
import torch.distributed as dist

from .base import (CommBackend, StepLog, check_compress_state, check_exact_diffusion_state, check_global_avg_state,
                   check_choco_state, check_local_steps_state, check_qg_state, check_slowmo_state, check_topology_state,
                   check_tracking_state, check_trigger_state, slowmo_state)
from .topology import chebyshev_coefficients, is_match
from .trigger import (Q8_BLOCK, TriggerConfig, TriggerState, cheb_combine_, choco_mix_, codec_of, consensus_stats,
                      drift_norms, mix2_, mix3_, mixk_, qg_sgd_, rank_mean, sgd_, slowmo_sync_, topk_select,
                      trigger_step)


class CollectiveBackend(CommBackend):
    name = "collective"

    def __init__(self, cfg, arena, ring, group=None):
        super().__init__(cfg, arena, ring)
        self.group = group
        self.name = dist.get_backend(group) if dist.is_initialized() else "local"
        t = arena.table
        dev = arena.theta.device
        self.tcfg = TriggerConfig.from_train(cfg)
        self.state = TriggerState(t.n_tensors, cfg.sent_history, dev)
        self.events = 0
        self.bytes = 0
        self.recv_rms = cfg.dataset == "mnist"      # MNIST logs RMS, CIFAR L2 (SURVEY H5)
        gossip = cfg.algo in ("decent", "event", "spevent")
        # --compress int8 (decent/event, ring): fired tensors travel as int8 codes of theta - prev plus one scale per
        # block; prev and the neighbour replicas start from theta_0 (identical on all ranks), the mix reads the replicas
        self.compress = getattr(cfg, "compress", "none")
        self.q8 = gossip and self.compress in ("int8", "sign")
        # --choco-gamma (int8 / sign): the CHOCO consensus step on the public copies replaces the mix of the replicas
        self.choco_gamma = float(getattr(cfg, "choco_gamma", 0.0)) if self.q8 else 0.0
        if self.q8:
            self.prev = arena.theta.clone()
            self.rep_l = arena.theta.clone()
            self.rep_r = arena.theta.clone()
        elif gossip:
            if cfg.algo == "spevent":
                # Q8: replicas / prev start from theta_0 (identical on all ranks), not fresh random nets
                self.prev = arena.theta.clone()
                self.rep_l = arena.theta.clone()
                self.rep_r = arena.theta.clone()
                self.k = t.topk_counts(cfg.topk_percent)
            elif getattr(ring, "is_ring", True):
                # RMA window halves, zero-initialised (event.cpp:144-147)
                self.inbox_l = torch.zeros_like(arena.theta)
                self.inbox_r = torch.zeros_like(arena.theta)
            else:
                # circulant or one-peer graph (parallel/topology.py): one zero-initialised inbox per slot
                self.inbox = [torch.zeros_like(arena.theta) for _ in range(ring.n_slots)]
        # drift trigger: what my receivers hold of my parameters (event: zero like their inboxes, the pushed theta_k of
        # every fired tensor afterwards; spevent: prev, which the top-k pushes already keep element-wise)
        self.drift = cfg.algo in ("event", "spevent") and self.tcfg.metric == "drift"
        if self.drift:
            self.sent = self.prev if (cfg.algo == "spevent" or self.q8) else torch.zeros_like(arena.theta)
        # --gradient-tracking (decent, ring): y, the previous gradient and the y inboxes, all zero at start.  R = 1 runs
        # the plain step (tracking reduces to SGD on g)
        self.gt = cfg.algo == "decent" and bool(getattr(cfg, "gradient_tracking", False)) and ring.world > 1
        if self.gt:
            self.y, self.g_prev = torch.zeros_like(arena.theta), torch.zeros_like(arena.theta)
            self.y_in_l, self.y_in_r = torch.zeros_like(arena.theta), torch.zeros_like(arena.theta)
        # --exact-diffusion (decent, ring): psi, the previous optimizer output, starts at theta_0 (identical on every
        # rank).  R = 1 runs the plain step
        self.ed = cfg.algo == "decent" and bool(getattr(cfg, "exact_diffusion", False)) and ring.world > 1
        if self.ed:
            self.psi = arena.theta.clone()
        # --local-steps H (decent): step k gossips iff H divides k, as round k / H; the other steps are _opt() alone
        self.local_steps = int(getattr(cfg, "local_steps", 1)) if cfg.algo == "decent" else 1
        # --global-avg-period P (decent): step k with P dividing k averages theta over all ranks instead of gossiping
        self.global_avg_period = int(getattr(cfg, "global_avg_period", 0)) if cfg.algo == "decent" else 0
        # --quasi-global-momentum: step() snapshots theta_k, and _opt() runs qg_sgd_ on it (every step, also local and
        # serial ones)
        self.qg = gossip and bool(getattr(cfg, "quasi_global_momentum", False))
        # --slowmo-period tau (decent): step k with tau dividing k averages theta over all ranks, then the outer update of
        # x (theta_0 at start) and u (zero at start), identical on every rank; the other steps are the base steps
        self.slowmo_period = int(getattr(cfg, "slowmo_period", 0)) if cfg.algo == "decent" else 0
        self.slowmo_beta = float(getattr(cfg, "slowmo_beta", 0.5))
        self.slowmo_lr = float(getattr(cfg, "slowmo_lr", 1.0))
        if self.slowmo_period:
            self.slowmo_x, self.slowmo_u = arena.theta.clone(), torch.zeros_like(arena.theta)
        # --consensus-every N: after step k with N dividing k, (k, D, A) of every rank's theta; the all_gather is not
        # counted in bytes_sent
        self.consensus_every = int(getattr(cfg, "consensus_every", 0)) if gossip else 0
        self.consensus_rows = []
        # --gossip-rounds Q (decent, R >= 2): Q - 1 mix-only rounds before the decent step's exchange
        self.gossip_rounds = int(getattr(cfg, "gossip_rounds", 1)) if cfg.algo == "decent" and ring.world > 1 else 1
        # --gossip-accel chebyshev (decent, R >= 2): each of the Q rounds combines its mix with x_{q-1} and x_{q-2} by
        # the fp32 (alpha_q, omega_q) of parallel/topology.py, as 0-dim tensors on theta's device
        self.cheb_coef = None
        if getattr(cfg, "gossip_accel", "none") == "chebyshev" and cfg.algo == "decent" and ring.world > 1:
            f = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)
            self.cheb_coef = [(f(al), f(om)) for al, om in
                              chebyshev_coefficients(ring.offsets, ring.world, self.gossip_rounds)]
        self.theta_k = None
        if self.want_logs:
            z = lambda: torch.zeros(t.n_tensors, dtype=torch.float32, device=dev)
            self.last_recv_norm_l, self.last_recv_norm_r = z(), z()

    # ------------------------------------------------------------------ helpers
    def _flat(self, buf, i):
        return self.arena.flat(buf, i)

    def _exchange(self, to_left: List[torch.Tensor], to_right: List[torch.Tensor],
                  from_left: List[torch.Tensor], from_right: List[torch.Tensor]) -> None:
        """One rendezvous with both neighbours. When left == right (R == 2) the two payloads are
        identical by construction, so a single message is sent and used for both halves."""
        ring = self.ring
        if ring.world == 1:
            for d, s in zip(from_right, to_left):
                d.copy_(s)
            for d, s in zip(from_left, to_right):
                d.copy_(s)
            return
        ops = []
        if ring.left == ring.right:
            peer = ring.left
            for s in to_left:
                ops.append(dist.P2POp(dist.isend, s, peer, self.group))
            for d in from_left:
                ops.append(dist.P2POp(dist.irecv, d, peer, self.group))
            if ops:
                for w in dist.batch_isend_irecv(ops):
                    w.wait()
            for d, s in zip(from_right, from_left):
                d.copy_(s)
            return
        for s in to_left:
            ops.append(dist.P2POp(dist.isend, s, ring.left, self.group))
        for s in to_right:
            ops.append(dist.P2POp(dist.isend, s, ring.right, self.group))
        for d in from_left:
            ops.append(dist.P2POp(dist.irecv, d, ring.left, self.group))
        for d in from_right:
            ops.append(dist.P2POp(dist.irecv, d, ring.right, self.group))
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()

    def _active_slots(self) -> List[int]:
        """Slots that take part in this step: all of a static graph, the one active slot of a one-peer graph."""
        g = self.ring
        return [g.active(self.pass_num // self.local_steps)] if g.period else list(range(g.n_slots))

    def _exchange_slots(self, payload: torch.Tensor, recv: List[torch.Tensor]) -> None:
        """Graph rendezvous over the active slots: `payload` goes into every active slot I feed (out-slot j = slot j of
        its peer), recv[s] receives active slot s (the other entries are left alone).  The tag is the slot index, so
        two slots fed by the same peer (offset R/2) cannot cross.  One-peer graph: one isend to the step's out-peer
        and one irecv from its in-peer."""
        g = self.ring
        act, outs, ins = self._active_slots(), g.out_slots(), g.slots()
        ops = [dist.P2POp(dist.isend, payload, outs[j][0], self.group, tag=outs[j][1]) for j in act]
        ops += [dist.P2POp(dist.irecv, recv[s], ins[s], self.group, tag=s) for s in act]
        for w in dist.batch_isend_irecv(ops):
            w.wait()

    def _mix_slots(self) -> None:
        """Static graph: mixk_ over every slot.  One-peer graph: (theta + active slot) / 2, the slot of this round."""
        if self.ring.period:
            mix2_(self.arena.theta, self.inbox[self.ring.active(self.pass_num // self.local_steps)])
        else:
            mixk_(self.arena.theta, self.inbox)

    def _opt(self) -> None:
        a, cfg = self.arena, self.cfg
        if self.qg:
            qg_sgd_(a.theta, self.theta_k, a.grad, a.mom, self.step_lr(self.pass_num), cfg.momentum, cfg.weight_decay,
                    cfg.nesterov)
            return
        sgd_(a.theta, a.grad, a.mom, self.step_lr(self.pass_num), cfg.momentum, cfg.weight_decay, cfg.nesterov)

    # ------------------------------------------------------------------ step
    @torch.no_grad()
    def step(self) -> None:
        self.pass_num += 1
        algo = self.cfg.algo
        if self.qg:
            self.theta_k = self.arena.theta.clone()    # before the exchange and the mix
        if algo == "cent":
            self._step_cent()
        elif self.slowmo_period and self.pass_num % self.slowmo_period == 0:
            self._step_slowmo()                        # also at R = 1: the outer update on the own theta
        elif not self.comm_enabled or self.pass_num % self.local_steps:
            self._opt()                                # serial step / local step of --local-steps
        elif self.global_avg_period and self.pass_num % self.global_avg_period == 0:
            self._step_global_avg()
        elif algo == "decent":
            self._step_decent()
        elif algo == "event":
            self._step_event()
        else:
            self._step_spevent()
        if self.consensus_every and self.pass_num % self.consensus_every == 0:
            self.consensus_rows.append((self.pass_num, *self.measure_consensus()))

    def measure_consensus(self):
        """(D, A) of every rank's current theta: all_gather, then consensus_stats (zeros at R = 1, no collective)."""
        a = self.arena
        if self.ring.world == 1:
            z = torch.zeros(a.table.n_tensors, dtype=torch.float64)
            return z, z.clone()
        parts = [torch.empty_like(a.theta) for _ in range(self.ring.world)]
        dist.all_gather(parts, a.theta, group=self.group)
        return consensus_stats(parts, a.table)

    def drain_consensus(self):
        out, self.consensus_rows = self.consensus_rows, []
        return out

    def _step_cent(self) -> None:
        a = self.arena
        if self.ring.world > 1:
            dist.all_reduce(a.grad, op=dist.ReduceOp.SUM, group=self.group)
            a.grad.div_(self.ring.world)
            self.bytes += a.table.n_elems * 4
        self._opt()

    def _step_decent(self) -> None:
        a = self.arena
        if self.q8:
            return self._step_q8([True] * a.table.n_tensors, None)
        if self.gt:
            return self._step_tracking()
        if self.ed:
            return self._step_ed()
        if self.cheb_coef is not None:
            # --gossip-accel chebyshev: theta <- P_Q(W) theta, one exchange, mix and combine per round
            x_prev = None
            for alpha, omega in self.cheb_coef:
                x = a.theta.clone()
                self._mix_round()
                cheb_combine_(a.theta, x, x_prev, alpha, omega)
                x_prev = x
            return self._opt()
        for _ in range(self.gossip_rounds):            # --gossip-rounds Q: Q - 1 mix-only rounds, then the step's mix
            self._mix_round()
        self._opt()

    def _mix_round(self) -> None:
        """Exchange theta with every neighbour slot and mix it in (mix3_ on the ring, mixk_ on a graph): the decent
        step without its optimizer, and one round of --gossip-rounds."""
        a = self.arena
        if is_match(self.ring):
            return self._match_round()
        if hasattr(self, "inbox"):
            self._exchange_slots(a.theta, self.inbox)
            self.bytes += self.ring.fanout * a.table.n_elems * 4
            self._mix_slots()
            return
        self._exchange([a.theta], [a.theta], [self.inbox_l], [self.inbox_r])
        self.bytes += 2 * a.table.n_elems * 4
        mix3_(a.theta, self.inbox_l, self.inbox_r)

    def _match_round(self) -> None:
        """random-match: swap theta with this step's partner and mix (theta + received) / 2 -- add_ then div_(2), the
        kernel's __fadd_rn / __fdiv_rn.  Both partners form the same sum, so they hold bitwise-equal theta after it.
        An idle rank (odd R) exchanges nothing."""
        a = self.arena
        p = self.ring.partner(self.pass_num)
        if p is None:
            return
        ops = [dist.P2POp(dist.isend, a.theta, p, self.group), dist.P2POp(dist.irecv, self.inbox[0], p, self.group)]
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        self.bytes += a.table.n_elems * 4
        mix2_(a.theta, self.inbox[0])

    def _step_global_avg(self) -> None:
        """Global-averaging step, the simulator's ops: theta <- rank_mean(every rank's theta), then SGD on the own
        gradient and momentum.  all_gather gives every rank the same R tensors, so every rank forms the same mean."""
        a = self.arena
        if self.ring.world > 1:
            parts = [torch.empty_like(a.theta) for _ in range(self.ring.world)]
            dist.all_gather(parts, a.theta, group=self.group)
            a.theta.copy_(rank_mean(parts))
            self.bytes += a.table.n_elems * 4
        self._opt()

    def _step_slowmo(self) -> None:
        """SlowMo sync step, the simulator's ops: avg = rank_mean(every rank's theta), slowmo_sync_(x, u, avg), theta <- x,
        then SGD on the own gradient and momentum.  Every rank forms the same mean and runs the same update, so x and u
        stay identical across ranks."""
        a = self.arena
        if self.ring.world > 1:
            parts = [torch.empty_like(a.theta) for _ in range(self.ring.world)]
            dist.all_gather(parts, a.theta, group=self.group)
            self.bytes += a.table.n_elems * 4
        else:
            parts = [a.theta]
        slowmo_sync_(self.slowmo_x, self.slowmo_u, rank_mean(parts), self.step_lr(self.pass_num), self.slowmo_beta,
                     self.slowmo_lr)
        a.theta.copy_(self.slowmo_x)
        self._opt()

    def _step_tracking(self) -> None:
        """Gradient tracking: theta_k and y_{k-1} to both neighbours in one batched exchange, then the simulator's ops:
        y <- mix3_(y, yL, yR) + (g - g_prev), g_prev <- g, theta <- mix3_(theta, L, R), SGD along y."""
        a = self.arena
        self._exchange([a.theta, self.y], [a.theta, self.y], [self.inbox_l, self.y_in_l], [self.inbox_r, self.y_in_r])
        self.bytes += 2 * 2 * a.table.n_elems * 4
        mix3_(self.y, self.y_in_l, self.y_in_r).add_(a.grad.sub(self.g_prev))
        self.g_prev.copy_(a.grad)
        mix3_(a.theta, self.inbox_l, self.inbox_r)
        sgd_(a.theta, self.y, a.mom, self.step_lr(self.pass_num), self.cfg.momentum, self.cfg.weight_decay,
             self.cfg.nesterov)

    def _step_ed(self) -> None:
        """Exact diffusion, the simulator's ops: p = SGD(theta_k), phi = p + (theta_k - psi), psi <- p, phi to both
        neighbours in the ring exchange, theta <- (phi + mix3_(phi, L, R)) / 2."""
        a = self.arena
        t = a.theta.clone()
        self._opt()                                    # theta <- p
        phi = a.theta.add(t.sub_(self.psi))
        self.psi.copy_(a.theta)
        self._exchange([phi], [phi], [self.inbox_l], [self.inbox_r])
        self.bytes += 2 * a.table.n_elems * 4
        a.theta.copy_(phi.add(mix3_(phi.clone(), self.inbox_l, self.inbox_r)).div_(2))

    def _fire(self):
        a = self.arena
        t = a.table
        norms = drift_norms(a.theta, self.sent, t.offsets, t.numels) if self.drift else a.tensor_norms()
        fire = trigger_step(self.state, norms, self.pass_num, self.tcfg)
        return norms, fire

    def _mark_sent(self, mine) -> None:
        """Drift trigger, event: the fired tensors' theta_k is now what the receivers hold."""
        if self.drift and self.cfg.algo == "event":
            for i, f in enumerate(mine):
                if f:
                    self._flat(self.sent, i).copy_(self._flat(self.arena.theta, i))

    def _masks(self, fire: torch.Tensor):
        """Exchange fire masks with both neighbours; returns host bool lists (mine, left's, right's)."""
        m = fire.to(torch.uint8)
        ml, mr = torch.empty_like(m), torch.empty_like(m)
        self._exchange([m], [m], [ml], [mr])
        return fire.tolist(), ml.bool().tolist(), mr.bool().tolist()

    def _step_event_graph(self) -> None:
        """event on a graph: fire masks per active slot, then one payload of my fired tensors into every active slot
        (every slot of a static graph, the step's one slot of a one-peer graph)."""
        a, t = self.arena, self.arena.table
        n, fan = len(self.inbox), self.ring.fanout
        act = self._active_slots()
        _, fire = self._fire()
        m = fire.to(torch.uint8)
        masks = [torch.empty_like(m) for _ in range(n)]
        self._exchange_slots(m, masks)
        mine = fire.tolist()
        self.events += fan * sum(mine)
        sent = [self._flat(a.theta, i) for i in range(t.n_tensors) if mine[i]]
        payload = torch.cat(sent) if sent else a.theta.new_empty(0)
        self._mark_sent(mine)
        self.bytes += fan * payload.numel() * 4
        masks = {s: masks[s].bool().tolist() for s in act}
        bufs = [None] * n
        for s in act:
            bufs[s] = a.theta.new_empty(sum(t.numels[i] for i in range(t.n_tensors) if masks[s][i]))
        self._exchange_slots(payload, bufs)
        for s in act:
            off = 0
            for i in range(t.n_tensors):
                if masks[s][i]:
                    k = t.numels[i]
                    self._flat(self.inbox[s], i).copy_(bufs[s][off:off + k])
                    off += k
        self._mix_slots()
        self._opt()

    def _padded(self, buf, i):
        """Tensor i's whole tiles: the blocks of the int8 codec (parallel/trigger.py q8_encode)."""
        t = self.arena.table
        return buf[t.offsets[i]: t.offsets[i] + t.tile_count[i] * t.tile]

    def _step_q8(self, mine, masks) -> None:
        """Compressed ring step: my fired tensors' codes of theta - prev (int8: one byte per element; sign: one bit,
        packed 8 to a byte) and their block scales go to both neighbours (decent: every tensor; event: after the
        fire-mask exchange, `masks` = (left's, right's)); each side adds the dequantized delta to prev / to its replica of
        the sender's prev, then theta <- ((theta + rep_l) + rep_r) / 3 (--choco-gamma: choco_mix_) and SGD."""
        a, t = self.arena, self.arena.table
        enc, dec, msg = codec_of(self.compress)
        per = 8 if self.compress == "sign" else 1          # arena elements per code byte
        cdt = torch.uint8 if self.compress == "sign" else torch.int8
        lm, rm = masks if masks is not None else (mine, mine)
        qs, ss = [], []
        for i in range(t.n_tensors):
            if mine[i]:
                pv = self._padded(self.prev, i)
                q, s = enc(self._padded(a.theta, i) - pv)
                pv.add_(dec(q, s, t.numels[i]))
                qs.append(q)
                ss.append(s)
                self.bytes += 2 * msg(t.numels[i])
        pq = torch.cat(qs) if qs else torch.empty(0, dtype=cdt, device=a.theta.device)
        ps = torch.cat(ss) if ss else a.theta.new_empty(0)
        blocks = [t.tile_count[i] * t.tile for i in range(t.n_tensors)]
        nl = sum(blocks[i] for i in range(t.n_tensors) if lm[i])
        nr = sum(blocks[i] for i in range(t.n_tensors) if rm[i])
        ql = torch.empty(nl // per, dtype=cdt, device=a.theta.device)
        qr = torch.empty(nr // per, dtype=cdt, device=a.theta.device)
        sl, sr = a.theta.new_empty(nl // Q8_BLOCK), a.theta.new_empty(nr // Q8_BLOCK)
        self._exchange([pq, ps], [pq, ps], [ql, sl], [qr, sr])
        for mask, qb, sb, rep in ((lm, ql, sl, self.rep_l), (rm, qr, sr, self.rep_r)):
            off = 0
            for i in range(t.n_tensors):
                if mask[i]:
                    n = blocks[i]
                    self._padded(rep, i).add_(dec(qb[off // per:(off + n) // per],
                                                  sb[off // Q8_BLOCK:(off + n) // Q8_BLOCK], t.numels[i]))
                    off += n
        if self.choco_gamma:
            choco_mix_(a.theta, self.prev, self.rep_l, self.rep_r, self.choco_gamma)
        else:
            mix3_(a.theta, self.rep_l, self.rep_r)
        self._opt()

    def _step_event(self) -> None:
        if hasattr(self, "inbox"):
            return self._step_event_graph()
        if self.q8:
            _, fire = self._fire()
            mine, lm, rm = self._masks(fire)
            self.events += 2 * sum(mine)
            return self._step_q8(mine, (lm, rm))
        a, t = self.arena, self.arena.table
        thres_used = None
        if self.want_logs:
            # threshold as used in the comparison (after the horizon decay / constant set)
            tmp = self.state.clone()
        norms, fire = self._fire()
        mine, lm, rm = self._masks(fire)
        nfired = sum(mine)
        self.events += 2 * nfired
        sent = [self._flat(a.theta, i) for i in range(t.n_tensors) if mine[i]]
        payload = torch.cat(sent) if sent else a.theta.new_empty(0)
        self._mark_sent(mine)
        self.bytes += 2 * payload.numel() * 4
        nl = sum(t.numels[i] for i in range(t.n_tensors) if lm[i])
        nr = sum(t.numels[i] for i in range(t.n_tensors) if rm[i])
        bl, br = a.theta.new_empty(nl), a.theta.new_empty(nr)
        self._exchange([payload], [payload], [bl], [br])
        for mask, buf, inbox in ((lm, bl, self.inbox_l), (rm, br, self.inbox_r)):
            off = 0
            for i in range(t.n_tensors):
                if mask[i]:
                    n = t.numels[i]
                    self._flat(inbox, i).copy_(buf[off:off + n])
                    off += n
        if self.want_logs:
            self._log(tmp, norms, fire, self.inbox_l, self.inbox_r)
        mix3_(a.theta, self.inbox_l, self.inbox_r)
        self._opt()

    def _step_spevent(self) -> None:
        a, t = self.arena, self.arena.table
        if self.want_logs:
            tmp = self.state.clone()
        norms, fire = self._fire()
        mine, lm, rm = self._masks(fire)
        self.events += 2 * sum(mine)
        vals, idxs = [], []
        for i in range(t.n_tensors):
            if mine[i]:
                th, pv = self._flat(a.theta, i), self._flat(self.prev, i)
                v, ix = topk_select(th, pv, self.k[i])
                pv[ix] = v                                   # spevent.cpp:407-413
                vals.append(v)
                idxs.append(ix.to(torch.int32))
        if vals:
            payload = torch.cat([torch.cat(vals), torch.cat(idxs).view(torch.float32)])
        else:
            payload = a.theta.new_empty(0)
        self.bytes += 2 * payload.numel() * 4
        kl = sum(self.k[i] for i in range(t.n_tensors) if lm[i])
        kr = sum(self.k[i] for i in range(t.n_tensors) if rm[i])
        bl, br = a.theta.new_empty(2 * kl), a.theta.new_empty(2 * kr)
        self._exchange([payload], [payload], [bl], [br])
        for mask, buf, ktot, rep in ((lm, bl, kl, self.rep_l), (rm, br, kr, self.rep_r)):
            off = 0
            for i in range(t.n_tensors):
                if mask[i]:
                    k = self.k[i]
                    v = buf[off:off + k]
                    ix = buf[ktot + off: ktot + off + k].view(torch.int32).long()
                    self._flat(rep, i)[ix] = v               # spevent.cpp:438-448
                    off += k
        if self.want_logs:
            self._log(tmp, norms, fire, self.rep_l, self.rep_r)
        mix3_(a.theta, self.rep_l, self.rep_r)
        self._opt()

    # ------------------------------------------------------------------ logging
    def _log(self, before: TriggerState, norms, fire, lbuf, rbuf) -> None:
        t = self.arena.table
        if self.tcfg.thres_type == 1:
            thres_used = before.thres * float(torch.tensor(self.tcfg.horizon, dtype=torch.float32))
        else:
            thres_used = torch.full_like(before.thres, self.tcfg.constant)
        ln = self.arena.tensor_norms(lbuf)
        rn = self.arena.tensor_norms(rbuf)
        if self.recv_rms:
            n = torch.tensor(t.numels, dtype=torch.float32, device=ln.device)
            ln, rn = ln / n.sqrt(), rn / n.sqrt()
        lnew = (ln - self.last_recv_norm_l).abs() > 0
        rnew = (rn - self.last_recv_norm_r).abs() > 0
        self.last_recv_norm_l = torch.where(lnew, ln, self.last_recv_norm_l)
        self.last_recv_norm_r = torch.where(rnew, rn, self.last_recv_norm_r)
        self.logs.append(StepLog(self.pass_num, norms.cpu(), thres_used.cpu(), fire.cpu(),
                                 ln.cpu(), rn.cpu(), lnew.cpu(), rnew.cpu()))

    # ------------------------------------------------------------------ end of training
    @torch.no_grad()
    def final_average(self) -> None:
        """All-reduce the parameters (event.cpp:509-519). The reference divides on rank 0 only
        (Q5); by default every rank divides so all ranks hold the averaged model."""
        if self.ring.world == 1:
            return
        a = self.arena
        dist.all_reduce(a.theta, op=dist.ReduceOp.SUM, group=self.group)
        if self.cfg.final_divide_all or self.ring.rank == 0:
            a.theta.div_(self.ring.world)

    def num_events(self) -> int:
        return int(self.events)

    def total_events(self) -> int:
        if self.ring.world == 1:
            return int(self.events)
        e = torch.tensor([self.events], dtype=torch.int64, device=self.arena.theta.device)
        dist.all_reduce(e, group=self.group)
        return int(e.item())

    def bytes_sent(self) -> int:
        return int(self.bytes)

    def synchronize(self) -> None:
        if self.arena.theta.is_cuda:
            torch.cuda.synchronize()

    def state_dict(self):
        sd = {"pass_num": self.pass_num, "events": self.events, "bytes": self.bytes,
              "fsm": self.state.state_dict()}
        for k in ("inbox_l", "inbox_r", "prev", "rep_l", "rep_r"):
            if hasattr(self, k):
                sd[k] = getattr(self, k).cpu().clone()
        if self.cfg.algo == "decent":
            sd["gradient_tracking"] = self.gt
            sd["local_steps"] = self.local_steps
            if self.global_avg_period:
                sd["global_avg_period"] = self.global_avg_period
            sd["exact_diffusion"] = self.ed
            sd.update(slowmo_state(self))
            if self.gt:
                for k in ("y", "g_prev", "y_in_l", "y_in_r"):
                    sd[k] = getattr(self, k).cpu().clone()
            if self.ed:
                sd["psi"] = self.psi.cpu().clone()
        if self.qg:
            sd["quasi_global_momentum"] = True      # the arena's momentum holds m_hat
        if self.cfg.algo in ("decent", "event"):
            sd["compress"] = self.compress          # int8 / sign: prev / rep_l / rep_r are saved above
            if self.choco_gamma:
                sd["choco_gamma"] = self.choco_gamma
        if self.cfg.algo in ("event", "spevent"):
            sd["trigger"] = self.tcfg.metric
            if self.drift and self.cfg.algo == "event" and not self.q8:
                sd["sent"] = self.sent.cpu().clone()
        if hasattr(self, "inbox"):
            sd["topology_offsets"] = list(self.ring.offsets)
            if self.ring.period:
                sd["topology"] = self.ring.kind
            if is_match(self.ring):
                sd["topology"], sd["topology_seed"] = self.ring.kind, int(self.ring.seed)
            for s, ib in enumerate(self.inbox):
                sd[f"inbox_{s}"] = ib.cpu().clone()
        return sd

    def load_state_dict(self, sd):
        self.pass_num = int(sd["pass_num"])
        self.events = int(sd["events"])
        self.bytes = int(sd.get("bytes", 0))
        check_topology_state(sd, self.ring, self.cfg.algo)
        check_trigger_state(sd, self.tcfg.metric, self.cfg.algo)
        check_compress_state(sd, self.compress, self.cfg.algo)
        check_choco_state(sd, self.choco_gamma, self.cfg.algo)
        check_tracking_state(sd, self.gt, self.cfg.algo)
        check_local_steps_state(sd, self.local_steps, self.cfg.algo)
        check_global_avg_state(sd, self.global_avg_period, self.cfg.algo)
        check_exact_diffusion_state(sd, self.ed, self.cfg.algo)
        check_qg_state(sd, self.qg, self.cfg.algo)
        check_slowmo_state(sd, self.slowmo_period, self.slowmo_beta, self.slowmo_lr, self.cfg.algo)
        self.state.load_state_dict(sd["fsm"])
        if self.slowmo_period:
            self.slowmo_x.copy_(sd["slowmo_x"].to(self.slowmo_x.device))
            self.slowmo_u.copy_(sd["slowmo_u"].to(self.slowmo_u.device))
        if self.ed:
            self.psi.copy_(sd["psi"].to(self.psi.device))
        if self.gt:
            for k in ("y", "g_prev", "y_in_l", "y_in_r"):
                getattr(self, k).copy_(sd[k].to(getattr(self, k).device))
        if self.drift and self.cfg.algo == "event" and not self.q8:
            self.sent.copy_(sd["sent"].to(self.sent.device))
        if hasattr(self, "inbox"):
            for s, ib in enumerate(self.inbox):
                ib.copy_(sd[f"inbox_{s}"].to(ib.device))
        for k in ("inbox_l", "inbox_r", "prev", "rep_l", "rep_r"):
            if hasattr(self, k) and k in sd:
                getattr(self, k).copy_(sd[k].to(getattr(self, k).device))
