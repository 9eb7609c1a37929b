"""Reference-STRUCTURED backend: what a straight port of the reference's main() looks like.

The real reference cannot be built offline (no MPI / OpenCV C++ / datasets, DESIGN.md section 7), so this
backend reproduces its *structure* on torch.distributed for same-box A/B measurements:

  * one pass over the parameter tensors per step, in named_parameters() order;
  * per tensor: flatten + pack, `norm().item()` (a host sync per tensor, event.cpp:300), the scalar
    trigger logic on the host (event.cpp:301-355), a per-tensor message to each neighbour (the
    MPI_Put pair, :322-332 -- emulated as flag + payload sends because torch.distributed has no
    one-sided RMA), unpack of both inbox halves with their norms `.item()` (:372-424), and the
    three in-place ops add_, add_, div_(3) (:459-461);
  * then optimizer.step() over the whole model (:479).

Numerically identical to CollectiveBackend / the simulator (same arithmetic, iter-sync exchange);
it exists only to be slow in exactly the way the reference is.  `bench.py --impl refport`.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from .collective import CollectiveBackend


class ReferenceStyleBackend(CollectiveBackend):
    name = "refport"

    def __init__(self, cfg, arena, ring, group=None):
        super().__init__(cfg, arena, ring, group)
        t = arena.table
        H = max(1, cfg.sent_history)
        # host-resident scalar state, exactly like the calloc'ed arrays of the reference (event.cpp:150-194)
        self.h_thres = [0.0] * t.n_tensors
        self.h_last_norm = [0.0] * t.n_tensors
        self.h_last_iter = [0.0] * t.n_tensors
        self.h_slopes = [[0.0] * H for _ in range(t.n_tensors)]
        self.host_syncs = 0

    @staticmethod
    def _f32(x: float) -> float:
        return float(torch.tensor(x, dtype=torch.float32))

    def _send_recv_tensor(self, fired: bool, payload: torch.Tensor, inbox_l: torch.Tensor, inbox_r: torch.Tensor):
        """Per-tensor exchange with both neighbours: a 1-element 'fired' flag, then the tensor if fired."""
        ring = self.ring
        dev = payload.device
        flag = torch.tensor([1.0 if fired else 0.0], device=dev)
        fl, fr = torch.zeros(1, device=dev), torch.zeros(1, device=dev)
        if ring.world == 1:
            fl.copy_(flag); fr.copy_(flag)
            if fired:
                inbox_l.copy_(payload); inbox_r.copy_(payload)
            return
        peers = [(ring.left, fl, inbox_l)] if ring.left == ring.right else [(ring.left, fl, inbox_l), (ring.right, fr, inbox_r)]
        ops = []
        for peer, f_in, _ in peers:
            ops.append(dist.P2POp(dist.isend, flag, peer, self.group))
            ops.append(dist.P2POp(dist.irecv, f_in, peer, self.group))
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        ops = []
        for peer, f_in, box in peers:
            if fired:
                ops.append(dist.P2POp(dist.isend, payload, peer, self.group))
            self.host_syncs += 1
            if f_in.item() > 0:                                   # host sync, like every MPI call of the reference
                ops.append(dist.P2POp(dist.irecv, box, peer, self.group))
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        if ring.left == ring.right:
            inbox_r.copy_(inbox_l)

    @torch.no_grad()
    def _step_event(self) -> None:
        a, t, cfg = self.arena, self.arena.table, self.cfg
        f32 = self._f32
        for i in range(t.n_tensors):
            flat = self._flat(a.theta, i)
            temp = flat.clone()                                    # pack (memcpy, event.cpp:296-297)
            curr_norm = f32(torch.linalg.vector_norm(flat).item())
            self.host_syncs += 1
            value_diff = f32(abs(f32(curr_norm - self.h_last_norm[i])))
            iter_diff = f32(self.pass_num - self.h_last_iter[i])
            self.h_thres[i] = f32(self.h_thres[i] * f32(cfg.horizon)) if cfg.thres_type == 1 else f32(cfg.constant)
            fired = value_diff >= self.h_thres[i] or self.pass_num < cfg.initial_comm_passes
            if fired:
                self.events += 2
                self.bytes += 2 * t.numels[i] * 4
                sl = self.h_slopes[i]
                sl[:] = sl[1:] + [f32(value_diff / iter_diff)]
                if cfg.thres_type == 1:
                    self.h_thres[i] = f32(sum(sl) / cfg.sent_history)
                self.h_last_norm[i] = curr_norm
                self.h_last_iter[i] = float(self.pass_num)
            il, ir = self._flat(self.inbox_l, i), self._flat(self.inbox_r, i)
            self._send_recv_tensor(fired, temp, il, ir)
            _ = torch.linalg.vector_norm(il).item(), torch.linalg.vector_norm(ir).item()   # receive-side norms (:379,:423)
            self.host_syncs += 2
            flat.add_(il).add_(ir).div_(3)                         # event.cpp:459-461
        self._opt()

    @torch.no_grad()
    def _step_decent(self) -> None:
        a, t, cfg = self.arena, self.arena.table, self.cfg
        for i in range(t.n_tensors):                               # per-tensor Issend/Recv/Wait (decent.cpp:172-243)
            flat = self._flat(a.theta, i)
            il, ir = self._flat(self.inbox_l, i), self._flat(self.inbox_r, i)
            self._send_recv_tensor(True, flat.clone(), il, ir)
            flat.add_(il).add_(ir).div_(3)
        self.bytes += 2 * t.n_elems * 4
        self._opt()

    def _step_cent(self) -> None:
        a, t = self.arena, self.arena.table
        if self.ring.world > 1:
            for i in range(t.n_tensors):                           # per-tensor MPI_Allreduce + divide (cent.cpp:130-142)
                g = self._flat(a.grad, i)
                dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group)
                g.div_(self.ring.world)
            self.bytes += t.n_elems * 4
        self._opt()

    # host-resident FSM state travels with the checkpoint too (plain floats: weights_only-safe)
    def state_dict(self):
        sd = super().state_dict()
        sd["h_fsm"] = {"thres": [float(v) for v in self.h_thres], "last_norm": [float(v) for v in self.h_last_norm],
                       "last_iter": [float(v) for v in self.h_last_iter],
                       "slopes": [[float(v) for v in row] for row in self.h_slopes]}
        return sd

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        h = sd.get("h_fsm")
        if h is not None:
            self.h_thres, self.h_last_norm = list(h["thres"]), list(h["last_norm"])
            self.h_last_iter, self.h_slopes = list(h["last_iter"]), [list(r) for r in h["slopes"]]
