"""R virtual ranks of the p2p backend inside ONE process on ONE GPU.

Each virtual rank has its own window, arena, backend and CUDA stream; "peer-mapped" pointers
are simply the other virtual ranks' device pointers.  The complete cross-rank protocol of the
fused kernels (pushes, per-group release/acquire flags, acks, the all-reduce barriers) runs
unchanged -- the kernels of the R ranks are launched on R streams and spin on each other, so
the persistent grid per rank is capped to keep all R grids co-resident.  This is how the
`gpu`-marked tests validate multi-rank behaviour on the single-GPU test tier, and it is also a
handy deterministic debugging harness.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import List

import torch

from ..config import TrainConfig
from ..parallel.arena import ParamArena
from ..parallel.p2p import P2PBackend, preallocate_arena_buffers
from ..parallel.topology import Graph, Ring
from ..parallel.window import LocalBootstrap


class LocalWorld:
    def __init__(self, cfg: TrainConfig, world: int, model_fn, device="cuda:0", grid_cap: int = 8,
                 topology=None, table_mode: bool = False, **backend_kw):
        """`topology`: gossip graph name or offsets (default cfg.topology, parallel/topology.py).  `table_mode`: the
        step kernel reads per-tensor gradient tensors in place (P2PBackend.update_grad_table) instead of the grad
        arena; step() then hands each rank's flat gradient to the kernel as per-tensor views."""
        if topology is not None:
            if isinstance(topology, (tuple, list)):
                topology = ",".join(str(int(o)) for o in topology)
            cfg = cfg.replace(topology=str(topology)).validate()
        cfg = cfg.for_world(world)          # a name that resolves to {1} is the ring, with the ring's defaults
        topology = cfg.topology
        self.cfg, self.world = cfg, world
        self.table_mode = table_mode
        self.device = torch.device(device)
        self.boot = LocalBootstrap(world)
        self.models, self.arenas, self.backends, self.streams = [], [], [], []
        for r in range(world):
            env = SimpleNamespace(rank=r, world=world, local_rank=0, device=self.device, backend="local")
            torch.manual_seed(cfg.seed)
            model = model_fn()
            theta, grad, symm = preallocate_arena_buffers(model, cfg, env, bootstrap=self.boot.for_rank(r))
            arena = ParamArena(model, self.device, theta=theta, grad=grad)
            if table_mode:
                arena.enable_table_mode(shadow=False)
            g = Graph.build(r, world, topology, seed=cfg.topology_seed)
            be = P2PBackend(cfg, arena, Ring(r, world) if g.is_ring else g, env, symm=symm, grid_cap=grid_cap,
                            defer_connect=True, **backend_kw)
            self.models.append(model)
            self.arenas.append(arena)
            self.backends.append(be)
            self.streams.append(torch.cuda.Stream(self.device))
        torch.cuda.synchronize(self.device)
        for be in self.backends:
            be.connect()
        torch.cuda.synchronize(self.device)

    def step(self, grads: List[torch.Tensor]) -> None:
        """One synchronous training step with externally supplied flat gradients."""
        cur = torch.cuda.current_stream(self.device)
        for r in range(self.world):
            if self.table_mode:
                a = self.arenas[r]
                for i, c in enumerate(a.compute):
                    c.grad = a.flat(grads[r], i).reshape(c.shape).clone()
                self.backends[r].update_grad_table(a.compute)
            else:
                self.arenas[r].grad.copy_(grads[r])
        for st in self.streams:
            st.wait_stream(cur)
        for r in range(self.world):
            with torch.cuda.stream(self.streams[r]):
                self.backends[r].step()
        for st in self.streams:
            cur.wait_stream(st)

    def final_average(self) -> None:
        cur = torch.cuda.current_stream(self.device)
        for st in self.streams:
            st.wait_stream(cur)
        for r in range(self.world):
            with torch.cuda.stream(self.streams[r]):
                self.backends[r].final_average_nocheck()
        for st in self.streams:
            cur.wait_stream(st)
        torch.cuda.synchronize(self.device)
        for be in self.backends:
            be.check_status()

    def measure_consensus(self):
        """One ungated consensus measurement (--consensus-every) of every rank's current theta, all R launches in
        flight together; returns each rank's (D, A)."""
        cur = torch.cuda.current_stream(self.device)
        for st in self.streams:
            st.wait_stream(cur)
        for r in range(self.world):
            with torch.cuda.stream(self.streams[r]):
                self.backends[r].launch_consensus_now()
        for st in self.streams:
            cur.wait_stream(st)
        torch.cuda.synchronize(self.device)
        out = []
        for be in self.backends:
            be.check_status()
            if not be.cons:
                out.append(be.measure_consensus())          # R = 1: zeros, nothing launched
                continue
            rows = be.drain_consensus()
            be._cons_held = rows[:-1]
            out.append(rows[-1][1:])
        return out

    def close(self) -> None:
        torch.cuda.synchronize(self.device)
        for be in self.backends:
            be.close()
