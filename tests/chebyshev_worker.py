"""Multi-process worker for Chebyshev-accelerated gossip rounds (--gossip-accel chebyshev, decent) on a real process
group.

    torchrun --nproc-per-node R tests/chebyshev_worker.py --mode sim --gossip-rounds Q --topology T
             [--accel chebyshev|none] [--backend gloo|nccl|p2p]
        every rank's parameters, momentum and byte counter equal the single-process simulator's bit for bit after every
        one of --steps steps (momentum, weight decay, Nesterov and a multistep + warm-up lr schedule)
    torchrun --nproc-per-node R tests/chebyshev_worker.py --mode resume --gossip-rounds Q --resume-rounds Q2
             --accel A --resume-accel A2
        a backend checkpointed after --steps // 2 steps and restored into a fresh backend with Q2 rounds and accel A2
        equals the simulator that switches at that step, bit for bit (theta, momentum, bytes)
Used by tests/test_chebyshev_cpu.py (gloo) and tests/test_gpu_chebyshev.py (nccl, p2p).
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from eventgrad_b200.config import TrainConfig  # noqa: E402
from eventgrad_b200.engine.lr_schedule import lr_table  # noqa: E402
from eventgrad_b200.engine.simulator import RingSimulator  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.parallel import Graph, ParamArena, Ring, make_backend  # noqa: E402
from eventgrad_b200.parallel.topology import chebyshev_coefficients  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

STEPS_PER_EPOCH = 3


def _gather(t, world):
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t)
    return [x.cpu() for x in out]


def _cfg(a, env, Q, accel):
    return TrainConfig(algo="decent", dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, weight_decay=5e-4,
                       nesterov=True, lr_schedule="multistep", lr_milestones=(2,), lr_gamma=0.1,
                       lr_warmup_epochs=0.5, epochs=5, backend=a.backend, sync_mode="iter", topology=a.topology,
                       gossip_rounds=Q, gossip_accel=accel, overlap_push=False,
                       double_buffer=False).validate().for_world(env.world)


def _backend(a, env, cfg):
    torch.manual_seed(0)
    model = build_model(cfg.model)
    g = Graph.build(env.rank, env.world, cfg.topology)
    ring = Ring(env.rank, env.world) if g.is_ring else g
    if a.backend == "p2p":
        from eventgrad_b200.parallel.p2p import P2PBackend, preallocate_arena_buffers
        theta, grad, symm = preallocate_arena_buffers(model, cfg, env)
        arena = ParamArena(model, env.device, theta=theta, grad=grad)
        be = P2PBackend(cfg, arena, ring, env, symm=symm, timeout_ns=10_000_000_000)
    else:
        arena = ParamArena(model, env.device)
        be = make_backend(cfg, arena, ring, env)
    be.set_lr_table(lr_table(cfg, STEPS_PER_EPOCH))
    return arena, be


def run(a, env):
    Q = a.gossip_rounds
    cfg = _cfg(a, env, Q, a.accel)
    table = lr_table(cfg, STEPS_PER_EPOCH)
    arena, be = _backend(a, env, cfg)
    t = arena.table
    theta0 = arena.theta.detach().cpu().clone()
    mask = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        mask[o:o + n] = 1

    def grad_of(step, rank):
        gen = torch.Generator().manual_seed(step * 1000 + rank)
        return torch.randn(t.n_padded, generator=gen) * 0.05 * mask

    W = env.world
    sim = RingSimulator(W, theta0, t, "decent", lr=cfg.lr, momentum=cfg.momentum, serial_skip=False,
                        weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table, offsets=cfg.topology,
                        gossip_rounds=Q, gossip_accel=a.accel)
    switch = a.steps // 2 if a.mode == "resume" else -1
    ok = True
    dev = arena.theta.device
    for s in range(a.steps):
        if s == switch:
            # checkpoint, then a fresh backend with the other Q restored from it (and the arena's theta / momentum)
            sd = be.state_dict()
            th, mo = arena.theta.detach().clone(), arena.mom.detach().clone()
            be.close()
            arena, be = _backend(a, env, _cfg(a, env, a.resume_rounds, a.resume_accel))
            arena.theta.copy_(th)
            arena.mom.copy_(mo)
            be.load_state_dict(sd)
            sim.gossip_rounds = a.resume_rounds
            sim.cheb_coef = (chebyshev_coefficients(sim.offsets, W, a.resume_rounds)
                             if a.resume_accel == "chebyshev" else None)
        arena.grad.copy_(grad_of(s, env.rank).to(arena.grad.device))
        be.step()
        be.synchronize()
        allth = _gather(arena.theta.detach().clone(), W)
        allmom = _gather(arena.mom.detach().clone(), W)
        allcnt = _gather(torch.tensor([be.bytes_sent()], dtype=torch.int64, device=dev), W)
        sim.step([grad_of(s, r) for r in range(W)])
        if env.rank != 0:
            continue
        for r in range(W):
            if not torch.equal(allth[r], sim.theta[r]):
                ok = False
                print(f"step {s + 1} rank {r}: theta differs, max {(allth[r] - sim.theta[r]).abs().max().item():.3e}")
            if not torch.equal(allmom[r], sim.mom[r]):
                ok = False
                print(f"step {s + 1} rank {r}: momentum differs")
            if int(allcnt[r][0]) != sim.bytes[r]:
                ok = False
                print(f"step {s + 1} rank {r}: bytes {int(allcnt[r][0])} vs {sim.bytes[r]}")
    if hasattr(be, "check_status"):
        be.check_status()
    if env.rank == 0:
        if a.mode == "sim":
            ok = ok and all(b == a.steps * Q * sim.fanout * t.n_elems * 4 for b in sim.bytes)
        print("WORKER_OK" if ok else "WORKER_FAIL",
              f"mode={a.mode} backend={a.backend} topology={cfg.topology} Q={Q} accel={a.accel} world={W}", flush=True)
    be.close()
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="sim", choices=["sim", "resume"])
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--gossip-rounds", type=int, default=2)
    ap.add_argument("--resume-rounds", type=int, default=3)
    ap.add_argument("--accel", default="chebyshev", choices=["none", "chebyshev"])
    ap.add_argument("--resume-accel", default="none", choices=["none", "chebyshev"])
    ap.add_argument("--topology", default="ring")
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl", "p2p"])
    a = ap.parse_args()
    env = init_distributed("cpu" if a.backend == "gloo" else "cuda")
    ok = run(a, env)
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
