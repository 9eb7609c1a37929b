"""Multi-process worker for SlowMo (--slowmo-period tau, decent) on a real process group.

    torchrun --nproc-per-node R tests/slowmo_worker.py --mode sim --slowmo-period tau --local-steps H --topology T
             [--backend gloo|nccl|p2p] [--slowmo-beta B] [--slowmo-lr A]
        every rank's parameters, momentum, outer iterate x, slow momentum u and byte counter equal the single-process
        simulator's bit for bit after every one of --steps steps (momentum, weight decay, Nesterov and a multistep +
        warm-up lr schedule whose milestone falls in the run), and x and u are identical on every rank
    torchrun --nproc-per-node R tests/slowmo_worker.py --mode resume --ckpt-dir DIR --slowmo-period tau --local-steps H
        a Trainer resumed from a checkpoint taken at step 5 equals an uninterrupted run, and resuming it under another
        --slowmo-period, --slowmo-beta or --slowmo-lr raises
Used by tests/test_slowmo_cpu.py (gloo) and tests/test_gpu_slowmo.py (nccl, p2p).
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from eventgrad_b200.config import TrainConfig, preset  # noqa: E402
from eventgrad_b200.engine.lr_schedule import lr_table  # noqa: E402
from eventgrad_b200.engine.simulator import RingSimulator  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.parallel import Graph, ParamArena, Ring, make_backend  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

STEPS_PER_EPOCH = 3


def _gather(t, world):
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t)
    return [x.cpu() for x in out]


def run_sim(a, env):
    tau, H = a.slowmo_period, a.local_steps
    cfg = TrainConfig(algo="decent", dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, weight_decay=5e-4,
                      nesterov=True, lr_schedule="multistep", lr_milestones=(2,), lr_gamma=0.1,
                      lr_warmup_epochs=0.5, epochs=5, backend=a.backend, sync_mode="iter", topology=a.topology,
                      local_steps=H, slowmo_period=tau, slowmo_beta=a.slowmo_beta, slowmo_lr=a.slowmo_lr,
                      overlap_push=False).validate().for_world(env.world)
    table = lr_table(cfg, STEPS_PER_EPOCH)
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
    assert be.slowmo_period == tau
    be.set_lr_table(table)
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
                        local_steps=H, slowmo_period=tau, slowmo_beta=a.slowmo_beta, slowmo_lr=a.slowmo_lr)
    ok = True
    dev = arena.theta.device
    for s in range(a.steps):
        arena.grad.copy_(grad_of(s, env.rank).to(arena.grad.device))
        be.step()
        be.synchronize()
        got = {"theta": _gather(arena.theta.detach().clone(), W), "momentum": _gather(arena.mom.detach().clone(), W),
               "x": _gather(be.slowmo_x.clone(), W), "u": _gather(be.slowmo_u.clone(), W)}
        allcnt = _gather(torch.tensor([be.bytes_sent()], dtype=torch.int64, device=dev), W)
        sim.step([grad_of(s, r) for r in range(W)])
        if env.rank != 0:
            continue
        want = {"theta": sim.theta, "momentum": sim.mom, "x": sim.slowmo_x, "u": sim.slowmo_u}
        for r in range(W):
            for k in got:
                if not torch.equal(got[k][r], want[k][r]):
                    ok = False
                    print(f"step {s + 1} rank {r}: {k} differs, max {(got[k][r] - want[k][r]).abs().max().item():.3e}")
            if int(allcnt[r][0]) != sim.bytes[r]:
                ok = False
                print(f"step {s + 1} rank {r}: bytes {int(allcnt[r][0])} vs {sim.bytes[r]}")
        if not all(torch.equal(got[k][0], got[k][r]) for k in ("x", "u") for r in range(W)):
            ok = False
            print(f"step {s + 1}: x or u differs across ranks")
    if hasattr(be, "check_status"):
        be.check_status()
    if env.rank == 0:
        syncs = a.steps // tau
        per = 0 if H == tau else sim.fanout
        ok = ok and all(b == (syncs + (a.steps - syncs) * per) * t.n_elems * 4 for b in sim.bytes)
        print("WORKER_OK" if ok else "WORKER_FAIL", f"mode=sim backend={a.backend} topology={cfg.topology} tau={tau} "
              f"H={H} world={W}", flush=True)
    be.close()
    return ok


def run_resume(a, env):
    from eventgrad_b200.data import synthetic_source
    from eventgrad_b200.engine.trainer import Trainer
    from eventgrad_b200.utils.ckpt import ckpt_path
    spe, tau, H = 5, a.slowmo_period, a.local_steps      # checkpoint at step 5
    n_train = 32 * spe * env.world

    def trainer(**kw):
        base = dict(device="cpu", backend="gloo", model="cnn2", train_samples=n_train, test_samples=64,
                    batch_size=32, batch_mode="per_rank", sampler="random", epochs=2, quiet=True, momentum=0.9,
                    nesterov=True, weight_decay=5e-4, lr=0.05, slowmo_period=tau, local_steps=H, slowmo_beta=0.7)
        base.update(kw)
        torch.manual_seed(0)
        return Trainer(preset("decent", **base), env,
                       train_source=synthetic_source("mnist", n_train),
                       test_source=synthetic_source("mnist", 64, train=False))

    full = trainer()
    assert full.backend.slowmo_period == tau
    full.fit()
    th_full = full.arena.theta.clone()
    x_full, u_full = full.backend.slowmo_x.clone(), full.backend.slowmo_u.clone()
    by_full = full.backend.bytes_sent()
    K = 2 * spe
    per = 0 if H == tau else 2
    ok = by_full == ((K // tau) + (K - K // tau) * per) * full.arena.table.n_elems * 4
    part = trainer(ckpt_dir=a.ckpt_dir, ckpt_every=1, max_steps=spe)      # stops after epoch 1
    part.fit()
    ok = ok and part.epoch == 1 and part.backend.pass_num == spe
    ok = ok and not torch.equal(part.arena.theta, th_full)
    res = trainer(resume=ckpt_path(a.ckpt_dir, env.rank))
    ok = ok and res.backend.pass_num == spe
    res.fit()
    ok = ok and torch.equal(res.arena.theta, th_full) and res.backend.bytes_sent() == by_full
    ok = ok and torch.equal(res.backend.slowmo_x, x_full) and torch.equal(res.backend.slowmo_u, u_full)
    for other in (dict(slowmo_period=tau + 1, local_steps=1), dict(slowmo_period=0, local_steps=1),
                  dict(slowmo_beta=0.5), dict(slowmo_lr=0.5)):
        try:
            trainer(resume=ckpt_path(a.ckpt_dir, env.rank), **other)
            ok = False
            print(f"rank {env.rank}: resuming a --slowmo-period {tau} checkpoint under {other} did not raise")
        except ValueError as e:
            ok = ok and ("slowmo" in str(e) or "local-steps" in str(e))
    flags = [None] * env.world
    dist.all_gather_object(flags, ok)
    if env.rank == 0:
        print("WORKER_OK" if all(flags) else "WORKER_FAIL", f"mode=resume world={env.world} tau={tau} H={H}",
              flush=True)
    return all(flags)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="sim", choices=["sim", "resume"])
    ap.add_argument("--steps", type=int, default=13)
    ap.add_argument("--slowmo-period", type=int, default=2)
    ap.add_argument("--slowmo-beta", type=float, default=0.5)
    ap.add_argument("--slowmo-lr", type=float, default=1.0)
    ap.add_argument("--local-steps", type=int, default=1)
    ap.add_argument("--topology", default="ring")
    ap.add_argument("--ckpt-dir", default="")
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl", "p2p"])
    a = ap.parse_args()
    env = init_distributed("cpu" if a.backend == "gloo" else "cuda")
    ok = run_sim(a, env) if a.mode == "sim" else run_resume(a, env)
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
