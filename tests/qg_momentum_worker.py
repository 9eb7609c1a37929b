"""Multi-process worker for quasi-global momentum (--quasi-global-momentum) on a real process group.

    torchrun --nproc-per-node R tests/qg_momentum_worker.py --mode sim --algo A --topology T [--local-steps H]
             [--trigger norm|drift] [--backend gloo|nccl|p2p]
        every rank's parameters, momentum buffer (m_hat), event and byte counters equal the single-process simulator's
        bit for bit after every one of --steps steps (momentum, weight decay, Nesterov and a multistep + warm-up lr
        schedule whose milestone falls in the run)
    torchrun --nproc-per-node R tests/qg_momentum_worker.py --mode resume --ckpt-dir DIR
        a Trainer with --quasi-global-momentum resumed from a checkpoint in the middle of the run equals an
        uninterrupted run, and resuming it without the flag raises
Used by tests/test_qg_momentum_cpu.py (gloo) and tests/test_gpu_qg_momentum.py (nccl, p2p).
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
from eventgrad_b200.parallel.trigger import TriggerConfig  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

STEPS_PER_EPOCH = 3


def _gather(t, world):
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t)
    return [x.cpu() for x in out]


def run_sim(a, env):
    cfg = TrainConfig(algo=a.algo, dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, weight_decay=5e-4,
                      nesterov=True, lr_schedule="multistep", lr_milestones=(2,), lr_gamma=0.1,
                      lr_warmup_epochs=0.5, epochs=5, horizon=1.0, thres_type=1, initial_comm_passes=3,
                      topk_percent=10.0, backend=a.backend, sync_mode="iter", topology=a.topology,
                      trigger=a.trigger, local_steps=a.local_steps, quasi_global_momentum=True,
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
    assert be.qg
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
    sim = RingSimulator(W, theta0, t, cfg.algo, TriggerConfig.from_train(cfg), lr=cfg.lr, momentum=cfg.momentum,
                        topk_percent=cfg.topk_percent, serial_skip=False, weight_decay=cfg.weight_decay,
                        nesterov=cfg.nesterov, lr_table=table, offsets=cfg.topology, local_steps=cfg.local_steps,
                        quasi_global=True)
    ok = True
    dev = arena.theta.device
    for s in range(a.steps):
        arena.grad.copy_(grad_of(s, env.rank).to(arena.grad.device))
        be.step()
        be.synchronize()
        allth = _gather(arena.theta.detach().clone(), W)
        allmom = _gather(arena.mom.detach().clone(), W)
        allcnt = _gather(torch.tensor([be.num_events(), be.bytes_sent()], dtype=torch.int64, device=dev), W)
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
            if int(allcnt[r][0]) != sim.events[r] or int(allcnt[r][1]) != sim.bytes[r]:
                ok = False
                print(f"step {s + 1} rank {r}: counters {allcnt[r].tolist()} vs {sim.events[r]} {sim.bytes[r]}")
    if hasattr(be, "check_status"):
        be.check_status()
    if env.rank == 0:
        print("WORKER_OK" if ok else "WORKER_FAIL",
              f"mode=sim backend={a.backend} algo={cfg.algo} topology={cfg.topology} H={cfg.local_steps} "
              f"trigger={cfg.trigger} world={W}", flush=True)
    be.close()
    return ok


def run_resume(a, env):
    from eventgrad_b200.data import synthetic_source
    from eventgrad_b200.engine.trainer import Trainer
    from eventgrad_b200.utils.ckpt import ckpt_path
    spe = 4
    n_train = 32 * spe * env.world

    def trainer(**kw):
        base = dict(device="cpu", backend="gloo", model="cnn2", train_samples=n_train, test_samples=64,
                    batch_size=32, batch_mode="per_rank", sampler="random", epochs=2, quiet=True, momentum=0.9,
                    nesterov=True, weight_decay=5e-4, lr=0.05, quasi_global_momentum=True)
        base.update(kw)
        torch.manual_seed(0)
        return Trainer(preset("decent", **base), env,
                       train_source=synthetic_source("mnist", n_train),
                       test_source=synthetic_source("mnist", 64, train=False))

    full = trainer()
    assert full.backend.qg
    full.fit()
    th_full, mom_full = full.arena.theta.clone(), full.arena.mom.clone()
    part = trainer(ckpt_dir=a.ckpt_dir, ckpt_every=1, max_steps=spe)      # stops after epoch 1
    part.fit()
    ok = part.epoch == 1 and part.backend.pass_num == spe and not torch.equal(part.arena.theta, th_full)
    res = trainer(resume=ckpt_path(a.ckpt_dir, env.rank))
    ok = ok and res.backend.pass_num == spe
    res.fit()
    ok = ok and torch.equal(res.arena.theta, th_full) and torch.equal(res.arena.mom, mom_full)
    try:
        trainer(resume=ckpt_path(a.ckpt_dir, env.rank), quasi_global_momentum=False)
        ok = False
        print(f"rank {env.rank}: resuming a --quasi-global-momentum checkpoint without it did not raise")
    except ValueError as e:
        ok = ok and "quasi-global-momentum" in str(e)
    flags = [None] * env.world
    dist.all_gather_object(flags, ok)
    if env.rank == 0:
        print("WORKER_OK" if all(flags) else "WORKER_FAIL", f"mode=resume world={env.world}", flush=True)
    return all(flags)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="sim", choices=["sim", "resume"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--algo", default="decent", choices=["decent", "event", "spevent"])
    ap.add_argument("--topology", default="ring")
    ap.add_argument("--local-steps", type=int, default=1)
    ap.add_argument("--trigger", default="norm", choices=["norm", "drift"])
    ap.add_argument("--ckpt-dir", default="")
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl", "p2p"])
    a = ap.parse_args()
    env = init_distributed("cpu" if a.backend == "gloo" else "cuda")
    ok = run_sim(a, env) if a.mode == "sim" else run_resume(a, env)
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
