"""Multi-process worker for exact diffusion (--exact-diffusion, decent on the ring) on a real process group.

    torchrun --nproc-per-node R tests/exact_diffusion_worker.py --mode sim --backend gloo|nccl|p2p
        every rank's parameters, momentum, psi and byte counter equal the single-process simulator's bit for bit
        after every one of --steps steps (momentum, weight decay, Nesterov and a multistep + warm-up lr schedule whose
        milestone falls in the run); the gradients differ per rank and have a rank-dependent mean, as on skewed shards
    torchrun --nproc-per-node R tests/exact_diffusion_worker.py --mode resume --ckpt-dir DIR
        an exact-diffusion Trainer on label-sorted shards resumed from a checkpoint equals an uninterrupted run, and
        resuming it without exact diffusion raises
Used by tests/test_exact_diffusion_cpu.py (gloo) and tests/test_gpu_exact_diffusion.py (nccl, p2p).
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
from eventgrad_b200.parallel import ParamArena, Ring, make_backend  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

STEPS_PER_EPOCH = 3


def _gather(t, world):
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t)
    return [x.cpu() for x in out]


def run_sim(a, env):
    cfg = TrainConfig(algo="decent", dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, weight_decay=5e-4,
                      nesterov=True, lr_schedule="multistep", lr_milestones=(2,), lr_gamma=0.1,
                      lr_warmup_epochs=0.5, epochs=4, backend=a.backend, sync_mode="iter", exact_diffusion=True,
                      overlap_push=False).validate()
    table = lr_table(cfg, STEPS_PER_EPOCH)
    torch.manual_seed(0)
    model = build_model(cfg.model)
    ring = Ring(env.rank, env.world)
    if a.backend == "p2p":
        from eventgrad_b200.parallel.p2p import P2PBackend, preallocate_arena_buffers
        theta, grad, symm = preallocate_arena_buffers(model, cfg, env)
        arena = ParamArena(model, env.device, theta=theta, grad=grad)
        be = P2PBackend(cfg, arena, ring, env, symm=symm, timeout_ns=10_000_000_000)
    else:
        arena = ParamArena(model, env.device)
        be = make_backend(cfg, arena, ring, env)
    assert be.ed
    be.set_lr_table(table)
    t = arena.table
    theta0 = arena.theta.detach().cpu().clone()
    mask = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        mask[o:o + n] = 1

    def grad_of(step, rank):
        g = torch.Generator().manual_seed(step * 1000 + rank)
        return (torch.randn(t.n_padded, generator=g) * 0.05 + 0.01 * (rank - 1)) * mask

    W = env.world
    sim = RingSimulator(W, theta0, t, "decent", lr=cfg.lr, momentum=cfg.momentum, serial_skip=False,
                        weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table, exact_diffusion=True)
    ok = True
    dev = arena.theta.device
    for s in range(a.steps):
        arena.grad.copy_(grad_of(s, env.rank).to(arena.grad.device))
        be.step()
        be.synchronize()
        got = {name: _gather(buf.detach().clone(), W) for name, buf in
               (("theta", arena.theta), ("momentum", arena.mom), ("psi", be.psi))}
        allcnt = _gather(torch.tensor([be.bytes_sent()], dtype=torch.int64, device=dev), W)
        sim.step([grad_of(s, r) for r in range(W)])
        if env.rank != 0:
            continue
        for r in range(W):
            want = {"theta": sim.theta[r], "momentum": sim.mom[r], "psi": sim.psi[r]}
            for name, bufs in got.items():
                if not torch.equal(bufs[r], want[name]):
                    ok = False
                    print(f"step {s + 1} rank {r}: {name} differs, max {(bufs[r] - want[name]).abs().max().item():.3e}")
            if int(allcnt[r][0]) != sim.bytes[r]:
                ok = False
                print(f"step {s + 1} rank {r}: bytes {int(allcnt[r][0])} vs {sim.bytes[r]}")
    if hasattr(be, "check_status"):
        be.check_status()
    if env.rank == 0:
        print("WORKER_OK" if ok else "WORKER_FAIL", f"mode=sim backend={a.backend} world={W}", flush=True)
    be.close()
    return ok


def run_resume(a, env):
    from eventgrad_b200.data import synthetic_source
    from eventgrad_b200.engine.trainer import Trainer
    from eventgrad_b200.utils.ckpt import ckpt_path
    spe = 5                                            # steps per epoch: the checkpoint is taken at step 5
    n_train = 32 * spe * env.world

    def trainer(**kw):
        base = dict(device="cpu", backend="gloo", model="cnn2", train_samples=n_train, test_samples=64,
                    batch_size=32, batch_mode="per_rank", sampler="random", epochs=2, quiet=True, momentum=0.9,
                    lr=0.05, exact_diffusion=True, partition="label")
        base.update(kw)
        torch.manual_seed(0)
        return Trainer(preset("decent", **base), env,
                       train_source=synthetic_source("mnist", n_train),
                       test_source=synthetic_source("mnist", 64, train=False))

    full = trainer()
    assert full.backend.ed
    full.fit()
    th_full = full.arena.theta.clone()
    by_full = full.backend.bytes_sent()
    part = trainer(ckpt_dir=a.ckpt_dir, ckpt_every=1, max_steps=spe)      # stops after epoch 1
    part.fit()
    ok = part.epoch == 1 and part.backend.pass_num == spe and not torch.equal(part.arena.theta, th_full)
    res = trainer(resume=ckpt_path(a.ckpt_dir, env.rank))
    ok = ok and res.backend.pass_num == spe
    res.fit()
    ok = ok and torch.equal(res.arena.theta, th_full) and res.backend.bytes_sent() == by_full
    for k in ("psi", "inbox_l", "inbox_r"):
        ok = ok and torch.equal(getattr(res.backend, k), getattr(full.backend, k))
    try:
        trainer(resume=ckpt_path(a.ckpt_dir, env.rank), exact_diffusion=False)
        ok = False
        print(f"rank {env.rank}: resuming an exact-diffusion checkpoint without it did not raise")
    except ValueError as e:
        ok = ok and "exact-diffusion" in str(e)
    flags = [None] * env.world
    dist.all_gather_object(flags, ok)
    if env.rank == 0:
        print("WORKER_OK" if all(flags) else "WORKER_FAIL", f"mode=resume world={env.world}", flush=True)
    return all(flags)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="sim", choices=["sim", "resume"])
    ap.add_argument("--steps", type=int, default=9)
    ap.add_argument("--ckpt-dir", default="")
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl", "p2p"])
    a = ap.parse_args()
    env = init_distributed("cpu" if a.backend == "gloo" else "cuda")
    ok = run_sim(a, env) if a.mode == "sim" else run_resume(a, env)
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
