"""Multi-process worker for random pairwise matchings (parallel/topology.py RandomMatch) on a real process group.

    torchrun --nproc-per-node R tests/random_match_worker.py --mode sim [--backend gloo|nccl|p2p] [--seed S]
        every rank's parameters, momentum and byte counter equal the single-process simulator's bit for bit after every
        one of --steps steps (decent, iter-sync; momentum, weight decay, Nesterov and a multistep lr schedule whose
        milestone falls in the run), and matched partners hold bitwise-equal theta before their SGD step
    torchrun --nproc-per-node R tests/random_match_worker.py --mode resume --ckpt-dir DIR
        a Trainer resumed from a checkpoint mid-run continues the same matching sequence and equals an uninterrupted
        run; resuming it under another --topology-seed or another topology raises
Used by tests/test_random_match_cpu.py (gloo) and tests/test_gpu_random_match.py (one process per GPU: nccl, p2p).
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
from eventgrad_b200.parallel import Graph, ParamArena, make_backend  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

STEPS_PER_EPOCH = 3
TOPOLOGY = "random-match"


def _gather(t, world):
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t)
    return [x.cpu() for x in out]


def run_sim(a, env):
    cfg = TrainConfig(algo="decent", dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, weight_decay=5e-4,
                      nesterov=True, lr_schedule="multistep", lr_milestones=(1,), lr_gamma=0.1,
                      lr_warmup_epochs=0.5, epochs=3, backend=a.backend, sync_mode="iter", topology=TOPOLOGY,
                      topology_seed=a.seed).validate()
    table = lr_table(cfg, STEPS_PER_EPOCH)
    torch.manual_seed(0)
    model = build_model(cfg.model)
    graph = Graph.build(env.rank, env.world, cfg.topology, seed=cfg.topology_seed)
    assert graph.kind == TOPOLOGY and graph.fanout == 1, graph
    if a.backend == "p2p":
        from eventgrad_b200.parallel.p2p import P2PBackend, preallocate_arena_buffers
        theta, grad, symm = preallocate_arena_buffers(model, cfg, env)
        arena = ParamArena(model, env.device, theta=theta, grad=grad)
        be = P2PBackend(cfg, arena, graph, env, symm=symm, timeout_ns=10_000_000_000)
    else:
        arena = ParamArena(model, env.device)
        be = make_backend(cfg, arena, graph, env)
    be.set_lr_table(table)
    t = arena.table
    theta0 = arena.theta.detach().cpu().clone()
    mask = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        mask[o:o + n] = 1

    def grad_of(step, rank):
        g = torch.Generator().manual_seed(step * 1000 + rank)
        return torch.randn(t.n_padded, generator=g) * 0.05 * mask

    W = env.world
    sim = RingSimulator(W, theta0, t, "decent", lr=cfg.lr, momentum=cfg.momentum, serial_skip=False,
                        weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table, offsets=TOPOLOGY,
                        topology_seed=a.seed)
    ok = True
    for s in range(a.steps):
        arena.grad.copy_(grad_of(s, env.rank).to(arena.grad.device))
        be.step()
        if hasattr(be, "synchronize"):
            be.synchronize()
        allth = _gather(arena.theta.detach().clone(), W)
        allmom = _gather(arena.mom.detach().clone(), W)
        cnt = torch.tensor([be.num_events(), be.bytes_sent()], dtype=torch.int64, device=arena.theta.device)
        allcnt = _gather(cnt, W)
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
            if int(allcnt[r][0]) != 0 or int(allcnt[r][1]) != sim.bytes[r]:
                ok = False
                print(f"step {s + 1} rank {r}: counters {allcnt[r].tolist()} vs bytes {sim.bytes[r]}")
    if hasattr(be, "check_status"):
        be.check_status()
    if env.rank == 0:
        print("WORKER_OK" if ok else "WORKER_FAIL", f"mode=sim backend={a.backend} seed={a.seed} world={W}",
              flush=True)
    be.close()
    return ok


def run_resume(a, env):
    from eventgrad_b200.data import synthetic_source
    from eventgrad_b200.engine.trainer import Trainer
    from eventgrad_b200.utils.ckpt import ckpt_path
    n_train = 32 * STEPS_PER_EPOCH * env.world

    def trainer(**kw):
        base = dict(algo="decent", device="cpu", backend="gloo", model="cnn2", train_samples=n_train,
                    test_samples=64, batch_size=32, epochs=3, quiet=True, momentum=0.9, weight_decay=5e-4,
                    nesterov=True, lr_schedule="multistep", lr_milestones=(2,), lr_gamma=0.1, topology=TOPOLOGY,
                    topology_seed=11)
        base.update(kw)
        torch.manual_seed(0)
        return Trainer(preset("mnist_event", **base), env,
                       train_source=synthetic_source("mnist", n_train),
                       test_source=synthetic_source("mnist", 64, train=False))

    full = trainer()
    full.fit()
    th_full = full.arena.theta.clone()
    by_full = full.backend.bytes_sent()
    part = trainer(ckpt_dir=a.ckpt_dir, ckpt_every=1, max_steps=STEPS_PER_EPOCH)      # stops after epoch 1
    part.fit()
    ok = part.epoch == 1 and part.backend.pass_num == STEPS_PER_EPOCH
    res = trainer(resume=ckpt_path(a.ckpt_dir, env.rank))
    ok = ok and res.backend.pass_num == STEPS_PER_EPOCH
    res.fit()
    ok = ok and torch.equal(res.arena.theta, th_full) and res.backend.bytes_sent() == by_full
    ok = ok and not torch.equal(part.arena.theta, th_full)
    for other in (dict(topology_seed=12), dict(topology="ring"), dict(topology="onepeer-exp")):
        try:
            trainer(resume=ckpt_path(a.ckpt_dir, env.rank), **other)
            ok = False
            print(f"rank {env.rank}: resuming a {TOPOLOGY} checkpoint under {other} did not raise")
        except ValueError as e:
            ok = ok and "topology" in str(e)
    flags = [None] * env.world
    dist.all_gather_object(flags, ok)
    if env.rank == 0:
        print("WORKER_OK" if all(flags) else "WORKER_FAIL", f"mode=resume world={env.world}", flush=True)
    return all(flags)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="sim", choices=["sim", "resume"])
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--ckpt-dir", default="")
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl", "p2p"])
    a = ap.parse_args()
    env = init_distributed("cpu" if a.backend == "gloo" else "cuda")
    ok = run_sim(a, env) if a.mode == "sim" else run_resume(a, env)
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
