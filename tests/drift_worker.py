"""Multi-process worker for the drift trigger (--trigger drift: fire when ||theta - sent|| >= thres) on a real process
group.

    torchrun --nproc-per-node R tests/drift_worker.py --mode sim --algo event|spevent --topology ring|exp|onepeer-exp
        every rank's parameters, momentum, `sent` (spevent: prev), fire masks, event and byte counters equal the
        single-process simulator's bit for bit after every one of --steps steps (iter-sync; momentum, weight decay,
        Nesterov and a multistep lr schedule whose milestone falls in the run)
    torchrun --nproc-per-node R tests/drift_worker.py --mode resume --ckpt-dir DIR
        a drift Trainer resumed from a checkpoint equals an uninterrupted run, and resuming it under --trigger norm raises
Used by tests/test_drift_trigger_cpu.py (gloo).
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
                      lr_warmup_epochs=0.5, epochs=4, horizon=1.0, thres_type=1, initial_comm_passes=3,
                      backend=a.backend, sync_mode="iter", topology=a.topology, trigger="drift").validate()
    cfg = cfg.for_world(env.world)
    table = lr_table(cfg, STEPS_PER_EPOCH)
    torch.manual_seed(0)
    model = build_model(cfg.model)
    graph = Graph.build(env.rank, env.world, cfg.topology)
    ring = Ring(env.rank, env.world) if graph.is_ring else graph
    arena = ParamArena(model, env.device)
    be = make_backend(cfg, arena, ring, env)
    fire_of = be._fire
    decided = []

    def _fire():
        norms, fire = fire_of()
        decided.append(fire.clone().bool().cpu())
        return norms, fire
    be._fire = _fire
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
    sim = RingSimulator(W, theta0, t, a.algo, TriggerConfig.from_train(cfg), lr=cfg.lr, momentum=cfg.momentum,
                        serial_skip=False, weight_decay=cfg.weight_decay, nesterov=cfg.nesterov,
                        lr_table=table, offsets=a.topology)
    assert sim.drift
    ok, n_fired, n_held = True, 0, 0
    for s in range(a.steps):
        arena.grad.copy_(grad_of(s, env.rank).to(arena.grad.device))
        be.step()
        fire = decided[-1]
        be.synchronize()
        allth = _gather(arena.theta.detach().clone(), W)
        allmom = _gather(arena.mom.detach().clone(), W)
        allsent = _gather(be.sent.detach().clone(), W)
        cnt = torch.tensor([be.num_events(), be.bytes_sent()], dtype=torch.int64, device=arena.theta.device)
        allcnt = _gather(cnt, W)
        allfire = _gather(fire.to(torch.uint8).to(arena.theta.device), W)
        sim.step([grad_of(s, r) for r in range(W)])
        if env.rank != 0:
            continue
        for r in range(W):
            for name, got, want in (("theta", allth[r], sim.theta[r]), ("momentum", allmom[r], sim.mom[r]),
                                    ("sent", allsent[r], sim.sent[r])):
                if not torch.equal(got, want):
                    ok = False
                    print(f"step {s + 1} rank {r}: {name} differs, max {(got - want).abs().max().item():.3e}")
            if not torch.equal(allfire[r].bool(), sim.fire_history[-1][r]):
                ok = False
                print(f"step {s + 1} rank {r}: fire mask differs")
            n_fired += int(allfire[r].sum())
            n_held += int((~allfire[r].bool()).sum())
            if int(allcnt[r][0]) != sim.events[r] or int(allcnt[r][1]) != sim.bytes[r]:
                ok = False
                print(f"step {s + 1} rank {r}: counters {allcnt[r].tolist()} vs events {sim.events[r]} "
                      f"bytes {sim.bytes[r]}")
    if env.rank == 0:
        ok = ok and sum(sim.events) == sim.fanout * n_fired
        print("WORKER_OK" if ok else "WORKER_FAIL", f"mode=sim algo={a.algo} topology={a.topology} world={W} "
              f"fired={n_fired} held={n_held}", flush=True)
    be.close()
    return ok


def run_resume(a, env):
    from eventgrad_b200.data import synthetic_source
    from eventgrad_b200.engine.trainer import Trainer
    from eventgrad_b200.utils.ckpt import ckpt_path
    n_train = 32 * STEPS_PER_EPOCH * env.world

    def trainer(**kw):
        base = dict(device="cpu", backend="gloo", model="cnn2", train_samples=n_train, test_samples=64,
                    batch_size=32, epochs=3, quiet=True, momentum=0.9, initial_comm_passes=2, trigger="drift")
        base.update(kw)
        torch.manual_seed(0)
        return Trainer(preset("mnist_event", **base), env,
                       train_source=synthetic_source("mnist", n_train),
                       test_source=synthetic_source("mnist", 64, train=False))

    full = trainer()
    full.fit()
    th_full = full.arena.theta.clone()
    ev_full = full.backend.num_events()
    part = trainer(ckpt_dir=a.ckpt_dir, ckpt_every=1, max_steps=STEPS_PER_EPOCH)      # stops after epoch 1
    part.fit()
    ok = part.epoch == 1 and part.backend.pass_num == STEPS_PER_EPOCH
    res = trainer(resume=ckpt_path(a.ckpt_dir, env.rank))
    ok = ok and res.backend.pass_num == STEPS_PER_EPOCH
    ok = ok and torch.equal(res.backend.sent, part.backend.sent)
    res.fit()
    ok = ok and torch.equal(res.arena.theta, th_full) and res.backend.num_events() == ev_full
    ok = ok and not torch.equal(part.arena.theta, th_full)
    try:
        trainer(resume=ckpt_path(a.ckpt_dir, env.rank), trigger="norm")
        ok = False
        print(f"rank {env.rank}: resuming a drift checkpoint under --trigger norm did not raise")
    except ValueError as e:
        ok = ok and "trigger" in str(e)
    flags = [None] * env.world
    dist.all_gather_object(flags, ok)
    if env.rank == 0:
        print("WORKER_OK" if all(flags) else "WORKER_FAIL", f"mode=resume world={env.world}", flush=True)
    return all(flags)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="sim", choices=["sim", "resume"])
    ap.add_argument("--algo", default="event", choices=["event", "spevent"])
    ap.add_argument("--topology", default="ring")
    ap.add_argument("--steps", type=int, default=9)
    ap.add_argument("--ckpt-dir", default="")
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl"])
    a = ap.parse_args()
    env = init_distributed("cpu" if a.backend == "gloo" else "cuda")
    ok = run_sim(a, env) if a.mode == "sim" else run_resume(a, env)
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
