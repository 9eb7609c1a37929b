"""Multi-process worker for the one-peer exponential graph (parallel/topology.py OnePeerExp) on a real process group.

    torchrun --nproc-per-node R tests/onepeer_worker.py --mode sim --algo decent|event [--backend gloo|nccl|p2p]
        every rank's parameters, momentum, fire masks, event and byte counters equal the single-process simulator's
        bit for bit after every one of --steps steps (iter-sync; momentum, weight decay, Nesterov and a multistep lr
        schedule whose milestone falls in the run; p2p: the simulator takes the kernel's own trigger decisions)
    torchrun --nproc-per-node R tests/onepeer_worker.py --mode resume --ckpt-dir DIR
        a Trainer resumed from a checkpoint taken at a step that is not a multiple of the period equals an
        uninterrupted run, and resuming it under the ring or the static exp graph raises
Used by tests/test_onepeer_cpu.py (gloo) and tests/test_gpu_onepeer.py (one process per GPU: nccl, p2p).
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
from eventgrad_b200.parallel.trigger import TriggerConfig  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

STEPS_PER_EPOCH = 3
TOPOLOGY = "onepeer-exp"


def _gather(t, world):
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t)
    return [x.cpu() for x in out]


def run_sim(a, env):
    cfg = TrainConfig(algo=a.algo, dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, weight_decay=5e-4,
                      nesterov=True, lr_schedule="multistep", lr_milestones=(1,), lr_gamma=0.1,
                      lr_warmup_epochs=0.5, epochs=3, horizon=1.0, thres_type=1, initial_comm_passes=3,
                      backend=a.backend, sync_mode="iter", topology=TOPOLOGY).validate()
    table = lr_table(cfg, STEPS_PER_EPOCH)
    torch.manual_seed(0)
    model = build_model(cfg.model)
    graph = Graph.build(env.rank, env.world, cfg.topology)
    assert graph.period >= 1 and graph.fanout == 1, graph
    if a.backend == "p2p":
        from eventgrad_b200.parallel.p2p import P2PBackend, preallocate_arena_buffers
        theta, grad, symm = preallocate_arena_buffers(model, cfg, env)
        arena = ParamArena(model, env.device, theta=theta, grad=grad)
        be = P2PBackend(cfg, arena, graph, env, symm=symm, timeout_ns=10_000_000_000)
    else:
        arena = ParamArena(model, env.device)
        be = make_backend(cfg, arena, graph, env)
        if a.algo == "event":          # record the host trigger's decision of every step
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
                        lr_table=table, offsets=TOPOLOGY)
    ok = True
    for s in range(a.steps):
        fire = None
        if a.backend == "p2p" and a.algo == "event":
            fire = be.fire.clone().bool().cpu()          # the kernel's decision for this step
        arena.grad.copy_(grad_of(s, env.rank).to(arena.grad.device))
        be.step()
        if a.backend != "p2p" and a.algo == "event":
            fire = decided[-1]
        if hasattr(be, "synchronize"):
            be.synchronize()
        allth = _gather(arena.theta.detach().clone(), W)
        allmom = _gather(arena.mom.detach().clone(), W)
        cnt = torch.tensor([be.num_events(), be.bytes_sent()], dtype=torch.int64, device=arena.theta.device)
        allcnt = _gather(cnt, W)
        allfire = _gather(fire.to(torch.uint8).to(arena.theta.device), W) if fire is not None else None
        if a.backend == "p2p" and allfire is not None:
            sim.step([grad_of(s, r) for r in range(W)], fires=[allfire[r].bool() for r in range(W)])
        else:
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
            if allfire is not None and not torch.equal(allfire[r].bool(), sim.fire_history[-1][r]):
                ok = False
                print(f"step {s + 1} rank {r}: fire mask differs")
            want_ev = sim.events[r] if a.algo == "event" else 0
            if int(allcnt[r][0]) != want_ev or int(allcnt[r][1]) != sim.bytes[r]:
                ok = False
                print(f"step {s + 1} rank {r}: counters {allcnt[r].tolist()} vs events {want_ev} bytes {sim.bytes[r]}")
    if hasattr(be, "check_status"):
        be.check_status()
    if env.rank == 0:
        if a.algo == "event":
            fired = sum(int(f.sum()) for fr in sim.fire_history for f in fr)
            ok = ok and sum(sim.events) == fired
            if fired == t.n_tensors * a.steps * W:
                print("note: every tensor fired at every step")
        print("WORKER_OK" if ok else "WORKER_FAIL",
              f"mode=sim algo={a.algo} backend={a.backend} period={graph.period} world={W}", flush=True)
    be.close()
    return ok


def run_resume(a, env):
    from eventgrad_b200.data import synthetic_source
    from eventgrad_b200.engine.trainer import Trainer
    from eventgrad_b200.utils.ckpt import ckpt_path
    n_train = 32 * STEPS_PER_EPOCH * env.world

    def trainer(**kw):
        base = dict(device="cpu", backend="gloo", model="cnn2", train_samples=n_train, test_samples=64,
                    batch_size=32, epochs=3, quiet=True, momentum=0.9, weight_decay=5e-4, nesterov=True,
                    lr_schedule="multistep", lr_milestones=(2,), lr_gamma=0.1, topology=TOPOLOGY)
        base.update(kw)
        torch.manual_seed(0)
        return Trainer(preset("mnist_event", **base), env,
                       train_source=synthetic_source("mnist", n_train),
                       test_source=synthetic_source("mnist", 64, train=False))

    full = trainer()
    full.fit()
    th_full = full.arena.theta.clone()
    ev_full = full.backend.num_events()
    period = full.ring.period
    part = trainer(ckpt_dir=a.ckpt_dir, ckpt_every=1, max_steps=STEPS_PER_EPOCH)      # stops after epoch 1
    part.fit()
    ok = part.epoch == 1 and part.backend.pass_num == STEPS_PER_EPOCH and STEPS_PER_EPOCH % period != 0
    res = trainer(resume=ckpt_path(a.ckpt_dir, env.rank))
    ok = ok and res.backend.pass_num == STEPS_PER_EPOCH
    res.fit()
    ok = ok and torch.equal(res.arena.theta, th_full) and res.backend.num_events() == ev_full
    ok = ok and not torch.equal(part.arena.theta, th_full)
    for other in ("ring", "exp"):
        try:
            trainer(resume=ckpt_path(a.ckpt_dir, env.rank), topology=other)
            ok = False
            print(f"rank {env.rank}: resuming a {TOPOLOGY} checkpoint under {other} did not raise")
        except ValueError as e:
            ok = ok and "topology" in str(e)
    flags = [None] * env.world
    dist.all_gather_object(flags, ok)
    if env.rank == 0:
        print("WORKER_OK" if all(flags) else "WORKER_FAIL", f"mode=resume period={period} world={env.world}",
              flush=True)
    return all(flags)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="sim", choices=["sim", "resume"])
    ap.add_argument("--algo", default="event")
    ap.add_argument("--steps", type=int, default=0, help="default: 2 * period + 1")
    ap.add_argument("--ckpt-dir", default="")
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl", "p2p"])
    a = ap.parse_args()
    env = init_distributed("cpu" if a.backend == "gloo" else "cuda")
    if a.steps <= 0:
        a.steps = 2 * Graph.build(env.rank, env.world, TOPOLOGY).period + 1
    ok = run_sim(a, env) if a.mode == "sim" else run_resume(a, env)
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
