"""Multi-process worker for the sign codec (--compress sign) and the CHOCO mix (--choco-gamma) on a real process group.

    torchrun --nproc-per-node R tests/choco_worker.py --mode sim --backend gloo|nccl|p2p --algo decent|event
             [--trigger norm|drift] [--compress int8|sign] [--gamma G]
        every rank's parameters, momentum, prev, rep_l, rep_r, event and byte counters equal the single-process
        simulator's bit for bit after every one of --steps steps (ring, iter-sync; momentum, weight decay, Nesterov and
        a multistep + warm-up lr schedule whose milestone falls in the run).  gloo: the simulator takes its own trigger
        decisions and they must equal the backend's; nccl / p2p: the simulator follows the backend's decisions (their
        norms are reduced on the GPU)
    torchrun --nproc-per-node R tests/choco_worker.py --mode resume --ckpt-dir DIR [--compress C] [--gamma G]
        a Trainer resumed from a checkpoint equals an uninterrupted run, and resuming it under another --choco-gamma or
        another --compress raises
Used by tests/test_choco_cpu.py (gloo) and tests/test_gpu_choco.py (nccl, p2p).
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
                      backend=a.backend, sync_mode="iter", trigger=a.trigger, compress=a.compress,
                      choco_gamma=a.gamma,
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
        assert be.q8
    else:
        arena = ParamArena(model, env.device)
        be = make_backend(cfg, arena, ring, env)
        assert be.q8
    decided = []
    if a.backend != "p2p":
        fire_of = be._fire

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
                        lr_table=table, compress=a.compress, choco_gamma=a.gamma)
    follow = a.backend != "gloo" and a.algo == "event"
    ok, n_fired, n_held = True, 0, 0
    dev = arena.theta.device
    for s in range(a.steps):
        if a.backend == "p2p":
            fire = be.fire.clone().bool().cpu()
        arena.grad.copy_(grad_of(s, env.rank).to(arena.grad.device))
        be.step()
        if a.backend != "p2p":
            fire = decided[-1] if decided else torch.ones(t.n_tensors, dtype=torch.bool)
        be.synchronize()
        got = {name: _gather(buf.detach().clone(), W) for name, buf in
               (("theta", arena.theta), ("momentum", arena.mom), ("prev", be.prev), ("rep_l", be.rep_l),
                ("rep_r", be.rep_r))}
        cnt = torch.tensor([be.num_events(), be.bytes_sent()], dtype=torch.int64, device=dev)
        allcnt = _gather(cnt, W)
        allfire = _gather(fire.to(torch.uint8).to(dev), W)
        sim.step([grad_of(s, r) for r in range(W)], fires=[f.bool() for f in allfire] if follow else None)
        if env.rank != 0:
            continue
        for r in range(W):
            want = {"theta": sim.theta[r], "momentum": sim.mom[r], "prev": sim.prev[r], "rep_l": sim.rep_l[r],
                    "rep_r": sim.rep_r[r]}
            for name, bufs in got.items():
                if not torch.equal(bufs[r], want[name]):
                    ok = False
                    print(f"step {s + 1} rank {r}: {name} differs, max {(bufs[r] - want[name]).abs().max().item():.3e}")
            if a.algo == "event" and not torch.equal(allfire[r].bool(), sim.fire_history[-1][r]):
                ok = False
                print(f"step {s + 1} rank {r}: fire mask differs")
            n_fired += int(allfire[r].sum())
            n_held += int((~allfire[r].bool()).sum())
            if int(allcnt[r][0]) != sim.events[r] or int(allcnt[r][1]) != sim.bytes[r]:
                ok = False
                print(f"step {s + 1} rank {r}: counters {allcnt[r].tolist()} vs events {sim.events[r]} "
                      f"bytes {sim.bytes[r]}")
        # the replica invariant: my left neighbour's rep_r and my right neighbour's rep_l are my prev
        for r in range(W):
            L, R = (r - 1) % W, (r + 1) % W
            if not (torch.equal(got["rep_r"][L], got["prev"][r]) and torch.equal(got["rep_l"][R], got["prev"][r])):
                ok = False
                print(f"step {s + 1} rank {r}: replica invariant broken")
    if hasattr(be, "check_status"):
        be.check_status()
    if env.rank == 0:
        if a.algo == "event":
            ok = ok and sum(sim.events) == 2 * n_fired
        print("WORKER_OK" if ok else "WORKER_FAIL", f"mode=sim backend={a.backend} algo={a.algo} "
              f"trigger={a.trigger} compress={a.compress} gamma={a.gamma} world={W} fired={n_fired} held={n_held}", flush=True)
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
                    batch_size=32, epochs=2, quiet=True, momentum=0.9, initial_comm_passes=2, compress=a.compress,
                    choco_gamma=a.gamma)
        base.update(kw)
        torch.manual_seed(0)
        return Trainer(preset("mnist_event", **base), env,
                       train_source=synthetic_source("mnist", n_train),
                       test_source=synthetic_source("mnist", 64, train=False))

    full = trainer()
    full.fit()
    th_full = full.arena.theta.clone()
    ev_full, by_full = full.backend.num_events(), full.backend.bytes_sent()
    part = trainer(ckpt_dir=a.ckpt_dir, ckpt_every=1, max_steps=spe)      # stops after epoch 1
    part.fit()
    ok = part.epoch == 1 and part.backend.pass_num == spe and not torch.equal(part.arena.theta, th_full)
    res = trainer(resume=ckpt_path(a.ckpt_dir, env.rank))
    ok = ok and res.backend.pass_num == spe
    res.fit()
    ok = ok and torch.equal(res.arena.theta, th_full) and res.backend.num_events() == ev_full
    ok = ok and res.backend.bytes_sent() == by_full and torch.equal(res.backend.prev, full.backend.prev)
    ok = ok and torch.equal(res.backend.rep_l, full.backend.rep_l) and torch.equal(res.backend.rep_r, full.backend.rep_r)
    other = "int8" if a.compress == "sign" else "sign"
    for kw, key in (({"choco_gamma": 0.25 if a.gamma != 0.25 else 0.5}, "choco-gamma"),
                    ({"compress": other}, "compress")):
        try:
            trainer(resume=ckpt_path(a.ckpt_dir, env.rank), **kw)
            ok = False
            print(f"rank {env.rank}: resuming with {kw} did not raise")
        except ValueError as e:
            ok = ok and key in str(e)
    flags = [None] * env.world
    dist.all_gather_object(flags, ok)
    if env.rank == 0:
        print("WORKER_OK" if all(flags) else "WORKER_FAIL", f"mode=resume world={env.world}", flush=True)
    return all(flags)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="sim", choices=["sim", "resume"])
    ap.add_argument("--algo", default="event", choices=["decent", "event"])
    ap.add_argument("--trigger", default="norm", choices=["norm", "drift"])
    ap.add_argument("--steps", type=int, default=9)
    ap.add_argument("--compress", default="sign", choices=["int8", "sign"])
    ap.add_argument("--gamma", type=float, default=0.5)
    ap.add_argument("--ckpt-dir", default="")
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl", "p2p"])
    a = ap.parse_args()
    env = init_distributed("cpu" if a.backend == "gloo" else "cuda")
    ok = run_sim(a, env) if a.mode == "sim" else run_resume(a, env)
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
