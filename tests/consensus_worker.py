"""Multi-process worker for the consensus distance (--consensus-every N) on a real process group.

    torchrun --nproc-per-node R tests/consensus_worker.py --mode sim --algo A --topology T --feature F --every N
             [--backend gloo|nccl|p2p]
        every rank's parameters and byte counter equal the single-process simulator's bit for bit after every step,
        and the backend's measurements (step, D, A) equal the simulator's: exactly on gloo / nccl, to rtol 1e-5 on p2p
        (the kernel's fp64 sums run in another order), identically on every rank
    torchrun --nproc-per-node R tests/consensus_worker.py --mode trainer --log-dir DIR --ckpt-dir DIR
        a Trainer run writes consensus.csv / consensus_tensors.csv with one row per measurement (per tensor), reports
        consensus_last and consensus_before_final_average, prints the per-epoch line, and a resumed run continues the
        measurement cycle from the restored step counter with the same values as an uninterrupted run
Used by tests/test_consensus_cpu.py (gloo) and tests/test_gpu_consensus.py (nccl, p2p).
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from eventgrad_b200.config import TrainConfig, preset  # noqa: E402
from eventgrad_b200.engine.simulator import RingSimulator  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.parallel import Graph, ParamArena, Ring, make_backend  # noqa: E402
from eventgrad_b200.parallel.trigger import TriggerConfig  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

# TrainConfig fields of each gossip feature, and the simulator's names for them
FEATURES = {
    "plain": {},
    "int8": dict(compress="int8"),
    "gt": dict(gradient_tracking=True),
    "ed": dict(exact_diffusion=True),
    "local": dict(local_steps=2),
    "pga": dict(global_avg_period=3),
    "qg": dict(quasi_global_momentum=True),
    "slowmo": dict(slowmo_period=3),
}
SIM_NAME = {"quasi_global_momentum": "quasi_global"}


def _gather(t, world):
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t)
    return [x.cpu() for x in out]


def run_sim(a, env):
    feat = FEATURES[a.feature]
    cfg = TrainConfig(algo=a.algo, dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, epochs=5,
                      backend=a.backend, sync_mode="iter", topology=a.topology, overlap_push=False,
                      consensus_every=a.every, **feat).validate().for_world(env.world)
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
    t = arena.table
    theta0 = arena.theta.detach().cpu().clone()
    mask = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        mask[o:o + n] = 1

    def grad_of(step, rank):
        gen = torch.Generator().manual_seed(step * 1000 + rank)
        return torch.randn(t.n_padded, generator=gen) * 0.05 * mask

    W = env.world
    sim = RingSimulator(W, theta0, t, a.algo, tcfg=TriggerConfig.from_train(cfg), lr=cfg.lr, momentum=cfg.momentum,
                        serial_skip=False, offsets=cfg.topology, consensus_every=a.every,
                        **{SIM_NAME.get(k, k): v for k, v in feat.items()})
    exact = a.backend != "p2p"
    ok = True
    dev = arena.theta.device
    rows = []
    for s in range(a.steps):
        arena.grad.copy_(grad_of(s, env.rank).to(arena.grad.device))
        be.step()
        be.synchronize()
        got = _gather(arena.theta.detach().clone(), W)
        allcnt = _gather(torch.tensor([be.bytes_sent()], dtype=torch.int64, device=dev), W)
        sim.step([grad_of(s, r) for r in range(W)])
        rows += be.drain_consensus() if s % 4 == 3 or s == a.steps - 1 else []
        if env.rank != 0:
            continue
        for r in range(W):
            if not torch.equal(got[r], sim.theta[r]):
                ok = False
                print(f"step {s + 1} rank {r}: theta differs, max {(got[r] - sim.theta[r]).abs().max().item():.3e}")
            if int(allcnt[r][0]) != sim.bytes[r]:
                ok = False
                print(f"step {s + 1} rank {r}: bytes {int(allcnt[r][0])} vs {sim.bytes[r]}")
    if hasattr(be, "check_status"):
        be.check_status()
    # the measurements: the simulator's steps and values, and the same bits on every rank
    if [k for k, _, _ in rows] != [k for k, _, _ in sim.consensus]:
        ok = False
        print(f"rank {env.rank}: measured steps {[k for k, _, _ in rows]} vs {[k for k, _, _ in sim.consensus]}")
    for (k, D, A), (_, Ds, As) in zip(rows, sim.consensus):
        for name, x, y in (("D", D, Ds), ("A", A, As)):
            same = torch.equal(x, y) if exact else torch.allclose(x, y, rtol=1e-5, atol=1e-30)
            if not same:
                ok = False
                print(f"rank {env.rank} step {k}: {name} differs, max rel "
                      f"{((x - y).abs() / y.abs().clamp_min(1e-300)).max().item():.3e}")
    mine = torch.stack([torch.cat([D, A]) for _, D, A in rows]) if rows else torch.zeros(1)
    everyone = _gather(mine.to(dev) if a.backend == "nccl" else mine, W)
    if not all(torch.equal(everyone[0], x) for x in everyone):
        ok = False
        print("measurements differ across ranks")
    ok = ok and (W == 1 or any(float(D.sum()) > 0 for _, D, _ in rows))
    flags = [None] * W
    dist.all_gather_object(flags, ok)
    if env.rank == 0:
        print("WORKER_OK" if all(flags) else "WORKER_FAIL", f"mode=sim backend={a.backend} algo={a.algo} "
              f"topology={cfg.topology} feature={a.feature} every={a.every} world={W} rows={len(rows)}", flush=True)
    be.close()
    return all(flags)


def _read_csv(path):
    with open(path) as f:
        return [line.rstrip("\n").split(",") for line in f]


def run_trainer(a, env):
    from eventgrad_b200.data import synthetic_source
    from eventgrad_b200.engine.trainer import Trainer
    from eventgrad_b200.utils.ckpt import ckpt_path
    spe, N = 5, 2
    n_train = 32 * spe * env.world
    dev = "cpu" if a.backend == "gloo" else "cuda"

    def trainer(log_dir, **kw):
        base = dict(device=dev, backend=a.backend, model="cnn2", train_samples=n_train, test_samples=64,
                    batch_size=32, batch_mode="per_rank", sampler="random", epochs=2, quiet=env.rank != 0,
                    momentum=0.9, lr=0.05, consensus_every=N, log_dir=log_dir, cuda_graph=False)
        base.update(kw)
        torch.manual_seed(0)
        return Trainer(preset("decent", **base), env, train_source=synthetic_source("mnist", n_train),
                       test_source=synthetic_source("mnist", 64, train=False))

    fails = []

    def check(cond, what):
        if not cond:
            fails.append(what)
            print(f"rank {env.rank}: {what}", flush=True)
        return bool(cond)

    full_dir = os.path.join(a.log_dir, "full")
    full = trainer(full_dir)
    full.fit()
    th_full = full.arena.theta.cpu().clone()
    res = full.finalize(evaluate=False)
    check(res["consensus_last"] is not None and res["consensus_last"] > 0, f"consensus_last {res['consensus_last']}")
    check(res["consensus_before_final_average"] > 0, "consensus_before_final_average")
    if env.rank == 0:
        rows = _read_csv(os.path.join(full_dir, "consensus.csv"))
        check(rows[0] == ["step", "distance", "relative"], "consensus.csv header")
        check([int(r[0]) for r in rows[1:]] == list(range(N, 2 * spe + 1, N)), "consensus.csv steps")
        check(float(rows[-1][2]) == res["consensus_last"], "consensus_last is the last row")
        trows = _read_csv(os.path.join(full_dir, "consensus_tensors.csv"))
        nt = full.arena.table.n_tensors
        check(trows[0] == ["step", "tensor", "sq_dist", "sq_norm_mean"] and len(trows) == 1 + nt * (len(rows) - 1),
              "consensus_tensors.csv rows")
        check(trows[1][1] == full.arena.table.names[0], "tensor names")
        full_rows = rows
    part_dir = os.path.join(a.log_dir, "part")
    part = trainer(part_dir, ckpt_dir=a.ckpt_dir, ckpt_every=1, max_steps=spe)     # stops after epoch 1, at step 5
    part.fit()
    sd = torch.load(ckpt_path(a.ckpt_dir, env.rank), weights_only=True)
    check(not any("consensus" in k for k in sd) and not any("consensus" in k for k in sd["backend"]),
          "checkpoint keys")
    resumed = trainer(part_dir, resume=ckpt_path(a.ckpt_dir, env.rank))
    resumed.fit()
    check(torch.equal(resumed.arena.theta.cpu(), th_full), "resumed theta")
    if env.rank == 0:
        rows = _read_csv(os.path.join(part_dir, "consensus.csv"))
        check(rows == full_rows, f"resumed consensus.csv {rows} vs {full_rows}")
    flags = [None] * env.world
    dist.all_gather_object(flags, not fails)
    if env.rank == 0:
        print("WORKER_OK" if all(flags) else "WORKER_FAIL", f"mode=trainer backend={a.backend} world={env.world}",
              flush=True)
    return all(flags)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="sim", choices=["sim", "trainer"])
    ap.add_argument("--steps", type=int, default=9)
    ap.add_argument("--every", type=int, default=2)
    ap.add_argument("--algo", default="decent", choices=["decent", "event", "spevent"])
    ap.add_argument("--topology", default="ring")
    ap.add_argument("--feature", default="plain", choices=sorted(FEATURES))
    ap.add_argument("--log-dir", default="")
    ap.add_argument("--ckpt-dir", default="")
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl", "p2p"])
    a = ap.parse_args()
    env = init_distributed("cpu" if a.backend == "gloo" else "cuda")
    ok = run_sim(a, env) if a.mode == "sim" else run_trainer(a, env)
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
