"""Multi-process worker: one algorithm with weight decay, Nesterov momentum and a multistep learning-rate schedule
whose milestone falls inside the run, on a real process group; every rank's parameters must equal the
single-process simulator's bit for bit (iter-sync).

    torchrun --nproc-per-node R tests/optimizer_worker.py --algo event --backend gloo|refport ...
Used by tests/test_optimizer_cpu.py.
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
from eventgrad_b200.parallel import ParamArena, Ring, make_backend  # noqa: E402
from eventgrad_b200.parallel.trigger import TriggerConfig  # noqa: E402
from eventgrad_b200.utils.dist import init_distributed, shutdown  # noqa: E402

STEPS_PER_EPOCH = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--algo", default="event")
    ap.add_argument("--backend", default="gloo")
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    env = init_distributed("cpu")
    # milestone at epoch 1 = step 5: the run crosses it; warm-up over the first 2 steps
    cfg = TrainConfig(algo=a.algo, dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, weight_decay=5e-4,
                      nesterov=True, lr_schedule="multistep", lr_milestones=(1,), lr_gamma=0.1,
                      lr_warmup_epochs=0.5, epochs=3, horizon=1.0, thres_type=1, topk_percent=10.0,
                      initial_comm_passes=4, backend=a.backend, sync_mode="iter").validate()
    table = lr_table(cfg, STEPS_PER_EPOCH)
    torch.manual_seed(0)
    model = build_model(cfg.model)
    ring = Ring(env.rank, env.world)
    arena = ParamArena(model, env.device)
    be = make_backend(cfg, arena, ring, env)
    be.set_lr_table(table)
    t = arena.table
    theta0 = arena.theta.detach().cpu().clone()
    mask = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        mask[o:o + n] = 1

    def grad_of(step, rank):
        g = torch.Generator().manual_seed(step * 1000 + rank)
        return torch.randn(t.n_padded, generator=g) * 0.05 * mask

    for s in range(a.steps):
        arena.grad.copy_(grad_of(s, env.rank))
        be.step()
        if a.algo != "cent":       # (cent averages the gradient in place, by design)
            # the optimizer must not change the gradient it was given (weight decay works on a copy)
            assert torch.equal(arena.grad, grad_of(s, env.rank))
    W = env.world
    mine = arena.theta.detach().clone()
    allth = [torch.empty_like(mine) for _ in range(W)]
    dist.all_gather(allth, mine)
    ok = True
    if env.rank == 0:
        sim = RingSimulator(W, theta0, t, a.algo, TriggerConfig.from_train(cfg), lr=cfg.lr, momentum=cfg.momentum,
                            topk_percent=cfg.topk_percent, serial_skip=False, weight_decay=cfg.weight_decay,
                            nesterov=cfg.nesterov, lr_table=table)
        for s in range(a.steps):
            sim.step([grad_of(s, r) for r in range(W)])
        for r in range(W):
            if not torch.equal(allth[r], sim.theta[r]):
                ok = False
                print(f"MISMATCH rank {r}: max abs diff {(allth[r] - sim.theta[r]).abs().max().item():.3e}")
        # the schedule really changed the lr inside the run
        assert float(table[0]) < float(table[2]) and float(table[STEPS_PER_EPOCH]) < float(table[2])
        print("WORKER_OK" if ok else "WORKER_FAIL", f"algo={a.algo} backend={a.backend} world={W}", flush=True)
    be.close()
    shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
