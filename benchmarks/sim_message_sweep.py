#!/usr/bin/env python
"""Messages-saved study on the ORACLE (CPU, no GPU): R virtual ranks of the ring simulator, each with its
own shard, real autograd gradients of the real model, iteration-synchronous semantics -- the same
arithmetic the fused kernels reproduce bit-for-bit (tests/test_gpu_kernels.py).  Lets ring sizes that did
not fit the GPU budget (R = 8) be studied, and cross-checks the GPU sweeps at R = 2 / 4.

    python benchmarks/sim_message_sweep.py --world 8 --epochs 10 --horizons 1.0,0.9
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F
from torch.func import functional_call

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.data import ShardSampler, synthetic_source  # noqa: E402
from eventgrad_b200.data.augment import decode_augment_torch  # noqa: E402
from eventgrad_b200.engine.simulator import RingSimulator  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.parallel.arena import ParamArena  # noqa: E402
from eventgrad_b200.parallel.trigger import TriggerConfig  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--model", default="cnn2")
    ap.add_argument("--dataset", default="mnist")
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--lr", type=float, default=0.05)
    ap.add_argument("--momentum", type=float, default=0.0)
    ap.add_argument("--horizons", default="1.0,0.9")
    ap.add_argument("--algo", default="event", choices=["event", "spevent"])
    ap.add_argument("--topk", type=float, default=10.0)
    ap.add_argument("--sampler", default="sequential", choices=["sequential", "random"])
    ap.add_argument("--max-steps", type=int, default=0)
    ap.add_argument("--train-samples", type=int, default=60000)
    ap.add_argument("--trigger", default="norm", choices=["norm", "drift"],
                    help="trigger metric: norm (reference) or drift (||theta - sent||)")
    ap.add_argument("--compress", default="none", choices=["none", "int8"],
                    help="event on the ring: int8 error-feedback codes instead of fp32 messages (bytes_sent counts them)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    R = a.world
    src = synthetic_source(a.dataset, a.train_samples)
    test = synthetic_source(a.dataset, 2000, train=False)
    rows = []
    for hz in [float(x) for x in a.horizons.split(",")]:
        torch.manual_seed(0)
        model = build_model(a.model)
        arena = ParamArena(model)
        t = arena.table
        names = [n for n, _ in model.named_parameters()]
        sim = RingSimulator(R, arena.theta.clone(), t, a.algo, TriggerConfig(1, hz, 0.0, 2, 30, a.trigger), lr=a.lr,
                            momentum=a.momentum, topk_percent=a.topk, serial_skip=False, compress=a.compress)
        samplers = [ShardSampler(len(src), R, r, a.sampler) for r in range(R)]
        steps_per_epoch = samplers[0].num_batches(a.batch)
        t0 = time.perf_counter()
        model.train()
        for ep in range(a.epochs):
            orders = [s.indices() for s in samplers]
            for b in range(steps_per_epoch):
                grads = []
                for r in range(R):
                    idx = orders[r][b * a.batch:(b + 1) * a.batch]
                    x = decode_augment_torch(src.images[idx], src.scale, src.mean, src.std)
                    y = src.labels[idx]
                    th = sim.theta[r].detach().requires_grad_(True)
                    params = {n: th[t.offsets[i]: t.offsets[i] + t.numels[i]].view(t.shapes[i]) for i, n in enumerate(names)}
                    loss = F.cross_entropy(functional_call(model, params, (x,)), y)
                    g, = torch.autograd.grad(loss, th)
                    grads.append(g)
                sim.step(grads)
                if a.max_steps and sim.pass_num >= a.max_steps:
                    break
            if a.max_steps and sim.pass_num >= a.max_steps:
                break
        # evaluate the averaged model
        avg = sim.final_average()
        model.eval()
        with torch.no_grad():
            params = {n: avg[t.offsets[i]: t.offsets[i] + t.numels[i]].view(t.shapes[i]) for i, n in enumerate(names)}
            xt = decode_augment_torch(test.images, test.scale, test.mean, test.std)
            acc = 100.0 * float((functional_call(model, params, (xt,)).argmax(1) == test.labels).float().mean())
        row = {"oracle": "RingSimulator (CPU)", "model": a.model, "algo": a.algo,
               "topk_percent": a.topk if a.algo == "spevent" else None, "trigger": a.trigger, "compress": a.compress, "world": R, "horizon": hz, "epochs": a.epochs,
               "steps": sim.pass_num, "events_total": sim.total_events(), "dense_messages": sim.dense_messages(),
               "messages_saved": 1.0 - sim.total_events() / sim.dense_messages(), "bytes_sent_all_ranks": int(sum(sim.bytes)),
               "test_acc": acc, "wall_s": time.perf_counter() - t0}
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(rows, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
