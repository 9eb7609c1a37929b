"""Device time per step with a weight-gradient kernel in flight, from a torch.profiler trace of the headline step
(CIFAR ResNet-18, fp32, p2p with the gradient table, whole-step CUDA graph, per-GPU batch --batch).

The weight gradients (conv3x3_wgrad_kernel and its split reduce) run on a side stream.  Per step this prints: the
device-busy time (union of every kernel's interval), the time some wgrad kernel is in flight, the part of that time
in which another kernel runs as well (overlapped) and the part in which only wgrad kernels run (exposed).  With the
backward joining the side stream once per pass instead of once per layer, the overlapped share should grow.

    python benchmarks/wgrad_overlap.py [--batch 256] [--steps 5] [--trace FILE] [--out FILE]
"""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

WGRAD = ("conv3x3_wgrad_kernel", "conv_wgrad_reduce_kernel")


def _union(iv):
    out = []
    for a, b in sorted(iv):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def _length(iv):
    return sum(b - a for a, b in iv)


def _intersect(x, y):
    i = j = 0
    out = []
    while i < len(x) and j < len(y):
        a, b = max(x[i][0], y[j][0]), min(x[i][1], y[j][1])
        if a < b:
            out.append([a, b])
        if x[i][1] < y[j][1]:
            i += 1
        else:
            j += 1
    return out


def analyse(trace_path, steps):
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    kern = [(e["ts"], e["ts"] + e["dur"], e["name"]) for e in ev if e.get("cat") == "kernel" and "dur" in e]
    wg = _union([[a, b] for a, b, n in kern if any(w in n for w in WGRAD)])
    other = _union([[a, b] for a, b, n in kern if not any(w in n for w in WGRAD)])
    busy = _union([[a, b] for a, b, _ in kern])
    both = _intersect(wg, other)
    ms = lambda us: us / 1e3 / steps                                  # noqa: E731  (trace times are in us)
    return {"steps": steps, "busy_ms": ms(_length(busy)), "span_ms": ms(busy[-1][1] - busy[0][0]) if busy else 0.0,
            "wgrad_in_flight_ms": ms(_length(wg)), "wgrad_overlapped_ms": ms(_length(both)),
            "wgrad_exposed_ms": ms(_length(wg) - _length(both)),
            "wgrad_kernels": sum(1 for *_, n in kern if any(w in n for w in WGRAD)) // steps}


def main():
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--trace", default="", help="keep the chrome trace here (default: a temporary file)")
    p.add_argument("--out", default="")
    args = p.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from eventgrad_b200.config import preset
    from eventgrad_b200.data import synthetic_source
    from eventgrad_b200.engine.trainer import Trainer
    from eventgrad_b200.utils.dist import DistEnv
    if not torch.cuda.is_available():
        raise SystemExit("wgrad_overlap.py needs a CUDA GPU")
    cfg = preset("cifar_event", backend="p2p", device="cuda", dtype="fp32", batch_size=args.batch,
                 train_samples=4 * args.batch, test_samples=256, epochs=10 ** 6, quiet=True, augment=False)
    tr = Trainer(cfg, DistEnv(0, 1, 0, torch.device("cuda", 0), "none"),
                 train_source=synthetic_source("cifar10", 4 * args.batch).pin())
    pool = [(x.clone(), y.clone()) for (x, y), _ in zip(tr.loader, range(4))]
    for i in range(Trainer.GRAPH_WARMUP_STEPS + 3):                   # eager warm-up + graph capture
        tr.train_step(*pool[i % len(pool)])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            tr.train_step(*pool[i % len(pool)])
        torch.cuda.synchronize()
    trace = args.trace or os.path.join(tempfile.mkdtemp(), "wgrad_overlap.json")
    prof.export_chrome_trace(trace)
    r = analyse(trace, args.steps)
    r.update(batch=args.batch, cuda_graph=bool(tr.cfg.cuda_graph), gpu=torch.cuda.get_device_name(0))
    line = json.dumps(r)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    tr.close()


if __name__ == "__main__":
    main()
