#!/usr/bin/env python
"""Per-layer timing of the wgmma fp32-accuracy 3x3 convolution (csrc/conv_tc.cu) against cuDNN fp32 (TF32 off).

For every distinct 3x3/stride-1 conv of the reference ResNet (dcifar10/common/resnet.hpp) at the headline batch:
forward, data gradient and weight gradient -- the raw kernels on pre-split planes, the fp32->planes split passes,
and cuDNN's fp32 NCHW (its best fp32 layout) for the same op.  CUDA events, rotating buffers larger than L2.

    python benchmarks/conv_tc_bench.py --batch 256 --out conv_tc_bench.json
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.ops import conv_tc  # noqa: E402


def timed(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3     # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    ap.add_argument("--no-cudnn", action="store_true")
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    rows = []
    for (H, C) in [(32, 64), (16, 128), (8, 256), (4, 512)]:
        N, W = a.batch, H
        nrot = max(2, int(160e6 // (N * H * W * C * 4)) + 1)
        xs = [torch.randn(N, C, H, W, device="cuda").contiguous(memory_format=torch.channels_last) for _ in range(nrot)]
        dys = [torch.randn(N, C, H, W, device="cuda").contiguous(memory_format=torch.channels_last) for _ in range(nrot)]
        w = (torch.randn(C, C, 3, 3, device="cuda") * 0.05).contiguous(memory_format=torch.channels_last)
        xps = [conv_tc.split3(x) for x in xs]
        gps = [conv_tc.split3(g) for g in dys]
        wp = conv_tc.split3(w.permute(0, 2, 3, 1).contiguous())
        k = [0]

        def rot():
            k[0] = (k[0] + 1) % nrot
            return k[0]
        flops = 2.0 * N * H * W * C * C * 9
        r = {"N": N, "H": H, "W": W, "C": C, "gflop": flops / 1e9}
        r["fprop_us"] = timed(lambda: conv_tc.fprop_planes(xps[rot()], wp, N, H, W, C, C), a.iters)
        r["wgrad_us"] = timed(lambda: conv_tc.wgrad_planes(xps[rot()], gps[k[0]], N, H, W, C, C), a.iters)
        r["split_act_us"] = timed(lambda: conv_tc.split3(xs[rot()]), a.iters)
        r["fprop_TFLOPs"] = flops / r["fprop_us"] / 1e6
        r["wgrad_TFLOPs"] = flops / r["wgrad_us"] / 1e6
        # the autograd op end to end (split x, split w, fprop | split dy, flip w, dgrad, wgrad)
        xr = [x.clone().requires_grad_(True) for x in xs]
        wr = w.clone().requires_grad_(True)

        def fb_ours():
            i = rot()
            xr[i].grad = None
            wr.grad = None
            conv_tc.conv3x3_tc(xr[i], wr).backward(dys[i])
        r["ours_fwd_bwd_us"] = timed(fb_ours, a.iters)
        if not a.no_cudnn:
            xn = [x.contiguous().clone().requires_grad_(True) for x in xs]      # NCHW: cuDNN's fast fp32 layout
            dn = [g.contiguous() for g in dys]
            wn = w.contiguous().clone().requires_grad_(True)

            def fb_cudnn():
                i = rot()
                xn[i].grad = None
                wn.grad = None
                F.conv2d(xn[i], wn, padding=1).backward(dn[i])
            r["cudnn_fp32_nchw_fwd_bwd_us"] = timed(fb_cudnn, a.iters)
            r["cudnn_fp32_nchw_fwd_us"] = timed(lambda: F.conv2d(xn[rot()].detach(), wn.detach(), padding=1), a.iters)
            r["speedup_fwd_bwd"] = r["cudnn_fp32_nchw_fwd_bwd_us"] / r["ours_fwd_bwd_us"]
        print(json.dumps(r), flush=True)
        rows.append(r)
        del xs, dys, xps, gps, xr
        torch.cuda.empty_cache()
    if a.out:
        json.dump(rows, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
