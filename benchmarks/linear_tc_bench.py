#!/usr/bin/env python
"""wgmma fused Linear+bias+ReLU vs cuBLAS (torch F.linear + relu) on the MNIST-MLP shapes."""
import json, os, sys
import torch
import torch.nn.functional as F
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.ops.linear_tc import linear_tc_forward

def t(fn, n=50):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3

res = []
for M in (7500, 30000, 60000):
    K, N = 784, 128
    x = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda") * 0.03).to(torch.bfloat16)
    b = torch.randn(N, device="cuda")
    bb = b.to(torch.bfloat16)
    us_tc = t(lambda: linear_tc_forward(x, w, b, True, torch.bfloat16))
    us_cublas = t(lambda: F.relu(F.linear(x, w, bb)))
    flops = 2.0 * M * K * N
    res.append({"M": M, "K": K, "N": N, "wgmma_fused_us": us_tc, "cublas_plus_relu_us": us_cublas,
                "wgmma_TFLOPs": flops / us_tc / 1e6, "cublas_TFLOPs": flops / us_cublas / 1e6,
                "min_bytes_GBps_tc": (M * K * 2 + M * N * 2 + N * K * 2) / us_tc / 1e3})
    print(json.dumps(res[-1]))
if len(sys.argv) > 1:
    json.dump(res, open(sys.argv[1], "w"), indent=1)
