#!/usr/bin/env python
"""Two launches of each wgmma conv kernel instantiation at the headline shapes (batch 256): the ncu target.
    ncu --set full --import-source on --clock-control none -k regex:conv3x3 -o gpurun_out/conv_tc python benchmarks/conv_tc_ncu.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.ops import conv_tc  # noqa: E402

N = int(os.environ.get("BATCH", "256"))
for (H, C) in [(16, 128), (32, 64)]:
    x = torch.randn(N, C, H, H, device="cuda").contiguous(memory_format=torch.channels_last)
    g = torch.randn(N, C, H, H, device="cuda").contiguous(memory_format=torch.channels_last)
    w = (torch.randn(C, C, 3, 3, device="cuda") * 0.05).contiguous(memory_format=torch.channels_last)
    xp, gp = conv_tc.split3(x), conv_tc.split3(g)
    wp, _ = conv_tc.wprep(w.permute(0, 2, 3, 1).reshape(C, 9, C).contiguous(), False)
    for _ in range(2):
        conv_tc.fprop(xp, wp, N, H, H, C, C, conv_tc.TAPS_S1, 1, 9)
        conv_tc.wgrad(xp, gp, N, H, H, C, C, conv_tc.TAPS_S1, 1)
    torch.cuda.synchronize()
print("done")
