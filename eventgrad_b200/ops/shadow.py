"""bf16 shadow weights: Conv2d / Linear whose forward reads a bf16 copy of the fp32 master weight.

The fused step kernel writes the bf16 copy (`GossipParams.shadow`) in the same pass that updates
the fp32 master in the arena, so autocast never launches a cast kernel per weight, and autograd's
weight gradients (bf16, freshly allocated by cuDNN's wgrad) are consumed IN PLACE by the step
kernel through a pointer table -- no AccumulateGrad add, no fp32 grad arena, no zeroing.
The registered nn.Parameters stay the fp32 masters (names / order / state_dict unchanged).
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F


class ShadowConv2d(nn.Conv2d):
    w16 = None
    b16 = None

    def tc_kind(self, x: torch.Tensor):
        """The tensor-core convolution (ops/conv_tc.py kind) this layer runs on x, or None."""
        if (x.is_cuda and x.dtype == torch.float32 and self.bias is None and self.padding_mode == "zeros"
                and not torch.is_autocast_enabled() and not torch.backends.cudnn.allow_tf32):
            # reference precision (fp32): eligible convs run on the tensor cores at fp32 accuracy
            from .conv_tc import kind_of
            return kind_of(x, self.weight, self.stride, self.padding, self.dilation, self.groups)
        return None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.w16 is not None and x.is_cuda and torch.is_autocast_enabled():
            return self._conv_forward(x, self.w16, self.b16)
        kind = self.tc_kind(x)
        if kind is not None:
            from .conv_tc import conv_tc, mark_tc_output
            return mark_tc_output(conv_tc(x, self.weight, kind))
        return super().forward(x)


class ShadowLinear(nn.Linear):
    w16 = None
    b16 = None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.w16 is not None and x.is_cuda and torch.is_autocast_enabled():
            return F.linear(x, self.w16, self.b16)
        return super().forward(x)
