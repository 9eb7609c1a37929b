"""wgmma fused Linear + bias (+ ReLU): front-end of csrc/linear_tc_tma.cu (TMA, SWIZZLE_128B, persistent CTAs).

Forward runs on the Hopper tensor cores (wgmma.mma_async, accumulator in registers, bias/ReLU fused
into the register epilogue).  Backward uses plain library GEMMs (cuBLAS through torch): it is
the forward of the full-batch MNIST MLP (60000/R x 784 x 128 per step) that is the hot GEMM.
Eligibility: CUDA, bf16 operands, N % 16 == 0, 16 <= N <= 256, K % 8 == 0; otherwise F.linear.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn.functional as F


def tc_eligible(x: torch.Tensor, weight: torch.Tensor) -> bool:
    if os.environ.get("EGB_TC_LINEAR", "1") == "0":
        return False
    if not (x.is_cuda and x.dim() == 2 and weight.dim() == 2):
        return False
    n, k = weight.shape
    return n % 16 == 0 and 16 <= n <= 256 and k % 8 == 0 and x.shape[1] == k


def linear_tc_forward(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], relu: bool,
                      out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """Raw kernel call (no autograd). x [M,K], weight [N,K] -> [M,N]."""
    from . import ext
    xb = x.to(torch.bfloat16).contiguous()
    wb = weight.to(torch.bfloat16).contiguous()
    bf = None if bias is None else bias.to(torch.float32).contiguous()
    M, K = xb.shape
    N = wb.shape[0]
    y = torch.empty(M, N, dtype=out_dtype, device=x.device)
    with torch.cuda.device(x.device):
        stream = torch.cuda.current_stream(x.device).cuda_stream
        sm = torch.cuda.get_device_properties(x.device).multi_processor_count
        ext().linear_tc(xb.data_ptr(), wb.data_ptr(), 0 if bf is None else bf.data_ptr(), y.data_ptr(), M, N, K,
                        1 if relu else 0, 1 if out_dtype == torch.bfloat16 else 0, sm, stream)
    return y


class _LinearTcFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, relu):
        y = linear_tc_forward(x, weight, bias, relu, torch.bfloat16)
        ctx.save_for_backward(x, weight, y)
        ctx.relu, ctx.has_bias = relu, bias is not None
        ctx.x_dtype, ctx.w_dtype = x.dtype, weight.dtype
        ctx.b_dtype = None if bias is None else bias.dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, y = ctx.saved_tensors
        dz = dy.to(torch.bfloat16)
        if ctx.relu:
            dz = dz * (y > 0)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = (dz @ weight.to(torch.bfloat16)).to(ctx.x_dtype)
        if ctx.needs_input_grad[1]:
            dw = (dz.t() @ x.to(torch.bfloat16)).to(ctx.w_dtype)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dz.float().sum(0).to(ctx.b_dtype)
        return dx, dw, db, None


def linear_act(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], relu: bool) -> torch.Tensor:
    """act(x @ weight.T + bias); wgmma path when eligible, PyTorch otherwise."""
    if tc_eligible(x, weight) and (x.dtype == torch.bfloat16 or torch.is_autocast_enabled()):
        return _LinearTcFn.apply(x, weight, bias, relu)
    y = F.linear(x, weight, bias)
    return F.relu(y) if relu else y
