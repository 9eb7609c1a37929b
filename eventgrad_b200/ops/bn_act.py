"""Fused BatchNorm2d (+ residual add) (+ ReLU) for channels-last fp32 / bf16 activations.

Front-end of csrc/bn_act.cu.  `FusedBNAct` is a drop-in nn.BatchNorm2d subclass (same parameter
and buffer names, so the arena layout and state_dicts are unchanged) whose forward takes an
optional residual and a relu flag; the ResNet blocks of the reference
(/root/reference/dcifar10/common/resnet.hpp:39-52, :91-107) map onto it as
    bn(conv(x), relu=True)   and   bn(conv(x), residual=skip, relu=True).
The CUDA path is taken for fp32 (the reference's precision) or bf16 NHWC inputs on a GPU; anything else
(CPU, NCHW, channel counts that are not a multiple of 64) runs the equivalent PyTorch ops -- which are also the numerics oracle in tests/test_gpu_bn.py.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

_WS = {}


def _workspace(device):
    ws = _WS.get(device)
    if ws is None:
        from . import ext
        C = ext()
        sm = torch.cuda.get_device_properties(device).multi_processor_count
        rows = C.bn_partial_rows(sm)
        ctl = torch.zeros(512, dtype=torch.int32, device=device)   # tickets / flags / epochs / status
        ws = {"sm": sm, "partial": torch.empty(rows * 128, dtype=torch.float32, device=device), "ctl": ctl,
              # forward half | backward half: ticket[64], flag[32], epoch[1]
              "f": (ctl[0:].data_ptr(), ctl[128:].data_ptr(), ctl[192:].data_ptr()),
              "b": (ctl[64:].data_ptr(), ctl[160:].data_ptr(), ctl[200:].data_ptr()),
              "status": ctl[256:].data_ptr(), "C": C,
              # fp32 NCHW kernels (csrc/bn_nchw.cu): per-channel tickets (forward | backward) + partial pairs
              "nchw_ticket": torch.zeros(2 * 2048, dtype=torch.int32, device=device),
              "nchw_partial": torch.empty(2048 * 64 * 2, dtype=torch.float32, device=device),
              # single-launch (spin-flag) variant for small tensors: slower than the two-launch split path
              # inside a CUDA graph, so it is opt-in
              "fused": 1 if os.environ.get("EGB_BN_FUSED_SMALL", "0") == "1" else 0}
        _WS[device] = ws
    return ws


def _eligible_nchw(x: torch.Tensor, residual: Optional[torch.Tensor]) -> bool:
    """fp32 NCHW path (csrc/bn_nchw.cu): the layout of the reference-precision run (cuDNN's fp32 convs are NCHW)."""
    if os.environ.get("EGB_FUSED_BN", "1") == "0":
        return False
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.is_contiguous()):
        return False
    hw = x.shape[2] * x.shape[3]
    if hw % 4 or x.shape[1] > 2048 or x.numel() == 0:
        return False
    if residual is not None and not (residual.dtype == x.dtype and residual.shape == x.shape and residual.is_contiguous()):
        return False
    return True


def _eligible(x: torch.Tensor, residual: Optional[torch.Tensor]) -> bool:
    if os.environ.get("EGB_FUSED_BN", "1") == "0":
        return False
    if not (x.is_cuda and x.dtype in (torch.bfloat16, torch.float32) and x.dim() == 4):
        return False
    C = x.shape[1]
    if C % 64 or C > 2048:
        return False
    if not x.is_contiguous(memory_format=torch.channels_last):
        return False
    if residual is not None and not (residual.dtype == x.dtype and residual.shape == x.shape
                                     and residual.is_contiguous(memory_format=torch.channels_last)):
        return False
    return True


# ReLU mask source of the backward (csrc/bn_common.cuh BN_MASK_*): the saved output y, recomputed from the BN input x
# (no residual: y > 0 <=> fmaf(x, sc, sh) > 0), or the bit mask the forward wrote
MASK_Y, MASK_X, MASK_BITS = 0, 1, 2


def bn_forward(x, weight, bias, running_mean, running_var, nbt, residual, training, momentum, eps, relu,
               y_planes=None, mask=None):
    """Launch the forward kernels -> (y, mean, invstd, nchw_hw).  y_planes / mask (uint8 [numel/8]): optional extra
    outputs of the fp32 NHWC path (bf16 planes of y; the ReLU mask as bits)."""
    ws = _workspace(x.device)
    C_ext = ws["C"]
    N, C, H, W = x.shape
    M = N * H * W
    y = torch.empty_like(x)                       # preserves channels_last
    if training:
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        invstd = torch.empty(C, dtype=torch.float32, device=x.device)
        rm = running_mean.data_ptr() if running_mean is not None else 0
        rv = running_var.data_ptr() if running_var is not None else 0
        nb = nbt.data_ptr() if nbt is not None else 0
    else:
        mean = running_mean
        invstd = torch.rsqrt(running_var + eps)
        rm = rv = nb = 0
    stream = torch.cuda.current_stream(x.device).cuda_stream
    nchw = not _eligible(x, residual)              # caller guarantees one of the two layouts is eligible
    nchw_hw = H * W if nchw else 0
    with torch.cuda.device(x.device):
        C_ext.bn_forward(x.data_ptr(), residual.data_ptr() if residual is not None else 0, y.data_ptr(),
                         weight.data_ptr(), bias.data_ptr(), mean.data_ptr(), invstd.data_ptr(), rm, rv, nb,
                         (ws["nchw_partial"] if nchw else ws["partial"]).data_ptr(),
                         ws["nchw_ticket"].data_ptr() if nchw else ws["f"][0], ws["f"][1], ws["f"][2],
                         ws["status"], M, C,
                         float(eps), float(momentum), 1 if relu else 0, 1 if training else 0, ws["fused"],
                         ws["sm"], 1 if x.dtype == torch.float32 else 0, nchw_hw, stream,
                         y_planes.data_ptr() if (y_planes is not None and not nchw) else 0,
                         0 if mask is None else mask.data_ptr())
    return y, mean, invstd, nchw_hw


def bn_backward(x, y, dy, weight, bias, mean, invstd, relu, nchw_hw, dx, dres, dx_planes=None, mask_mode=MASK_Y,
                mask=None):
    """Launch the backward kernels into the given outputs (dx may be None when dx_planes is given) -> (dgamma, dbeta).
    y is read only for mask_mode MASK_Y."""
    ws = _workspace(x.device)
    C_ext = ws["C"]
    N, C, H, W = x.shape
    M = N * H * W
    dgamma = torch.empty(C, dtype=torch.float32, device=x.device)
    dbeta = torch.empty(C, dtype=torch.float32, device=x.device)
    ptr = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
    stream = torch.cuda.current_stream(x.device).cuda_stream
    with torch.cuda.device(x.device):
        C_ext.bn_backward(x.data_ptr(), ptr(y), dy.data_ptr(), ptr(dx), ptr(dres), weight.data_ptr(), mean.data_ptr(),
                          invstd.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(),
                          (ws["nchw_partial"] if nchw_hw else ws["partial"]).data_ptr(),
                          ws["nchw_ticket"][2048:].data_ptr() if nchw_hw else ws["b"][0], ws["b"][1], ws["b"][2],
                          ws["status"], M, C, 1 if relu else 0,
                          ws["fused"], ws["sm"], 1 if x.dtype == torch.float32 else 0, nchw_hw, stream,
                          ptr(dx_planes), ptr(bias), mask_mode, ptr(mask))
    return dgamma, dbeta


class _FusedBNActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, nbt, residual, training, momentum, eps, relu,
                y_planes=None, dx_planes_wanted=False):
        y, mean, invstd, ctx.nchw_hw = bn_forward(x, weight, bias, running_mean, running_var, nbt, residual, training,
                                                  momentum, eps, relu, y_planes)
        nchw = ctx.nchw_hw > 0
        ctx.dx_planes = bool(dx_planes_wanted) and not nchw and x.dtype == torch.float32
        ctx.save_for_backward(x, y, weight, mean, invstd)
        ctx.relu, ctx.has_res, ctx.training = relu, residual is not None, training
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, weight, mean, invstd = ctx.saved_tensors
        if not ctx.training:
            raise RuntimeError("FusedBNAct backward is only implemented for training mode")
        if ctx.nchw_hw:
            if dy.dtype != x.dtype or not dy.is_contiguous():
                dy = dy.to(x.dtype).contiguous()
        elif dy.dtype != x.dtype or not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.to(x.dtype).contiguous(memory_format=torch.channels_last)
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if ctx.has_res else None
        dxp = torch.empty(3, x.numel(), dtype=torch.bfloat16, device=x.device) if ctx.dx_planes else None
        dgamma, dbeta = bn_backward(x, y, dy, weight, None, mean, invstd, ctx.relu, ctx.nchw_hw, dx, dres, dxp)
        if dxp is not None:
            from .conv_tc import planes_put
            planes_put(dx, dxp)                     # the producing conv's backward finds its dY already split
        return dx, dgamma, dbeta, None, None, None, dres, None, None, None, None, None, None


def bn_act_reference(x, weight, bias, running_mean, running_var, residual, training, momentum, eps, relu):
    """Plain PyTorch composition (CPU / fp32 / NCHW path and the test oracle)."""
    y = F.batch_norm(x, running_mean, running_var, weight, bias, training, momentum, eps)
    if residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


class FusedBNAct(nn.BatchNorm2d):
    # set by the model (models/resnet.py) on layers whose output feeds a 3x3/stride-1 or 1x1/stride-1 convolution: in
    # fp32 those run on the tensor cores from three bf16 planes, which the apply kernel can write on the way out
    emit_planes = False

    def forward(self, x: torch.Tensor, residual: Optional[torch.Tensor] = None, relu: bool = False) -> torch.Tensor:
        training = self.training or (self.running_mean is None)
        nhwc = _eligible(x, residual)
        if (nhwc or _eligible_nchw(x, residual)) and self.affine and self.momentum is not None:
            yp, want_dxp = None, False
            if nhwc and x.dtype == torch.float32:
                from . import conv_tc
                if conv_tc.enabled():
                    want_dxp = bool(getattr(x, "_egb_tc", False)) and training and torch.is_grad_enabled()
                    if self.emit_planes:
                        yp = torch.empty(3, x.numel(), dtype=torch.bfloat16, device=x.device)
            y = _FusedBNActFn.apply(x, self.weight, self.bias, self.running_mean, self.running_var,
                                    self.num_batches_tracked if training else None, residual, training,
                                    self.momentum, self.eps, relu, yp, want_dxp)
            if yp is not None:
                conv_tc.planes_put(y, yp)
            return y
        if training and self.track_running_stats and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
        return bn_act_reference(x, self.weight, self.bias, self.running_mean, self.running_var, residual,
                                training, self.momentum if self.momentum is not None else 0.0, self.eps, relu)


def bn_status(device) -> int:
    """Sticky status word of the fused BN kernels on `device` (0 ok, 2 = a flag wait timed out)."""
    ws = _WS.get(torch.device(device))
    return 0 if ws is None else int(ws["ctl"][256].item())
