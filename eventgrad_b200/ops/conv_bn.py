"""Convolution + BatchNorm (+ residual) (+ ReLU) as ONE autograd node, for the fp32 NHWC training path of the ResNet
blocks: the same kernels as ops/conv_tc.py followed by ops/bn_act.py, with less memory traffic in the backward.

  * The BN backward writes its input gradient only as the three bf16 planes the convolution's backward reads: the
    fp32 copy that the separate ops hand from one node to the other is never read.
  * The ReLU mask is not read back from the saved output y, which is not saved at all.  Without a residual it is
    recomputed from the BN input x (y > 0 exactly when fmaf(x, sc, sh) > 0, the apply kernel's own expression); with a
    residual the forward writes it as one bit per element (M*C/8 bytes).
  * Identity blocks hand the skip-connection gradient over explicitly (`SkipGrad`): the node ending the block (residual
    BN) deposits the gradient it received and its ReLU mask instead of returning an fp32 residual gradient, and the node
    starting the block adds `mask ? dy : 0` in the epilogue of its data-gradient convolution.  The block input then
    receives one gradient instead of two, so autograd runs no add.  fp32 addition is commutative and the masked value is
    the +0.f the BN kernel would have written, so the stored sum is bitwise what the add produced.

Results are bitwise identical to the separate `conv_tc.conv2d` + `FusedBNAct` ops (tests/test_gpu_conv_bn.py).
"""
from __future__ import annotations

import os
import weakref
from typing import Optional

import torch

from . import bn_act, conv_tc


class SkipGrad:
    """The skip-connection gradient of an identity block, from the node ending the block to the node starting it.
    Made fresh by every block forward; graph order runs the depositing backward first (its output gradient is what
    the receiving node's output feeds)."""

    __slots__ = ("armed", "dy", "mask")

    def __init__(self):
        self.armed = False          # set when the receiving node took the fused path
        self.dy = self.mask = None

    def take(self):
        dy, mask = self.dy, self.mask
        self.dy = self.mask = None
        return dy, mask


class _ConvBNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, nbt, residual, kind, momentum, eps, relu,
                emit_planes, skip_in, skip_out):
        N, Ci, H, W = x.shape
        ctx.kind, ctx.geom, ctx.weight = kind, (N, Ci, H, W, weight.shape[0]), weakref.ref(weight)
        z, xp, wtp = conv_tc.conv_forward(x, weight, kind, ctx.needs_input_grad[0])
        z = z.permute(0, 3, 1, 2)                                       # conv output, logical NCHW, channels_last
        yp = torch.empty(3, z.numel(), dtype=torch.bfloat16, device=z.device) if emit_planes else None
        mask = None
        if relu and residual is not None:
            mask = torch.empty(z.numel() // 8, dtype=torch.uint8, device=z.device)
        y, mean, invstd, _ = bn_act.bn_forward(z, gamma, beta, running_mean, running_var, nbt, residual, True, momentum,
                                               eps, relu, yp, mask)
        if yp is not None:
            conv_tc.planes_put(y, yp)
        ctx.save_for_backward(xp, wtp, z, gamma, beta, mean, invstd, mask)
        ctx.relu, ctx.has_res, ctx.skip_in, ctx.skip_out = relu, residual is not None, skip_in, skip_out
        return y

    @staticmethod
    def backward(ctx, dy):
        xp, wtp, z, gamma, beta, mean, invstd, mask = ctx.saved_tensors
        dy = dy.contiguous(memory_format=torch.channels_last)          # no copy for the gradients the ResNet produces
        gp = torch.empty(3, z.numel(), dtype=torch.bfloat16, device=z.device)
        skip_out = ctx.skip_out
        dres = torch.empty_like(z) if (ctx.has_res and skip_out is None) else None
        mode = bn_act.MASK_BITS if mask is not None else bn_act.MASK_X
        dgamma, dbeta = bn_act.bn_backward(z, None, dy, gamma, beta, mean, invstd, ctx.relu, 0, None, dres, gp, mode,
                                           mask)
        if skip_out is not None:
            skip_out.dy, skip_out.mask = dy, mask
        addend = addmask = None
        if ctx.skip_in is not None:
            addend, addmask = ctx.skip_in.take()
        dx, dw = conv_tc.conv_backward(xp, wtp, gp, ctx.geom, ctx.kind, ctx.needs_input_grad[0],
                                       ctx.needs_input_grad[1], z.device, addend, addmask, ctx.weight())
        return dx, dw, dgamma, dbeta, None, None, None, dres, None, None, None, None, None, None, None


def _fused_kind(conv, bn, x, residual, relu):
    """tensor-core kind of conv when bn(conv(x), residual, relu) can run as one node (fp32, NHWC, training), else None"""
    if not (isinstance(bn, bn_act.FusedBNAct) and bn.training and bn.affine and bn.momentum is not None
            and bn.running_mean is not None and torch.is_grad_enabled()):
        return None
    if residual is not None and not relu:
        return None
    kind = conv.tc_kind(x)
    Co = conv.out_channels
    if kind is None or Co % 64 or Co > 2048 or os.environ.get("EGB_FUSED_BN", "1") == "0":
        return None
    if residual is not None:
        N, _, H, W = x.shape
        s = 2 if kind in ("s2", "p2") else 1
        if not (residual.dtype == torch.float32 and tuple(residual.shape) == (N, Co, H // s, W // s)
                and residual.is_contiguous(memory_format=torch.channels_last)):
            return None
    return kind


def conv_bn(conv, bn, x: torch.Tensor, residual: Optional[torch.Tensor] = None, relu: bool = False,
            skip_in: Optional[SkipGrad] = None, skip_out: Optional[SkipGrad] = None) -> torch.Tensor:
    """bn(conv(x), residual=residual, relu=relu), as one autograd node where it applies, else the two modules.
    skip_in: this node starts an identity block (x is the block input) and adds the skip gradient to its data gradient;
    skip_out: this node ends it (residual is the block input) and hands its residual gradient over instead of returning
    it.  The hand-off happens only when both nodes take the fused path.
    The fused path reads the modules' parameters and buffers but does not call the modules, so forward hooks registered
    on `conv` or `bn` do not run there (eval, bf16, NCHW and every other shape still call both modules)."""
    kind = _fused_kind(conv, bn, x, residual, relu)
    if kind is None:
        return bn(conv(x), residual=residual, relu=relu)
    if skip_in is not None:
        skip_in.armed = True
    if skip_out is not None and not skip_out.armed:
        skip_out = None
    return _ConvBNFn.apply(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked,
                           residual, kind, bn.momentum, bn.eps, relu, bool(bn.emit_planes), skip_in, skip_out)
