"""CIFAR ResNet family (BasicBlock / BottleNeck; 18/34/50/101/152).

Reference: /root/reference/dcifar10/common/resnet.hpp
  * bias-free convs (:3-9), 3x3 stride-1 stem, no max-pool (:145 commented out),
    stages 64/128/256/512, avg_pool2d(4), Linear(512*expansion, classes) (:141-157).
  * Quirk Q1 (:160-181): make_layer pushes the strided block and THEN loops
    i=0..blocks-1, so every stage holds blocks+1 blocks. The shipped "ResNet-18"
    ({2,2,2,2}) therefore has 12 BasicBlocks / 86 parameter tensors / 17 444 682
    elements. `variant="ref"` reproduces that topology (apples-to-apples message
    shapes); `variant="canonical"` builds the textbook blocks-per-stage network
    (62 tensors / 11 173 962 elements for ResNet-18).
BatchNorm layers are ops.bn_act.FusedBNAct (nn.BatchNorm2d subclass: same names/buffers) so that
bn->relu and bn->(+=skip)->relu run as fused sm_90a kernels on NHWC activations; in fp32 training each conv+bn pair
runs as one autograd node (ops/conv_bn.py).
Parameter registration order matches LibTorch's named_parameters() walk
(conv, bn, layer1..4 [conv1,bn1,conv2,bn2,(conv3,bn3),downsampler], fc) because the
arena layout (= the reference's running `disp`) is defined by that order.
"""
from __future__ import annotations

from typing import Sequence, Type

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.bn_act import FusedBNAct
from ..ops.conv_bn import SkipGrad, conv_bn
from ..ops.shadow import ShadowConv2d, ShadowLinear


def conv_op(cin: int, cout: int, k: int, stride: int, padding: int) -> nn.Conv2d:
    return ShadowConv2d(cin, cout, k, stride=stride, padding=padding, bias=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, cin: int, cout: int, stride: int = 1, downsample: nn.Module | None = None):
        super().__init__()
        self.conv1 = conv_op(cin, cout, 3, stride, 1)
        self.bn1 = FusedBNAct(cout)
        self.conv2 = conv_op(cout, cout, 3, 1, 1)
        self.bn2 = FusedBNAct(cout)
        self.downsampler = downsample

    def forward(self, x):
        skip = SkipGrad() if self.downsampler is None else None      # identity block: bn2 hands x's gradient to conv1
        out = conv_bn(self.conv1, self.bn1, x, relu=True, skip_in=skip)
        residual = self.downsampler(x) if self.downsampler is not None else x
        return conv_bn(self.conv2, self.bn2, out, residual=residual, relu=True, skip_out=skip)   # bn -> += skip -> relu


class BottleNeck(nn.Module):
    expansion = 4

    def __init__(self, cin: int, cout: int, stride: int = 1, downsample: nn.Module | None = None):
        super().__init__()
        self.conv1 = conv_op(cin, cout, 1, 1, 0)
        self.bn1 = FusedBNAct(cout)
        self.conv2 = conv_op(cout, cout, 3, stride, 1)
        self.bn2 = FusedBNAct(cout)
        self.conv3 = conv_op(cout, cout * self.expansion, 1, 1, 0)
        self.bn3 = FusedBNAct(cout * self.expansion)
        self.downsampler = downsample

    def forward(self, x):
        skip = SkipGrad() if self.downsampler is None else None      # identity block: bn3 hands x's gradient to conv1
        out = conv_bn(self.conv1, self.bn1, x, relu=True, skip_in=skip)
        out = conv_bn(self.conv2, self.bn2, out, relu=True)
        residual = self.downsampler(x) if self.downsampler is not None else x
        return conv_bn(self.conv3, self.bn3, out, residual=residual, relu=True, skip_out=skip)


class ResNet(nn.Module):
    def __init__(self, block: Type[nn.Module], layers: Sequence[int], classes: int = 10,
                 variant: str = "ref"):
        super().__init__()
        if variant not in ("ref", "canonical"):
            raise ValueError("variant must be 'ref' or 'canonical'")
        self.variant = variant
        self.in_channels = 64
        self.conv = conv_op(3, 64, 3, 1, 1)
        self.bn = FusedBNAct(64)
        self.layer1 = self._make_layer(block, 64, layers[0], 1)
        self.layer2 = self._make_layer(block, 128, layers[1], 2)
        self.layer3 = self._make_layer(block, 256, layers[2], 2)
        self.layer4 = self._make_layer(block, 512, layers[3], 2)
        self.fc = ShadowLinear(512 * block.expansion, classes)
        self._mark_plane_emitters()

    def _mark_plane_emitters(self) -> None:
        """BN layers whose output feeds a stride-1 convolution write it ALSO as bf16 planes (ops/bn_act.py
        emit_planes): inside a block every BN but the last, and a block's last BN when the NEXT block starts with a
        stride-1 conv that is the only conv reading it (no down-sampler: those read parity planes instead)."""
        blocks = [b for layer in (self.layer1, self.layer2, self.layer3, self.layer4) for b in layer]
        prev_last = self.bn
        for b in blocks:
            convs = [m for m in (getattr(b, "conv1", None), getattr(b, "conv2", None), getattr(b, "conv3", None))
                     if m is not None]
            bns = [m for m in (getattr(b, "bn1", None), getattr(b, "bn2", None), getattr(b, "bn3", None)) if m is not None]
            if b.downsampler is None and tuple(convs[0].stride) == (1, 1):
                prev_last.emit_planes = True
            for bn, nxt in zip(bns[:-1], convs[1:]):
                bn.emit_planes = tuple(nxt.stride) == (1, 1)
            prev_last = bns[-1]

    def _make_layer(self, block, cout: int, blocks: int, stride: int) -> nn.Sequential:
        downsample = None
        if stride != 1 or self.in_channels != cout * block.expansion:
            downsample = nn.Sequential(
                conv_op(self.in_channels, cout * block.expansion, 1, stride, 0),
                FusedBNAct(cout * block.expansion),
            )
        mods = [block(self.in_channels, cout, stride, downsample)]
        self.in_channels = cout * block.expansion
        extra = blocks if self.variant == "ref" else blocks - 1
        for _ in range(extra):
            mods.append(block(self.in_channels, cout))
        return nn.Sequential(*mods)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        out = conv_bn(self.conv, self.bn, x, relu=True)
        out = self.layer4(self.layer3(self.layer2(self.layer1(out))))
        out = F.avg_pool2d(out, 4)
        out = out.reshape(out.shape[0], -1)
        return self.fc(out)


_SPECS = {
    "resnet18": (BasicBlock, (2, 2, 2, 2)),
    "resnet34": (BasicBlock, (3, 4, 6, 3)),
    "resnet50": (BottleNeck, (3, 4, 6, 3)),
    "resnet101": (BottleNeck, (3, 4, 23, 3)),
    "resnet152": (BottleNeck, (3, 8, 36, 3)),
}


def make_resnet(name: str, classes: int = 10, variant: str = "ref") -> ResNet:
    block, layers = _SPECS[name]
    return ResNet(block, layers, classes, variant)
