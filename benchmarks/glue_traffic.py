#!/usr/bin/env python
"""Bytes per training step moved by the memory-bound glue around the convolutions of the flagship ResNet (fp32, NHWC,
tensor-core convolutions), counted from the layer shapes -- before and after the fused conv + BN node (ops/conv_bn.py).

Counted passes, per BatchNorm layer with an fp32 activation of S = 4*M*C bytes (M = batch*H*W):
  bn stats        read x                                               S
  bn apply        read x (+ residual), write y (+ bf16 planes 1.5 S) (+ bit mask S/32 in a residual node)
  bn reduce       read dy, x (+ y for the ReLU mask | + bit mask S/32)
  bn dx           read dy, x (+ y | + bit mask), write dx (S; the fused node writes only the planes) (+ planes 1.5 S)
                  (+ dres S)
  skip add        autograd's add of the two gradients of an identity block's input: read 2 S, write S.  The fused
                  node reads the skip gradient (S) and its mask (S/32) in the epilogue of the first conv's data
                  gradient instead.
The convolutions' own operand traffic is the same before and after and is not counted.  No GPU is needed: the shapes
come from a forward pass on the CPU at batch 1, scaled to the batch.

    python benchmarks/glue_traffic.py [--batch 256] [--model resnet18] [--per-layer]
"""
from __future__ import annotations

import argparse
import os
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def bn_layers(model_name):
    """[(name, C, H, W, residual, relu, emit_planes, fused, hands_over)] in forward order"""
    import torch
    from eventgrad_b200.models.resnet import make_resnet
    from eventgrad_b200.ops.bn_act import FusedBNAct
    model = make_resnet(model_name, variant="ref").train()
    seen = []
    names = {m: n for n, m in model.named_modules()}
    identity_res = set()                      # residual BNs of identity blocks (hand their gradient over)
    for n, m in model.named_modules():
        if hasattr(m, "downsampler") and m.downsampler is None:
            last = [c for c in ("bn3", "bn2") if hasattr(m, c)][0]
            identity_res.add(f"{n}.{last}")

    def hook(mod, args, kwargs):
        x = args[0]
        name = names[mod]
        fused = not name.endswith("downsampler.1")     # every conv+bn pair of the blocks and the stem
        seen.append((name, x.shape[1], x.shape[2], x.shape[3], kwargs.get("residual") is not None,
                     bool(kwargs.get("relu", False)), bool(mod.emit_planes), fused, name in identity_res))
    for m in model.modules():
        if isinstance(m, FusedBNAct):
            m.register_forward_pre_hook(hook, with_kwargs=True)
    with torch.no_grad():
        model(torch.zeros(1, 3, 32, 32))
    return seen


def traffic(layers, batch):
    """{pass: (bytes before, bytes after)}"""
    t = defaultdict(lambda: [0.0, 0.0])
    for (_, C, H, W, res, relu, planes, fused, hand) in layers:
        S = 4.0 * batch * H * W * C
        P = 1.5 * S if planes else 0.0
        t["bn stats"][0] += S
        t["bn stats"][1] += S
        apply = 2 * S + (S if res else 0) + P
        t["bn apply"][0] += apply
        t["bn apply"][1] += apply + (S / 32 if (fused and res and relu) else 0)
        # the ReLU mask in the backward: y before; x (no extra bytes) or the bit mask in a fused node
        mask_b = S if relu else 0.0
        mask_a = (S / 32 if res else 0.0) if fused and relu else mask_b
        t["bn reduce"][0] += 2 * S + mask_b
        t["bn reduce"][1] += 2 * S + mask_a
        # every BN here feeds a tensor-core conv's backward, so the dx kernel always writes the planes (1.5 S)
        t["bn dx"][0] += 2 * S + mask_b + S + 1.5 * S + (S if res else 0)
        t["bn dx"][1] += 2 * S + mask_a + (0 if fused else S) + 1.5 * S + (S if (res and not hand) else 0)
        if hand:
            t["skip add"][0] += 3 * S
            t["skip add"][1] += S + S / 32
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--per-layer", action="store_true")
    a = ap.parse_args()
    layers = bn_layers(a.model)
    if a.per_layer:
        for ly in layers:
            b, f = map(sum, zip(*traffic([ly], a.batch).values()))
            print(f"{ly[0]:24s} C={ly[1]:4d} {ly[2]:2d}x{ly[3]:<2d} res={int(ly[4])} fused={int(ly[7])} "
                  f"hand-off={int(ly[8])}  {b / 1e6:8.1f} -> {f / 1e6:8.1f} MB")
    t = traffic(layers, a.batch)
    S = sum(4.0 * a.batch * ly[1] * ly[2] * ly[3] for ly in layers)
    print(f"{a.model} (reference topology), batch {a.batch}: {len(layers)} BN layers, "
          f"fp32 activations S = {S / 1e6:.0f} MB")
    print(f"{'pass':12s} {'before GB':>10s} {'after GB':>10s} {'saved GB':>10s}")
    tb = ta = 0.0
    for k, (b, f) in t.items():
        print(f"{k:12s} {b / 1e9:10.3f} {f / 1e9:10.3f} {(b - f) / 1e9:10.3f}")
        tb, ta = tb + b, ta + f
    print(f"{'total':12s} {tb / 1e9:10.3f} {ta / 1e9:10.3f} {(tb - ta) / 1e9:10.3f}")


if __name__ == "__main__":
    main()
