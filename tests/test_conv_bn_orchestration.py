"""CPU oracle for the host side of the fused conv + BN node (ops/conv_bn.py).

The convolution primitives are emulated as in tests/test_conv_tc_orchestration.py, and the BN launches
(bn_act.bn_forward / bn_backward) by PyTorch code that follows the kernels' documented semantics: the ReLU mask as one
bit per element in memory order, the input gradient written only as bf16 planes, the optional residual gradient.  With
those the REAL autograd Function must reproduce autograd of F.conv2d + F.batch_norm (+ residual) + ReLU, and an identity
block must hand its skip gradient to its first convolution instead of returning it.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_conv_tc_orchestration as orch
from eventgrad_b200.ops import bn_act, conv_bn
from eventgrad_b200.ops import conv_tc as ct


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _pack(bits):
    return torch.from_numpy(np.packbits(bits.flatten().numpy().astype(np.uint8), bitorder="little"))


def _unpack(mask, n):
    return torch.from_numpy(np.unpackbits(mask.numpy(), bitorder="little")[:n].astype(bool))


def emu_bn_forward(x, weight, bias, running_mean, running_var, nbt, residual, training, momentum, eps, relu,
                   y_planes=None, mask=None):
    xd = x.detach()
    mean = xd.mean(dim=(0, 2, 3))
    invstd = torch.rsqrt(xd.var(dim=(0, 2, 3), unbiased=False) + eps)
    v = F.batch_norm(xd, running_mean, running_var, weight.detach(), bias.detach(), True, momentum, eps)
    if nbt is not None:
        nbt.add_(1)
    if residual is not None:
        v = v + residual.detach()
    y = (F.relu(v) if relu else v).contiguous(memory_format=torch.channels_last)
    if y_planes is not None:
        y_planes.copy_(orch.emu_split3(y))
    if mask is not None:
        mask.copy_(_pack(_nhwc(v) > 0))
    return y, mean, invstd, 0


def emu_bn_backward(x, y, dy, weight, bias, mean, invstd, relu, nchw_hw, dx, dres, dx_planes=None,
                    mask_mode=bn_act.MASK_Y, mask=None):
    sh = (1, -1, 1, 1)
    xhat = (x - mean.view(sh)) * invstd.view(sh)
    if not relu:
        keep = torch.ones_like(x, dtype=torch.bool)
    elif mask_mode == bn_act.MASK_X:
        keep = xhat * weight.view(sh) + bias.view(sh) > 0
    elif mask_mode == bn_act.MASK_BITS:
        keep = _unpack(mask, x.numel()).reshape(_nhwc(x).shape).permute(0, 3, 1, 2)
    else:
        keep = y > 0
    dz = torch.where(keep, dy, torch.zeros_like(dy))
    M = x.numel() // x.shape[1]
    dbeta = dz.sum(dim=(0, 2, 3))
    dgamma = (dz * xhat).sum(dim=(0, 2, 3))
    g = weight.view(sh) * invstd.view(sh) * (dz - dbeta.view(sh) / M - xhat * dgamma.view(sh) / M)
    if dx is not None:
        dx.copy_(g)
    if dx_planes is not None:
        dx_planes.copy_(orch.emu_split3(g.contiguous(memory_format=torch.channels_last)))
    if dres is not None:
        dres.copy_(dz)
    return dgamma, dbeta


def emu_fprop(*a, addend=None, addmask=None, **k):
    out = orch.emu_fprop(*a, **k)
    if addend is not None:
        keep = _unpack(addmask, out.numel()).reshape(out.shape)
        out += torch.where(keep, _nhwc(addend), torch.zeros_like(out))
    return out


def _emulate(monkeypatch):
    for name, fn in (("split3", orch.emu_split3), ("split3_parity", orch.emu_split3_parity),
                     ("split3_stem", orch.emu_split3_stem), ("wprep", orch.emu_wprep), ("fprop", emu_fprop),
                     ("wgrad", orch.emu_wgrad)):
        monkeypatch.setattr(ct, name, fn)
    monkeypatch.setattr(bn_act, "bn_forward", emu_bn_forward)
    monkeypatch.setattr(bn_act, "bn_backward", emu_bn_backward)
    ct._PARITY_CACHE.update({"ref": None, "ver": -1, "planes": None})


def _params(C, g):
    return dict(gamma=(torch.rand(C, generator=g) + 0.5).requires_grad_(True),
                beta=(torch.rand(C, generator=g) - 0.5).requires_grad_(True),
                rm=torch.zeros(C), rv=torch.ones(C), nbt=torch.zeros((), dtype=torch.long))


def _node(x, w, p, kind, residual=None, relu=True, skip_in=None, skip_out=None):
    return conv_bn._ConvBNFn.apply(x, w, p["gamma"], p["beta"], p["rm"], p["rv"], p["nbt"], residual, kind, 0.1, 1e-5,
                                   relu, False, skip_in, skip_out)


def _ref(x, w, p, stride, pad, residual=None, relu=True):
    z = F.conv2d(x, w, stride=stride, padding=pad)
    v = F.batch_norm(z, p["rm"], p["rv"], p["gamma"], p["beta"], True, 0.1, 1e-5)
    if residual is not None:
        v = v + residual
    return F.relu(v) if relu else v


def _close(a, b):
    return torch.allclose(a, b, atol=5e-5, rtol=1e-4)


@pytest.mark.parametrize("kind,k,st,pd,res", [("s1", 3, 1, 1, False), ("s1", 3, 1, 1, True), ("p1", 1, 1, 0, True),
                                              ("s2", 3, 2, 1, False), ("p2", 1, 2, 0, False)])
def test_node_reproduces_conv_bn_relu(kind, k, st, pd, res, monkeypatch):
    _emulate(monkeypatch)
    g = torch.Generator().manual_seed(5)
    cl = dict(memory_format=torch.channels_last)
    x = torch.randn(2, 8, 8, 8, generator=g).contiguous(**cl)
    w = (torch.randn(16, 8, k, k, generator=g) * 0.3).contiguous(**cl)
    Ho = 8 // st
    r = torch.randn(2, 16, Ho, Ho, generator=g).contiguous(**cl) if res else None
    gy = torch.randn(2, 16, Ho, Ho, generator=g).contiguous(**cl)
    p1 = _params(16, g)
    p2 = {n: (t.detach().clone().requires_grad_(t.requires_grad)) for n, t in p1.items()}
    x1, w1, r1 = x.clone().requires_grad_(True), w.clone().requires_grad_(True), None if r is None else r.clone().requires_grad_(True)
    x2, w2, r2 = x.clone().requires_grad_(True), w.clone().requires_grad_(True), None if r is None else r.clone().requires_grad_(True)
    y1 = _node(x1, w1, p1, kind, r1)
    y2 = _ref(x2, w2, p2, st, pd, r2)
    assert _close(y1, y2)
    y1.backward(gy)
    y2.backward(gy)
    for a, b in [(x1.grad, x2.grad), (w1.grad, w2.grad), (p1["gamma"].grad, p2["gamma"].grad),
                 (p1["beta"].grad, p2["beta"].grad)] + ([(r1.grad, r2.grad)] if res else []):
        assert _close(a, b)
    assert torch.allclose(p1["rm"], p2["rm"]) and torch.allclose(p1["rv"], p2["rv"]) and int(p1["nbt"]) == 1


def test_identity_block_hands_the_skip_gradient_to_its_first_conv(monkeypatch):
    _emulate(monkeypatch)
    returned = []
    real_bwd = conv_bn._ConvBNFn.backward
    monkeypatch.setattr(conv_bn._ConvBNFn, "backward",
                        staticmethod(lambda ctx, dy: (lambda r: (returned.append(r), r)[1])(real_bwd(ctx, dy))))
    g = torch.Generator().manual_seed(9)
    cl = dict(memory_format=torch.channels_last)
    x = torch.randn(2, 8, 4, 4, generator=g).contiguous(**cl)
    wa = (torch.randn(8, 8, 3, 3, generator=g) * 0.3).contiguous(**cl)
    wb = (torch.randn(8, 8, 3, 3, generator=g) * 0.3).contiguous(**cl)
    gy = torch.randn(2, 8, 4, 4, generator=g).contiguous(**cl)
    pa, pb = _params(8, g), _params(8, g)
    qa = {n: t.detach().clone().requires_grad_(t.requires_grad) for n, t in pa.items()}
    qb = {n: t.detach().clone().requires_grad_(t.requires_grad) for n, t in pb.items()}

    x1 = x.clone().requires_grad_(True)
    skip = conv_bn.SkipGrad()
    skip.armed = True
    out = _node(x1, wa, pa, "s1", skip_in=skip)
    y1 = _node(out, wb, pb, "s1", residual=x1, skip_out=skip)
    y1.backward(gy)

    x2 = x.clone().requires_grad_(True)
    y2 = _ref(_ref(x2, wa, qa, 1, 1), wb, qb, 1, 1, residual=x2)
    y2.backward(gy)

    assert returned[0][7] is None                 # the residual BN returned no gradient for the block input ...
    assert skip.dy is None and skip.mask is None  # ... the first conv consumed the hand-off ...
    assert _close(x1.grad, x2.grad)               # ... and the block input's gradient is still complete
    for a, b in [(pa["gamma"].grad, qa["gamma"].grad), (pb["beta"].grad, qb["beta"].grad)]:
        assert _close(a, b)
