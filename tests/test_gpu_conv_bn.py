"""The fused conv + BN node (ops/conv_bn.py) and the mask sources of the BN backward, against the separate ops: bitwise."""
import copy

import pytest
import torch
import torch.nn.functional as F

from eventgrad_b200.models.resnet import make_resnet
from eventgrad_b200.ops import bn_act, conv_bn

pytestmark = pytest.mark.gpu


def _step(model, x, labels):
    loss = F.cross_entropy(model(x), labels)
    loss.backward()
    return loss.detach()


@pytest.mark.parametrize("batch", [256, 32])          # 32: the K-split data gradients (the skip gradient in the reduce)
def test_resnet18_step_matches_separate_ops(batch, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    torch.manual_seed(0)
    fused = make_resnet("resnet18", variant="ref").cuda().to(memory_format=torch.channels_last).train()
    sep = copy.deepcopy(fused)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(batch, 3, 32, 32, generator=g, device="cuda").contiguous(memory_format=torch.channels_last)
    labels = torch.randint(0, 10, (batch,), generator=g, device="cuda")

    calls = []
    real = conv_bn._ConvBNFn.apply
    monkeypatch.setattr(conv_bn._ConvBNFn, "apply", lambda *a: (calls.append(a[-1] is not None), real(*a))[1])
    loss_f = _step(fused, x, labels)
    assert len(calls) == 1 + 12 * 2 and sum(calls) == 9     # stem + 2 per block; 9 identity blocks hand over
    monkeypatch.setattr(conv_bn, "_fused_kind", lambda *a: None)
    loss_s = _step(sep, x, labels)
    torch.cuda.synchronize()

    assert torch.equal(loss_f, loss_s)
    for (n, pf), (_, ps) in zip(fused.named_parameters(), sep.named_parameters()):
        assert torch.equal(pf.grad, ps.grad), n
    for (n, bf), (_, bs) in zip(fused.named_buffers(), sep.named_buffers()):
        assert torch.equal(bf, bs), n


@pytest.mark.parametrize("shape", [(256, 64, 32, 32), (32, 512, 4, 4)])
@pytest.mark.parametrize("res", [False, True])
def test_bn_backward_mask_sources_match_y(shape, res):
    N, C, H, W = shape
    g = torch.Generator(device="cuda").manual_seed(3)
    cl = dict(memory_format=torch.channels_last)
    x = (torch.randn(N, C, H, W, generator=g, device="cuda") * 1.3 + 0.2).contiguous(**cl)
    r = torch.randn(N, C, H, W, generator=g, device="cuda").contiguous(**cl) if res else None
    dy = torch.randn(N, C, H, W, generator=g, device="cuda").contiguous(**cl)
    gamma = torch.rand(C, generator=g, device="cuda") + 0.5
    beta = torch.rand(C, generator=g, device="cuda") - 0.5
    mask = torch.empty(x.numel() // 8, dtype=torch.uint8, device="cuda")
    y, mean, invstd, _ = bn_act.bn_forward(x, gamma, beta, None, None, None, r, True, 0.1, 1e-5, True, None, mask)

    def run(mode, fp32_dx):
        dx = torch.empty_like(x) if fp32_dx else None
        dres = torch.empty_like(x) if res else None
        planes = torch.empty(3, x.numel(), dtype=torch.bfloat16, device="cuda")
        dgamma, dbeta = bn_act.bn_backward(x, y if mode == bn_act.MASK_Y else None, dy, gamma, beta, mean, invstd, True,
                                           0, dx, dres, planes, mode, mask if mode == bn_act.MASK_BITS else None)
        return dgamma, dbeta, planes, dres, dx

    ref = run(bn_act.MASK_Y, True)
    modes = [bn_act.MASK_BITS] + ([] if res else [bn_act.MASK_X])
    for mode in modes:
        out = run(mode, False)
        for a, b in zip(ref[:3], out[:3]):
            assert torch.equal(a, b), mode
        if res:
            assert torch.equal(ref[3], out[3])
    # the bit mask is y > 0, one bit per element in memory order
    bits = ((mask.view(-1, 1) >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1).flatten().bool()
    assert torch.equal(bits, (y.permute(0, 2, 3, 1).flatten() > 0))
