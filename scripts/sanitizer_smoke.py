#!/usr/bin/env python
"""Tiny end-to-end exercise of every hand-written kernel, meant to run under compute-sanitizer:

    compute-sanitizer --tool memcheck  python scripts/sanitizer_smoke.py
    compute-sanitizer --tool racecheck python scripts/sanitizer_smoke.py     (shared-memory hazards)

Two virtual ranks on one GPU (ops.local_world) drive the cross-rank protocol of the exchange kernels;
the BN / Linear / augment kernels run on small tensors.  Exits non-zero on any numerical mismatch.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eventgrad_b200.config import TrainConfig  # noqa: E402
from eventgrad_b200.engine.simulator import RingSimulator  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.ops.local_world import LocalWorld  # noqa: E402
from eventgrad_b200.parallel.trigger import TriggerConfig  # noqa: E402


def exchange(algo, **kw):
    cfg = TrainConfig(algo=algo, dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, sync_mode="iter",
                      initial_comm_passes=2, topk_percent=10.0, **kw).validate()
    w = LocalWorld(cfg, 2, lambda: build_model("cnn2"), grid_cap=4, timeout_ns=20_000_000_000)
    t = w.arenas[0].table
    sim = RingSimulator(2, w.arenas[0].theta.cpu(), t, algo, TriggerConfig.from_train(cfg), lr=cfg.lr,
                        momentum=cfg.momentum, topk_percent=10.0, serial_skip=False, gossip_rounds=cfg.gossip_rounds,
                        offsets=cfg.for_world(2).topology, topology_seed=cfg.topology_seed,
                        gossip_accel=cfg.gossip_accel)
    mask = torch.zeros(t.n_padded, device="cuda")
    for o, n in zip(t.offsets, t.numels):
        mask[o:o + n] = 1
    for s in range(3):
        fires = [be.fire.clone().bool() for be in w.backends] if algo in ("event", "spevent") else None
        g = [torch.randn(t.n_padded, device="cuda", generator=torch.Generator("cuda").manual_seed(10 * s + r)) * 0.05 * mask
             for r in range(2)]
        w.step(g)
        if algo != "cent":
            sim.step([x.cpu() for x in g], fires=fires)
    torch.cuda.synchronize()
    for r, be in enumerate(w.backends):
        be.check_status()
        if algo != "cent":
            assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), (algo, r)
    if algo != "cent":
        w.final_average()
    w.close()
    print("ok", algo, kw)


def main():
    for algo in ("decent", "event", "spevent", "cent"):
        exchange(algo)
    exchange("decent", overlap_push=True)
    exchange("decent", overlap_push=False, gossip_rounds=2)       # the mix-only round kernel ahead of the step
    exchange("decent", topology="random-match", topology_seed=3)  # the single-inbox random-match step
    exchange("decent", overlap_push=False, gossip_rounds=2, gossip_accel="chebyshev")  # Chebyshev rounds, serial step
    # fused BN (+res)(+relu), both paths
    from eventgrad_b200.ops.bn_act import FusedBNAct, _workspace
    for fused in (0, 1):
        x = torch.randn(4, 128, 8, 8, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        r = torch.randn_like(x)
        _workspace(x.device)["fused"] = fused
        bn = FusedBNAct(128).cuda().train()
        xa = x.clone().requires_grad_(True)
        ra = r.clone().requires_grad_(True)
        y = bn(xa, residual=ra, relu=True)
        y.backward(torch.randn_like(y))
        assert torch.isfinite(xa.grad.float()).all()
    _workspace(x.device)["fused"] = 0
    print("ok bn")
    # wgmma linear
    from eventgrad_b200.ops.linear_tc import linear_tc_forward
    xx = torch.randn(200, 80, device="cuda").to(torch.bfloat16)
    ww = (torch.randn(32, 80, device="cuda") * 0.1).to(torch.bfloat16)
    bb = torch.randn(32, device="cuda")
    out = linear_tc_forward(xx, ww, bb, True, torch.float32)
    ref = (xx.float() @ ww.float().t() + bb).relu()
    assert torch.allclose(out, ref, rtol=2e-3, atol=2e-3)
    print("ok linear_tc")
    # decode/augment
    from eventgrad_b200.data.augment import decode_augment_torch, draw_augment_params
    from eventgrad_b200.ops.augment import decode_augment
    u = torch.randint(0, 256, (9, 3, 32, 32), dtype=torch.uint8, device="cuda")
    p = draw_augment_params(9, 4, "cuda")
    assert torch.allclose(decode_augment(u, 1.0, 0.0, 1.0, p), decode_augment_torch(u, 1.0, 0.0, 1.0, p))
    print("ok augment")
    # wgmma fp32-accuracy convolutions: every kind (forward, dgrad, wgrad; K-split and un-split grids), the fp32 BN
    # kernels handing bf16 planes over, against cuDNN fp32
    import torch.nn.functional as F
    from eventgrad_b200.ops import conv_tc
    torch.backends.cudnn.allow_tf32 = False
    cases = [(3, 64, 64, 3, 1, 1, 32), (20, 64, 64, 3, 1, 1, 32), (2, 64, 128, 3, 2, 1, 16), (2, 64, 128, 1, 2, 0, 16),
             (2, 64, 64, 1, 1, 0, 8), (2, 3, 64, 3, 1, 1, 32), (9, 128, 64, 3, 1, 1, 4)]
    bad = []
    for (n, ci, co, k, st, pd, hw) in cases:
        xc = torch.randn(n, ci, hw, hw, device="cuda").contiguous(memory_format=torch.channels_last)
        wc = (torch.randn(co, ci, k, k, device="cuda") * 0.05).contiguous(memory_format=torch.channels_last)
        need_dx = ci != 3
        x1, w1 = xc.clone().requires_grad_(need_dx), wc.clone().requires_grad_(True)
        y1 = conv_tc.conv2d(x1, w1, None, (st, st), (pd, pd), (1, 1), 1)
        gy = torch.randn_like(y1)
        y1.backward(gy)
        x2, w2 = xc.clone().requires_grad_(need_dx), wc.clone().requires_grad_(True)
        y2 = F.conv2d(x2, w2, stride=st, padding=pd)
        y2.backward(gy)
        assert conv_tc.kind_of(xc, wc, (st, st), (pd, pd), (1, 1), 1) is not None

        def err(a, b):            # relative to the largest element (cuDNN's own fp32 wgrad is only good to ~1e-5 of it)
            return float((a - b).abs().max()) / float(b.abs().max())
        e = [err(y1, y2), err(w1.grad, w2.grad)] + ([err(x1.grad, x2.grad)] if need_dx else [])
        print("conv case", (n, ci, co, k, st, hw), conv_tc.kind_of(xc, wc, (st, st), (pd, pd), (1, 1), 1),
              "max err vs cuDNN fp32 (y, dw, dx):", ["%.1e" % v for v in e])
        bad = bad + [(n, ci, co, k, st, hw)] if max(e) > 2e-4 else bad
    assert not bad, bad
    from eventgrad_b200.models.resnet import BasicBlock
    blk = BasicBlock(64, 64).cuda().to(memory_format=torch.channels_last).train()
    xb = torch.randn(4, 64, 16, 16, device="cuda").contiguous(memory_format=torch.channels_last).requires_grad_(True)
    blk(xb).sum().backward()
    assert torch.isfinite(xb.grad).all()
    print("ok conv_tc")
    print("SANITIZER_SMOKE_OK")


if __name__ == "__main__":
    main()
