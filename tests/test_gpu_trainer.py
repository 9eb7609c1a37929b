"""Trainer-level GPU tests (single GPU): table mode vs flat grad arena, CUDA graph vs eager,
fused-kernel training actually learns, checkpoint round trip on the p2p backend."""
import pytest
import torch

from eventgrad_b200.config import preset
from eventgrad_b200.data import synthetic_source
from eventgrad_b200.engine.trainer import Trainer
from eventgrad_b200.utils.dist import DistEnv

pytestmark = pytest.mark.gpu


def _env():
    return DistEnv(0, 1, 0, torch.device("cuda", 0), "none")


def _run(steps=4, **kw):
    base = dict(backend="p2p", device="cuda", train_samples=512, test_samples=128, batch_size=64,
                epochs=100, quiet=True, max_steps=steps, augment=False)
    base.update(kw)
    cfg = preset("cifar_event", **base)
    torch.manual_seed(0)
    tr = Trainer(cfg, _env(), train_source=synthetic_source("cifar10", 512).pin(),
                 test_source=synthetic_source("cifar10", 128, train=False).pin())
    tr.fit()
    tr.backend.check_status()
    th = tr.arena.theta.clone()
    return tr, th


def test_table_mode_equals_flat_grad_arena_fp32():
    torch.backends.cudnn.deterministic = True
    try:
        a, tha = _run(dtype="fp32", grad_table=True, model="lenet")
        b, thb = _run(dtype="fp32", grad_table=False, model="lenet")
    finally:
        torch.backends.cudnn.deterministic = False
    assert a.arena.table_mode and not b.arena.table_mode
    torch.testing.assert_close(tha, thb, rtol=1e-6, atol=1e-7)
    a.close(); b.close()


def test_shadow_weights_track_master_and_match_autocast():
    a, tha = _run(dtype="bf16", grad_table=True, channels_last=True)
    assert a.arena.shadow is not None
    t = a.arena.table
    for i in (0, 3, t.n_tensors - 2):
        m = a.arena.flat(a.arena.theta, i)
        s = a.arena.shadow[t.offsets[i]: t.offsets[i] + t.numels[i]]
        assert torch.equal(m.to(torch.bfloat16), s)                 # kernel writes rn(bf16) of the new master
    b, thb = _run(dtype="bf16", grad_table=False, channels_last=True)
    rel = float((tha - thb).norm() / thb.norm())
    assert rel < 5e-3, rel
    a.close(); b.close()


def test_cuda_graph_whole_step_matches_eager():
    a, tha = _run(steps=8, dtype="bf16", cuda_graph=True, channels_last=True)
    b, thb = _run(steps=8, dtype="bf16", cuda_graph=False, channels_last=True)
    assert len(a._graphs) == 1
    rel = float((tha - thb).norm() / thb.norm())
    assert rel < 5e-3, rel
    a.close(); b.close()


def test_mnist_event_self_loop_learns_and_counts():
    cfg = preset("mnist_event", backend="p2p", device="cuda", train_samples=2048, test_samples=512, epochs=2,
                 quiet=True, file_write=0)
    torch.manual_seed(0)
    tr = Trainer(cfg, _env(), train_source=synthetic_source("mnist", 2048).pin(),
                 test_source=synthetic_source("mnist", 512, train=False).pin())
    tr.fit()
    res = tr.finalize()
    assert res["test_acc"] > 50.0, res
    assert 0 < res["events_total"] <= res["dense_messages"] and res["events_total"] % 2 == 0
    tr.close()


def test_p2p_checkpoint_roundtrip(tmp_path):
    from eventgrad_b200.utils.ckpt import ckpt_path, load_checkpoint, save_checkpoint
    tr, th = _run(steps=3, dtype="bf16", model="lenet", algo="event", dataset="mnist") if False else _run(steps=3, dtype="bf16")
    path = ckpt_path(str(tmp_path), 0)
    save_checkpoint(path, epoch=1, arena=tr.arena, backend=tr.backend, model=tr.model)
    tr.arena.theta.add_(1.0)
    load_checkpoint(path, arena=tr.arena, backend=tr.backend, model=tr.model)
    torch.cuda.synchronize()
    assert torch.equal(tr.arena.theta, th)
    if tr.arena.shadow is not None:
        t = tr.arena.table
        assert torch.equal(tr.arena.flat(tr.arena.theta, 0).to(torch.bfloat16), tr.arena.shadow[:t.numels[0]])
    tr.close()


def test_native_loader_on_cuda_path():
    """--native-loader on: C++ prefetch thread (csrc/host_loader.h) feeding pinned slots + async H2D gives the same
    batches as the Python staging path."""
    from eventgrad_b200.data import BatchLoader, ShardSampler
    src = synthetic_source("cifar10", 1000).pin()
    a = BatchLoader(src, ShardSampler(1000, 1, 0, "sequential"), 64, "cuda", native="on")
    b = BatchLoader(src, ShardSampler(1000, 1, 0, "sequential"), 64, "cuda", native="off")
    assert a.native is not None
    for (xa, ya), (xb, yb) in zip(a, b):
        assert torch.equal(xa, xb) and torch.equal(ya, yb)


def test_p2p_file_write_logs(tmp_path):
    """Reference debug files (send<r>/recv<r>.txt, event.cpp:203-227) from the DEVICE log ring of the p2p backend
    (MNIST self-loop, 1 GPU): one row per step, 3 fields per tensor on the send side."""
    cfg = preset("mnist_event", backend="p2p", device="cuda", train_samples=640, test_samples=128, epochs=1,
                 quiet=True, file_write=1, log_dir=str(tmp_path))
    tr = Trainer(cfg, _env(), train_source=synthetic_source("mnist", 640).pin(),
                 test_source=synthetic_source("mnist", 128, train=False).pin())
    tr.fit()
    tr.finalize()
    send = open(tmp_path / "send0.txt").read().splitlines()
    recv = open(tmp_path / "recv0.txt").read().splitlines()
    assert len(send) == 10 and len(recv) == 10 and len(send[0].split(",  ")) == 8 * 3 + 1
    tr.close()


def test_gpu_defaults_are_the_fast_path_and_fp32_uses_fused_bn():
    """No execution flags: on a GPU the Trainer runs NHWC + whole-step CUDA graph; the fp32 activations go through
    the fused BN kernels (csrc/bn_act.cu instantiated for float) and the fp32 convolutions through the wgmma kernels
    (csrc/conv_tc.cu) -- counted through the extension's launch counter."""
    from eventgrad_b200.ops import ext
    C = ext()
    n0 = C.launch_count()
    tr, _ = _run(steps=6)                               # dtype defaults to fp32
    assert tr.cfg.dtype == "fp32" and tr.cfg.cuda_graph and tr.cfg.channels_last and tr.cfg.conv_tc
    assert len(tr._graphs) == 1
    per_step = tr.own_launches_per_step
    assert per_step.get("bn", 0) >= 4 * 13 and per_step.get("gossip", 0) >= 1, per_step
    assert per_step.get("conv", 0) >= 3 * 13, per_step      # every conv of the model: fprop + dgrad + wgrad (+ splits)
    assert C.launch_count() > n0
    tr.close()
