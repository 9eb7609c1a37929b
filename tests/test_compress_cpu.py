"""int8 error-feedback compression (--compress int8): the codec (parallel/trigger.py q8_encode / q8_decode), the
simulator's replica invariant, counters and consensus, the gloo backend against the simulator bit for bit
(tests/compress_worker.py), checkpoint resume, and the configuration rules."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import TILE, ParamArena
from eventgrad_b200.parallel.base import check_compress_state
from eventgrad_b200.parallel.trigger import Q8_BLOCK, TriggerConfig, q8_decode, q8_encode, q8_msg_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _table(model="cnn2"):
    return ParamArena(build_model(model), torch.device("cpu")).table


def _mask(t):
    m = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


def _np_encode(d):
    """The codec in numpy float32, element by element as the kernel computes it."""
    b = d.numpy().astype(np.float32).reshape(-1, Q8_BLOCK)
    a = np.abs(b).max(axis=1)
    s = (a / np.float32(127.0)).astype(np.float32)
    q = np.zeros_like(b)
    nz = s != 0
    q[nz] = np.clip(np.rint(b[nz] / s[nz, None]), -127, 127)
    return q.astype(np.int8).reshape(-1), s


# ---------------------------------------------------------------------------------------- codec
def test_codec_matches_numpy_and_error_bound():
    g = torch.Generator().manual_seed(3)
    d = torch.randn(64 * Q8_BLOCK, generator=g) * torch.logspace(-30, 30, 64).repeat_interleave(Q8_BLOCK)
    q, s = q8_encode(d)
    qn, sn = _np_encode(d)
    assert q.dtype == torch.int8 and s.dtype == torch.float32 and s.numel() == 64
    assert np.array_equal(q.numpy(), qn) and np.array_equal(s.numpy(), sn)
    deq = q8_decode(q, s)
    assert torch.equal(deq, (q.float().view(-1, Q8_BLOCK) * s[:, None]).view(-1))
    err = (deq - d).abs().view(-1, Q8_BLOCK)
    assert bool((err <= s[:, None] / 2 * (1 + 1e-6)).all())


def test_codec_zero_block_and_block_maximum():
    d = torch.zeros(3 * Q8_BLOCK)
    d[Q8_BLOCK + 5] = -2.5
    d[Q8_BLOCK + 9] = 1.0
    d[2 * Q8_BLOCK + 17] = 7.0
    q, s = q8_encode(d)
    assert s[0] == 0 and bool((q[:Q8_BLOCK] == 0).all())
    assert q[Q8_BLOCK + 5] == -127 and q[2 * Q8_BLOCK + 17] == 127
    assert s[1] == torch.tensor(2.5) / torch.tensor(127.0)
    assert torch.equal(q8_decode(q, s)[:Q8_BLOCK], torch.zeros(Q8_BLOCK))


def test_codec_ties_round_to_even():
    # s = 127 / 127 = 1 exactly, so d / s is d: the halves round to the even neighbour
    d = torch.zeros(Q8_BLOCK)
    d[0] = 127.0
    halves = [0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 126.5]
    d[1:1 + len(halves)] = torch.tensor(halves)
    q, s = q8_encode(d)
    assert s[0] == 1.0
    assert q[1:1 + len(halves)].tolist() == [0, 2, 2, 0, -2, -2, 126]


def test_codec_subnormal_and_underflowing_scale():
    tiny = torch.tensor(1e-45)                      # the smallest subnormal: a / 127 underflows to 0
    d = torch.zeros(2 * Q8_BLOCK)
    d[3] = tiny
    d[Q8_BLOCK + 1] = torch.tensor(1e-38)           # a / 127 is a (non-zero) subnormal scale
    d[Q8_BLOCK + 2] = torch.tensor(-3e-39)
    q, s = q8_encode(d)
    assert s[0] == 0 and bool((q[:Q8_BLOCK] == 0).all())
    assert 0 < s[1] < torch.finfo(torch.float32).tiny
    qn, sn = _np_encode(d)
    assert np.array_equal(q.numpy(), qn) and np.array_equal(s.numpy(), sn)
    assert q[Q8_BLOCK + 1] == 127


def test_codec_padding_and_tensor_boundaries():
    t = _table()
    g = torch.Generator().manual_seed(5)
    theta = torch.randn(t.n_padded, generator=g) * _mask(t)
    q, s = q8_encode(theta)
    pad = _mask(t) == 0
    assert bool((q[pad] == 0).all())
    # every tensor's blocks encode alone: the last (partial) tile of tensor i is independent of tensor i + 1
    for i in range(t.n_tensors):
        o, n = t.offsets[i], t.tile_count[i] * TILE
        qi, si = q8_encode(theta[o:o + n])
        assert torch.equal(qi, q[o:o + n]) and torch.equal(si, s[o // Q8_BLOCK:(o + n) // Q8_BLOCK])


def test_error_feedback_converges_on_a_fixed_theta():
    g = torch.Generator().manual_seed(9)
    theta = torch.randn(16 * Q8_BLOCK, generator=g)
    prev = torch.zeros_like(theta)
    err = (theta - prev).norm().item()
    for _ in range(6):
        prev = prev + q8_decode(*q8_encode(theta - prev))
        new = (theta - prev).norm().item()
        floor = 4 * torch.finfo(torch.float32).eps * theta.norm().item()
        assert new <= max(err / 100, floor), (err, new)
        err = new
    assert err <= 4 * torch.finfo(torch.float32).eps * theta.norm().item()


def test_msg_bytes_formula():
    assert q8_msg_bytes(1) == 5 and q8_msg_bytes(256) == 260 and q8_msg_bytes(257) == 265
    t = _table("resnet18")
    dense = sum(4 * n for n in t.numels)
    q8 = sum(q8_msg_bytes(n) for n in t.numels)
    assert 3.9 < dense / q8 < 4.0


# ---------------------------------------------------------------------------------------- simulator
def _sim(t, R, algo, theta0, **kw):
    return RingSimulator(R, theta0, t, algo, TriggerConfig(initial_comm_passes=3), lr=0.05, momentum=0.9,
                         serial_skip=False, compress="int8", **kw)


@pytest.mark.parametrize("R", [2, 3, 4, 5])
@pytest.mark.parametrize("algo", ["decent", "event"])
def test_simulator_replica_invariant_and_counters(R, algo):
    t = _table()
    m = _mask(t)
    g = torch.Generator().manual_seed(R)
    theta0 = torch.randn(t.n_padded, generator=g) * m * 0.1
    sim = _sim(t, R, algo, theta0)
    events = [0] * R
    nbytes = [0] * R
    for s in range(12):
        sim.step([torch.randn(t.n_padded, generator=g) * 0.05 * m for _ in range(R)])
        for r in range(R):
            L, Rn = (r - 1) % R, (r + 1) % R
            assert torch.equal(sim.rep_r[L], sim.prev[r]) and torch.equal(sim.rep_l[Rn], sim.prev[r]), (s, r)
            fired = sim.fire_history[-1][r]
            events[r] += 2 * int(fired.sum()) if algo == "event" else 0
            nbytes[r] += sum(2 * q8_msg_bytes(t.numels[i]) for i in range(t.n_tensors) if fired[i])
        assert sim.events == events and sim.bytes == nbytes
    for r in range(R):
        assert bool((sim.prev[r][m == 0] == 0).all())
    if algo == "event":
        assert 0 < sum(int(f.sum()) for h in sim.fire_history for f in h) < 12 * R * t.n_tensors


def test_simulator_drift_sent_is_prev():
    t = _table()
    sim = RingSimulator(3, torch.zeros(t.n_padded), t, "event", TriggerConfig(metric="drift"), compress="int8")
    assert sim.sent is sim.prev


@pytest.mark.parametrize("R", [2, 3, 4, 5])
def test_simulator_decent_lr0_reaches_consensus(R):
    t = _table()
    m = _mask(t)
    g = torch.Generator().manual_seed(11)
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", lr=0.0, serial_skip=False, compress="int8")
    for r in range(R):
        sim.theta[r] = torch.randn(t.n_padded, generator=g) * m
    zero = [torch.zeros(t.n_padded) for _ in range(R)]

    def spread():
        bar = sim.final_average()
        return max((th - bar).abs().max().item() for th in sim.theta)

    s0 = spread()
    for _ in range(60):
        sim.step(zero)
    assert spread() < s0 * 1e-4, (s0, spread())


def test_simulator_none_is_unchanged():
    t = _table()
    m = _mask(t)
    g = torch.Generator().manual_seed(2)
    theta0 = torch.randn(t.n_padded, generator=g) * m
    a = RingSimulator(3, theta0, t, "event", TriggerConfig(initial_comm_passes=2), lr=0.05, serial_skip=False)
    b = RingSimulator(3, theta0, t, "event", TriggerConfig(initial_comm_passes=2), lr=0.05, serial_skip=False,
                      compress="none")
    for s in range(5):
        gr = [torch.randn(t.n_padded, generator=g) * m for _ in range(3)]
        a.step(gr)
        b.step(gr)
    assert all(torch.equal(x, y) for x, y in zip(a.theta, b.theta)) and a.bytes == b.bytes
    assert not hasattr(b, "prev")


# ---------------------------------------------------------------------------------------- configuration
def _int8(**kw):
    base = dict(algo="event", compress="int8")
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("kw,match", [
    (dict(algo="cent"), "decent or event"),
    (dict(algo="spevent"), "spevent"),
    (dict(topology="2"), "ring"),
    (dict(topology="1,2"), "ring"),
    (dict(sync_mode="async"), "iter"),
    (dict(backend="refport"), "refport"),
    (dict(overlap_push=True), "overlap_push"),
    (dict(algo="decent", double_buffer=True), "double_buffer"),
    (dict(ce_push=True), "ce_push"),
    (dict(file_write=1), "file_write"),
    (dict(compress="int4"), "compress"),
])
def test_validation_rejects(kw, match):
    with pytest.raises(ValueError, match=match):
        _int8(**kw).validate()


@pytest.mark.parametrize("topology,world,ok", [("exp", 2, True), ("exp", 3, True), ("exp", 4, False),
                                               ("onepeer-exp", 1, True), ("onepeer-exp", 2, False),
                                               ("ring", 8, True)])
def test_topology_names_that_resolve_to_the_ring(topology, world, ok):
    cfg = _int8(topology=topology).validate()
    if ok:
        assert cfg.for_world(world).ring_topology
    else:
        with pytest.raises(ValueError, match="ring"):
            cfg.for_world(world)
        with pytest.raises(ValueError, match="ring"):
            cfg.resolved("cuda", world)


def test_resolved_keeps_the_fused_step():
    from eventgrad_b200.parallel.p2p import _wants_dbuf
    for algo in ("decent", "event"):
        c = _int8(algo=algo).validate().resolved("cuda", 4)
        assert c.overlap_push is False and not _wants_dbuf(c)
    assert TrainConfig(algo="decent").validate().resolved("cuda", 4).overlap_push is True


def test_cli_and_presets():
    for prog in ("decent", "mnist_event", "cifar_event"):
        assert parse_cli(prog, ["--compress", "int8"]).compress == "int8"
        assert parse_cli(prog, []).compress == "none"
    assert all(preset(name).compress == "none" for name in PRESETS)
    assert TrainConfig().compress == "none"


def test_check_compress_state():
    check_compress_state({}, "none", "event")
    check_compress_state({"compress": "int8"}, "int8", "decent")
    check_compress_state({"compress": "int8"}, "none", "spevent")      # no compression state there
    with pytest.raises(ValueError, match="compress"):
        check_compress_state({}, "int8", "event")
    with pytest.raises(ValueError, match="compress"):
        check_compress_state({"compress": "int8"}, "none", "decent")


# ---------------------------------------------------------------------------------------- gloo
_PORT = [33300 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "compress_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("algo,trigger", [("decent", "norm"), ("event", "norm"), ("event", "drift")])
def test_gloo_matches_simulator(world, algo, trigger):
    rc, out = _torchrun(world, "--mode", "sim", "--algo", algo, "--trigger", trigger, "--steps", "9")
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_resume_is_exact_and_refuses_dense(tmp_path):
    rc, out = _torchrun(3, "--mode", "resume", "--ckpt-dir", str(tmp_path))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
