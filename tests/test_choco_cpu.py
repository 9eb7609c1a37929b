"""The 1-bit scaled-sign codec (--compress sign) and the CHOCO mix (--choco-gamma): the codec against numpy with an
explicit xor tree (parallel/trigger.py sign_encode / sign_decode), its contraction and message size, the simulator's
average preservation, consensus and fixed point in float64, the gloo backend against the simulator bit for bit
(tests/choco_worker.py), checkpoint guards, and the configuration rules."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import ParamArena, TensorTable
from eventgrad_b200.parallel.base import check_choco_state
from eventgrad_b200.parallel.trigger import (Q8_BLOCK, TriggerConfig, choco_mix_, consensus_stats, consensus_values,
                                             q8_msg_bytes, sign_decode, sign_encode, sign_msg_bytes)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _small_table():
    """Two tensors whose last tiles are partial: 100 and 300 elements in tiles of 2048."""
    return TensorTable.from_named([("a", torch.empty(100)), ("b", torch.empty(300))])


def _mask(t, dtype=torch.float32):
    m = torch.zeros(t.n_padded, dtype=dtype)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


def _np_sign_encode(d):
    """The codec in numpy, lane by lane: left-to-right lane sums, then the butterfly a[j] + a[j ^ o] written out."""
    b = d.numpy().reshape(-1, 32, 8)
    dt = b.dtype.type
    a = np.zeros(b.shape[:2], dtype=b.dtype)
    for e in range(8):
        a = (a + np.abs(b[:, :, e])).astype(b.dtype)
    for o in (16, 8, 4, 2, 1):
        a = np.stack([a[:, j] + a[:, j ^ o] for j in range(32)], axis=1).astype(b.dtype)
    assert (a == a[:, :1]).all() or np.isnan(a).any()
    s = (a[:, 0] / dt(256.0)).astype(b.dtype)
    bits = np.zeros(b.shape[:2], dtype=np.uint8)
    for e in range(8):
        bits |= ((b[:, :, e] < 0).astype(np.uint8) << e)
    return bits.reshape(-1), s


# ---------------------------------------------------------------------------------------- codec
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_sign_codec_matches_numpy_xor_tree(dtype):
    g = torch.Generator().manual_seed(3)
    d = (torch.randn(64 * Q8_BLOCK, generator=g, dtype=torch.float64)
         * torch.logspace(-30, 30, 64, dtype=torch.float64).repeat_interleave(Q8_BLOCK)).to(dtype)
    bits, s = sign_encode(d)
    bn, sn = _np_sign_encode(d)
    assert bits.dtype == torch.uint8 and bits.numel() == d.numel() // 8 and s.dtype == dtype and s.numel() == 64
    assert np.array_equal(bits.numpy(), bn) and np.array_equal(s.numpy(), sn)
    deq = sign_decode(bits, s)
    want = torch.where(d < 0, -s.repeat_interleave(Q8_BLOCK), s.repeat_interleave(Q8_BLOCK))
    assert torch.equal(deq, want)


def test_sign_codec_zero_block_and_signed_zeros():
    d = torch.zeros(3 * Q8_BLOCK)
    d[Q8_BLOCK:Q8_BLOCK + 4] = torch.tensor([0.0, -0.0, 0.0, -0.0])
    d[2 * Q8_BLOCK + 7] = -2.0
    bits, s = sign_encode(d)
    assert s.tolist() == [0.0, 0.0, 2.0 / 256]
    assert int(bits[:64].sum()) == 0                            # +0 and -0 both send bit 0
    deq = sign_decode(bits, s)
    assert bool((deq[:2 * Q8_BLOCK] == 0).all())
    assert float(deq[2 * Q8_BLOCK + 7]) == -2.0 / 256 and float(deq[2 * Q8_BLOCK]) == 2.0 / 256


def test_sign_codec_subnormal_and_underflowing_scale():
    d = torch.zeros(2 * Q8_BLOCK)
    d[3] = -3e-38                                              # a / 256 is subnormal
    d[Q8_BLOCK + 5] = 1e-45                                    # a / 256 rounds to zero
    bits, s = sign_encode(d)
    assert 0.0 < float(s[0]) < torch.finfo(torch.float32).tiny
    assert float(s[1]) == 0.0
    assert float(sign_decode(bits, s)[3]) == -float(s[0])


def test_sign_codec_padding_and_tensor_boundaries():
    """On an arena the blocks are the tiles' warp slices: a block never straddles two tensors, and the zero padding of
    a partial tile encodes to zero blocks."""
    t = _small_table()
    m = _mask(t)
    g = torch.Generator().manual_seed(4)
    d = torch.randn(t.n_padded, generator=g) * m
    bits, s = sign_encode(d)
    for o, n, c in zip(t.offsets, t.numels, t.tile_count):
        first, last = o // Q8_BLOCK, (o + c * t.tile) // Q8_BLOCK
        full = -(-n // Q8_BLOCK)
        assert bool((s[first:first + full] > 0).all()) and bool((s[first + full:last] == 0).all())
        # encoding one tensor alone gives the same bytes and scales as the whole arena
        b1, s1 = sign_encode(d[o:o + c * t.tile])
        assert torch.equal(b1, bits[o // 8:(o + c * t.tile) // 8]) and torch.equal(s1, s[first:last])
    for o, n, c in zip(t.offsets, t.numels, t.tile_count):
        span = slice(o, o + c * t.tile)
        deq = sign_decode(bits[o // 8:(o + c * t.tile) // 8], s[o // Q8_BLOCK:(o + c * t.tile) // Q8_BLOCK], n)
        assert bool((deq[n:] == 0).all()) and torch.equal(deq[:n], sign_decode(bits, s)[span][:n])


def test_sign_codec_contraction():
    """Per block, ||d - deq||^2 = ||d||^2 - (sum |d|)^2 / 256 <= (1 - 1/256) ||d||^2 in float64: the scaled sign is a
    contractive compressor, the property CHOCO's convergence proof needs."""
    g = torch.Generator().manual_seed(5)
    shapes = [torch.randn(200 * Q8_BLOCK, generator=g, dtype=torch.float64),
              torch.randn(200 * Q8_BLOCK, generator=g, dtype=torch.float64) ** 5,
              torch.zeros(200 * Q8_BLOCK, dtype=torch.float64).index_fill_(0, torch.arange(0, 200 * Q8_BLOCK, 97), 1.0)]
    for d in shapes:
        e = (d - sign_decode(*sign_encode(d))).view(-1, Q8_BLOCK).square().sum(1)
        n = d.view(-1, Q8_BLOCK).square().sum(1)
        assert bool((e <= (1 - 1 / 256) * n * (1 + 1e-12)).all())


def test_sign_msg_bytes_resnet18():
    assert sign_msg_bytes(1) == 5 and sign_msg_bytes(8) == 5 and sign_msg_bytes(9) == 6
    assert sign_msg_bytes(256) == 36 and sign_msg_bytes(257) == 41
    t = ParamArena(build_model("resnet18"), torch.device("cpu")).table
    assert t.n_tensors == 86
    dense = 2 * sum(4 * n for n in t.numels)
    int8 = 2 * sum(q8_msg_bytes(n) for n in t.numels)
    sign = 2 * sum(sign_msg_bytes(n) for n in t.numels)
    assert (dense, int8, sign) == (139_557_456, 35_434_660, 4_906_468)     # per rank and step, every tensor fired


# ---------------------------------------------------------------------------------------- the CHOCO mix
def test_choco_mix_op_order():
    g = torch.Generator().manual_seed(6)
    th, pv, l, r = (torch.randn(4096, generator=g) for _ in range(4))
    want = th.numpy() + np.float32(0.3) * ((((pv.numpy() + l.numpy()) + r.numpy()) / np.float32(3)) - pv.numpy())
    got = choco_mix_(th.clone(), pv, l, r, 0.3)
    assert np.array_equal(got.numpy(), want.astype(np.float32))


# ---------------------------------------------------------------------------------------- simulator, float64
def _spread_sim(R, compress, gamma, seed=1, **kw):
    t = _small_table()
    m = _mask(t, torch.float64)
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(t.n_padded, generator=g, dtype=torch.float64) * m for _ in range(R)]
    sim = RingSimulator(R, xs[0], t, "decent", lr=0.0, serial_skip=False, compress=compress, choco_gamma=gamma, **kw)
    for r in range(R):
        sim.theta[r] = xs[r].clone()
    return sim, xs, [torch.zeros(t.n_padded, dtype=torch.float64) for _ in range(R)]


@pytest.mark.parametrize("compress", ["int8", "sign"])
@pytest.mark.parametrize("R", [2, 3, 4, 5, 8])
def test_choco_keeps_the_sum(R, compress):
    """lr = 0 from a spread start: sum_r theta_r stays where it started to 1e-12 relative, step after step, whatever
    the codec (sum_r (W prev - prev)_r = 0 for the doubly stochastic ring)."""
    sim, xs, zero = _spread_sim(R, compress, 0.5)
    s0 = torch.stack(xs).sum(0)
    for _ in range(200):
        sim.step(zero)
        assert float((torch.stack(sim.theta).sum(0) - s0).norm() / s0.norm()) < 1e-12


def test_choco_sign_reaches_consensus_at_the_initial_mean():
    """sign with gamma = 0.2 at R = 3: 1500 steps take the consensus distance from about 34 to about 1e-2 (the float64
    model's rate at this gamma), at the initial mean.  The consensus rows the simulator records every 100 steps agree
    with consensus_stats and shrink."""
    sim, xs, zero = _spread_sim(3, "sign", 0.2, consensus_every=100)
    mean0 = torch.stack(xs).mean(0)
    d0, _ = consensus_values(*consensus_stats(xs, sim.table), 3)
    for _ in range(1500):
        sim.step(zero)
    X = torch.stack(sim.theta)
    assert float((X.mean(0) - mean0).abs().max()) < 1e-12
    d, _ = consensus_values(*consensus_stats(sim.theta, sim.table), 3)
    assert d < 1e-3 * d0, (d, d0)
    rows = [consensus_values(D, A, 3)[0] for _, D, A in sim.consensus]
    assert [k for k, _, _ in sim.consensus] == list(range(100, 1501, 100))
    assert rows[-1] == d and all(b < a for a, b in zip(rows, rows[1:]))


@pytest.mark.parametrize("R", [3, 4])
def test_error_feedback_mix_with_sign_moves_the_mean(R):
    """Today's mix ((theta + rep_l) + rep_r) / 3 with the sign codec moves the average by the codec's residual: after
    300 steps at lr = 0 the mean is far from where it started (CHOCO keeps it, above)."""
    sim, xs, zero = _spread_sim(R, "sign", 0.0)
    mean0 = torch.stack(xs).mean(0)
    for _ in range(300):
        sim.step(zero)
    assert float((torch.stack(sim.theta).mean(0) - mean0).abs().max()) > 0.1


@pytest.mark.parametrize("compress,steps", [("int8", 500), ("sign", 3500)])
def test_choco_fixed_point_is_dpsgd_at_lr_over_gamma(compress, steps):
    """Heterogeneous quadratics f_r = a_r / 2 ||x - c_r||^2 at R = 4, lr = 0.05, gamma = 0.5: at a fixed point prev = theta,
    so CHOCO settles where plain D-PSGD at lr / gamma does, the solution of (W - I) x = (lr / gamma) a (x - c).  The
    float64 model reaches it to 2e-15 (int8, 500 steps) and 4e-11 (sign, 3500 steps; about 10x per 500 steps); the
    tolerance is 1e-9."""
    R, lr, gamma = 4, 0.05, 0.5
    t = _small_table()
    m = _mask(t, torch.float64)
    g = torch.Generator().manual_seed(0)
    a = torch.rand(R, generator=g, dtype=torch.float64) * 1.5 + 0.5
    c = [torch.randn(t.n_padded, generator=g, dtype=torch.float64) * m for _ in range(R)]
    W = torch.zeros(R, R, dtype=torch.float64)
    for r in range(R):
        for q in (r - 1, r, r + 1):
            W[r, q % R] += 1 / 3
    h = lr / gamma
    fixed = torch.linalg.solve(W - torch.eye(R, dtype=torch.float64) - h * torch.diag(a), -h * a[:, None] * torch.stack(c))
    sim = RingSimulator(R, torch.zeros(t.n_padded, dtype=torch.float64), t, "decent", lr=lr, serial_skip=False,
                        compress=compress, choco_gamma=gamma)
    for _ in range(steps):
        sim.step([a[r] * (sim.theta[r] - c[r]) for r in range(R)])
    assert float((torch.stack(sim.theta) - fixed).abs().max()) < 1e-9


@pytest.mark.parametrize("algo", ["decent", "event"])
@pytest.mark.parametrize("R", [2, 3, 5])
def test_simulator_replica_invariant_events_and_bytes(R, algo):
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    m = _mask(t)
    g = torch.Generator().manual_seed(R)
    theta0 = torch.randn(t.n_padded, generator=g) * m * 0.1
    sim = RingSimulator(R, theta0, t, algo, TriggerConfig(initial_comm_passes=3), lr=0.05, momentum=0.9,
                        serial_skip=False, compress="sign", choco_gamma=0.5)
    events, nbytes = [0] * R, [0] * R
    for s in range(10):
        sim.step([torch.randn(t.n_padded, generator=g) * 0.05 * m for _ in range(R)])
        for r in range(R):
            L, Rn = (r - 1) % R, (r + 1) % R
            assert torch.equal(sim.rep_r[L], sim.prev[r]) and torch.equal(sim.rep_l[Rn], sim.prev[r]), (s, r)
            fired = sim.fire_history[-1][r]
            events[r] += 2 * int(fired.sum()) if algo == "event" else 0
            nbytes[r] += sum(2 * sign_msg_bytes(t.numels[i]) for i in range(t.n_tensors) if fired[i])
        assert sim.events == events and sim.bytes == nbytes
    for r in range(R):
        assert bool((sim.prev[r][m == 0] == 0).all())
    if algo == "event":
        assert 0 < sum(int(f.sum()) for h in sim.fire_history for f in h) < 10 * R * t.n_tensors


def test_simulator_gamma_zero_is_the_int8_run():
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    m = _mask(t)
    g = torch.Generator().manual_seed(2)
    theta0 = torch.randn(t.n_padded, generator=g) * m
    a = RingSimulator(3, theta0, t, "event", TriggerConfig(initial_comm_passes=2), lr=0.05, serial_skip=False,
                      compress="int8")
    b = RingSimulator(3, theta0, t, "event", TriggerConfig(initial_comm_passes=2), lr=0.05, serial_skip=False,
                      compress="int8", choco_gamma=0.0)
    for s in range(5):
        gr = [torch.randn(t.n_padded, generator=g) * m for _ in range(3)]
        a.step(gr)
        b.step(gr)
    assert all(torch.equal(x, y) for x, y in zip(a.theta, b.theta)) and a.bytes == b.bytes


@pytest.mark.parametrize("kw,match", [(dict(choco_gamma=0.5), "int8 or sign"), (dict(choco_gamma=1.5), "choco_gamma"),
                                      (dict(compress="sign", choco_gamma=-0.1), "choco_gamma"),
                                      (dict(compress="sign", choco_gamma=True), "choco_gamma"),
                                      (dict(compress="sign", choco_gamma="0.5"), "choco_gamma")])
def test_simulator_rejects(kw, match):
    t = _small_table()
    with pytest.raises(ValueError, match=match):
        RingSimulator(2, torch.zeros(t.n_padded), t, "decent", **kw)


# ---------------------------------------------------------------------------------------- configuration
@pytest.mark.parametrize("kw,match", [
    (dict(choco_gamma=-0.1), "choco-gamma"),
    (dict(choco_gamma=1.01), "small gamma"),
    (dict(choco_gamma=float("nan")), "choco-gamma"),
    (dict(choco_gamma=True), "choco-gamma"),
    (dict(choco_gamma="0.5"), "choco-gamma"),
    (dict(compress="none", choco_gamma=0.5), "needs --compress"),
    (dict(algo="cent"), "decent or event"),
    (dict(algo="spevent"), "spevent"),
    (dict(topology="2"), "ring"),
    (dict(sync_mode="async"), "iter"),
    (dict(backend="refport"), "refport"),
    (dict(overlap_push=True), "overlap_push"),
    (dict(algo="decent", double_buffer=True), "double_buffer"),
    (dict(ce_push=True), "ce_push"),
    (dict(file_write=1), "file_write"),
    (dict(algo="decent", gradient_tracking=True), "compress sign"),
    (dict(algo="decent", exact_diffusion=True), "compress sign"),
    (dict(algo="decent", local_steps=2), "compress sign"),
    (dict(algo="decent", global_avg_period=2), "compress sign"),
    (dict(momentum=0.9, quasi_global_momentum=True), "compress sign"),
    (dict(algo="decent", slowmo_period=2), "compress sign"),
])
def test_validation_rejects(kw, match):
    base = dict(algo="event", compress="sign", choco_gamma=0.2)
    base.update(kw)
    with pytest.raises(ValueError, match=match):
        TrainConfig(**base).validate()


def test_validation_accepts_and_resolves():
    for compress in ("int8", "sign"):
        for gamma in (0.0, 0.2, 1.0, 1):
            c = TrainConfig(algo="decent", compress=compress, choco_gamma=gamma).validate()
            r = c.resolved("cuda", 4)
            assert r.choco_gamma == gamma and r.compress == compress and r.overlap_push is False
    with pytest.raises(ValueError, match="ring"):
        TrainConfig(algo="event", compress="sign", topology="exp").validate().for_world(4)


def test_cli_and_presets():
    for prog in ("decent", "mnist_event", "cifar_event"):
        c = parse_cli(prog, ["--compress", "sign", "--choco-gamma", "0.2"])
        assert c.compress == "sign" and c.choco_gamma == 0.2
        assert parse_cli(prog, []).choco_gamma == 0.0
    assert all(preset(name).choco_gamma == 0.0 for name in PRESETS)
    assert TrainConfig().choco_gamma == 0.0


def test_check_choco_state():
    check_choco_state({}, 0.0, "event")
    check_choco_state({"choco_gamma": 0.5}, 0.5, "decent")
    check_choco_state({"choco_gamma": 0.5}, 0.0, "spevent")        # no compression state there
    with pytest.raises(ValueError, match="choco-gamma"):
        check_choco_state({}, 0.5, "event")
    with pytest.raises(ValueError, match="choco-gamma"):
        check_choco_state({"choco_gamma": 0.5}, 0.2, "decent")
    with pytest.raises(ValueError, match="choco-gamma"):
        check_choco_state({"choco_gamma": 0.5}, 0.0, "decent")


# ---------------------------------------------------------------------------------------- gloo
_PORT = [35300 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "choco_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("algo,trigger", [("decent", "norm"), ("event", "norm"), ("event", "drift")])
@pytest.mark.parametrize("compress,gamma", [("sign", "0.5"), ("sign", "0"), ("int8", "0.2")])
def test_gloo_matches_simulator(world, algo, trigger, compress, gamma):
    rc, out = _torchrun(world, "--mode", "sim", "--algo", algo, "--trigger", trigger, "--compress", compress,
                        "--gamma", gamma, "--steps", "9")
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_resume_is_exact_and_refuses_other_gamma_or_codec(tmp_path):
    rc, out = _torchrun(3, "--mode", "resume", "--ckpt-dir", str(tmp_path), "--compress", "sign", "--gamma", "0.5")
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
