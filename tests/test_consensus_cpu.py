"""CPU: the consensus distance (--consensus-every N) -- the oracle parallel/trigger.py:consensus_stats against numpy,
its closed forms, the simulator's measurements (read-only, and the spectral identity of gossip at lr = 0), every
configuration rule, and the gloo backend and the Trainer on real process groups (tests/consensus_worker.py)."""
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import TILE, ParamArena, TensorTable
from eventgrad_b200.parallel.trigger import TriggerConfig, consensus_stats, consensus_values, rank_mean

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _table(sizes=(37, 300, 2049, 1)):
    w = [torch.nn.Parameter(torch.zeros(n)) for n in sizes]
    return TensorTable.from_named([(f"w{i}", p) for i, p in enumerate(w)], TILE)


def _mask(t, dtype=torch.float32):
    m = torch.zeros(t.n_padded, dtype=dtype)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


def _thetas(t, R, seed, dtype=torch.float32, pad=0.0):
    """R different arenas; `pad` fills the padding, which the statistics must ignore."""
    g = torch.Generator().manual_seed(seed)
    m = _mask(t, dtype)
    return [torch.randn(t.n_padded, generator=g, dtype=dtype) * m + pad * (1 - m) for _ in range(R)]


# ---------------------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("R", [1, 2, 3, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_matches_numpy_float64(R, dtype):
    """theta_bar is rank_mean in the arenas' dtype; the differences, squares and sums are float64 over the real elements
    only, the partial last tiles included (padding filled with garbage here)."""
    t = _table()
    th = _thetas(t, R, 3 + R, dtype, pad=123.0)
    D, A = consensus_stats(th, t)
    assert D.dtype == A.dtype == torch.float64 and D.shape == (t.n_tensors,)
    bar = rank_mean(th).numpy().astype(np.float64)
    xs = [x.numpy().astype(np.float64) for x in th]
    for i, (o, n) in enumerate(zip(t.offsets, t.numels)):
        a = bar[o:o + n]
        assert A[i].item() == pytest.approx(float(np.sum(a * a)), rel=1e-13)
        want = sum(float(np.sum((x[o:o + n] - a) ** 2)) for x in xs)
        assert D[i].item() == pytest.approx(want, rel=1e-12, abs=1e-300)


@pytest.mark.parametrize("R", [2, 3, 5, 8])
def test_identical_ranks_give_zero(R):
    """Integer-valued parameters keep every partial sum of the rank-order mean exact, so theta_bar is theta itself.  (In
    general ((x + x) + x) / 3 can differ from x in the last bit, and D is then of the order of the rounding.)"""
    t = _table()
    th = torch.round(_thetas(t, 1, 5)[0] * 100)
    D, A = consensus_stats([th.clone() for _ in range(R)], t)
    assert torch.equal(D, torch.zeros_like(D)) and bool((A > 0).all())
    assert consensus_values(D, A, R) == (0.0, 0.0)


def test_two_ranks_closed_form():
    """R = 2: D_i = ||a_i - b_i||^2 / 2 (float64 arenas, where the mean is exact up to the last bit)."""
    t = _table()
    a, b = _thetas(t, 2, 9, torch.float64)
    D, _ = consensus_stats([a, b], t)
    for i, (o, n) in enumerate(zip(t.offsets, t.numels)):
        assert D[i].item() == pytest.approx(float((a[o:o + n] - b[o:o + n]).square().sum()) / 2, rel=1e-12)


def test_values_are_design_definition():
    t = _table()
    th = _thetas(t, 4, 11, torch.float64)
    D, A = consensus_stats(th, t)
    d, rel = consensus_values(D, A, 4)
    m = _mask(t, torch.float64).bool()
    bar = torch.stack(th).mean(0)
    want = float(torch.stack([(x - bar)[m].square().sum() for x in th]).mean().sqrt())
    assert d == pytest.approx(want, rel=1e-12)
    assert rel == pytest.approx(want / float(bar[m].norm()), rel=1e-12)


# ---------------------------------------------------------------------------------------- the simulator
def _sim(R, t, algo="decent", N=1, dtype=torch.float32, lr=0.05, **kw):
    theta0 = torch.randn(t.n_padded, generator=torch.Generator().manual_seed(1), dtype=dtype) * _mask(t, dtype)
    return RingSimulator(R, theta0, t, algo, lr=lr, momentum=kw.pop("momentum", 0.9), serial_skip=False,
                         consensus_every=N, tcfg=kw.pop("tcfg", TriggerConfig(initial_comm_passes=2)), **kw)


def _spread(sim, t, seed):
    g = torch.Generator().manual_seed(seed)
    for th in sim.theta:
        th.add_(torch.randn(t.n_padded, generator=g, dtype=th.dtype) * _mask(t, th.dtype))


def _grads(t, R, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(t.n_padded, generator=g, dtype=dtype) * 0.05 * _mask(t, dtype) for _ in range(R)]


def test_lr_zero_right_after_a_global_average_is_exactly_zero():
    t = _table()
    sim = _sim(4, t, N=1, lr=0.0, global_avg_period=2, momentum=0.0)
    _spread(sim, t, 2)
    for s in range(4):
        sim.step(_grads(t, 4, s))
    (k1, D1, _), (k2, D2, _) = sim.consensus[0], sim.consensus[1]
    assert (k1, k2) == (1, 2) and float(D1.sum()) > 0 and torch.equal(D2, torch.zeros_like(D2))


@pytest.mark.parametrize("topology,R", [("ring", 5), ("exp", 8), ("onepeer-exp", 8), ("onepeer-exp", 6)])
def test_lr_zero_gossip_is_the_spectral_identity(topology, R):
    """float64, lr = 0: theta_k = W_k ... W_1 Theta_0, so sum_i D_i = ||(W_k ... W_1 - 11^T / R) Theta_0||_F^2."""
    t = _table((37, 300))
    sim = _sim(R, t, N=1, dtype=torch.float64, lr=0.0, momentum=0.0, offsets=topology)
    _spread(sim, t, 4)
    m = _mask(t, torch.float64).bool()
    theta0 = torch.stack([th[m] for th in sim.theta])
    P = torch.eye(R, dtype=torch.float64)
    J = torch.full((R, R), 1.0 / R, dtype=torch.float64)
    start = float(((torch.eye(R, dtype=torch.float64) - J) @ theta0).square().sum())
    for k in range(1, 9):
        P = sim.mixing_matrix(k) @ P
        sim.step([torch.zeros(t.n_padded, dtype=torch.float64)] * R)
        want = float(((P - J) @ theta0).square().sum())
        # (the one-peer graph at R = 2^m reaches the exact average after m rounds: want is then 0 up to rounding)
        assert float(sim.consensus[-1][1].sum()) == pytest.approx(want, rel=1e-10, abs=1e-24 * start)
        if k == 1:
            assert 0 < want < start


FEATURES = [("decent", "ring", {}), ("decent", "exp", {}), ("decent", "onepeer-exp", {}), ("event", "ring", {}),
            ("event", "exp", {}), ("spevent", "ring", {}), ("event", "ring", dict(compress="int8")),
            ("decent", "ring", dict(gradient_tracking=True)), ("decent", "ring", dict(exact_diffusion=True)),
            ("decent", "onepeer-exp", dict(local_steps=2)), ("decent", "exp", dict(global_avg_period=3)),
            ("event", "ring", dict(quasi_global=True)), ("decent", "ring", dict(slowmo_period=3)),
            ("decent", "ring", dict(slowmo_period=2, local_steps=2)),
            ("event", "ring", dict(tcfg=TriggerConfig(initial_comm_passes=2, metric="drift")))]


@pytest.mark.parametrize("algo,topology,kw", FEATURES)
def test_measurement_is_read_only(algo, topology, kw):
    """Every training quantity is bit for bit what it is without the flag; the measurements land at N | k only."""
    t = _table((37, 300, 2049))
    R, N = 4, 3
    sims = [_sim(R, t, algo, n, offsets=topology, **dict(kw)) for n in (0, N)]
    for s in sims:
        _spread(s, t, 7)
    for k in range(10):
        g = _grads(t, R, 50 + k)
        for s in sims:
            s.step(g)
    a, b = sims
    for r in range(R):
        assert torch.equal(a.theta[r], b.theta[r]) and torch.equal(a.mom[r], b.mom[r])
    assert a.events == b.events and a.bytes == b.bytes and a.consensus == []
    assert [k for k, _, _ in b.consensus] == [3, 6, 9]
    for k, D, A in b.consensus:
        assert D.dtype == torch.float64 and float(D.sum()) > 0 and float(A.sum()) > 0


def test_one_rank_records_zeros():
    t = _table()
    sim = _sim(1, t, N=2)
    for k in range(4):
        sim.step(_grads(t, 1, k))
    assert [k for k, _, _ in sim.consensus] == [2, 4]
    assert all(float(D.abs().sum()) == 0 for _, D, _ in sim.consensus)


def test_simulator_rejects():
    t = _table()
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError, match="consensus_every"):
            _sim(2, t, N=bad)
    with pytest.raises(ValueError, match="cent"):
        _sim(2, t, "cent", N=1)


# ---------------------------------------------------------------------------------------- configuration
def _c(**kw):
    base = dict(algo="decent", dataset="mnist", model="cnn2", sync_mode="iter", consensus_every=5)
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("kw,match", [
    (dict(consensus_every=-1), "--consensus-every"), (dict(consensus_every=2.0), "--consensus-every"),
    (dict(consensus_every=True), "--consensus-every"), (dict(consensus_every="3"), "--consensus-every"),
    (dict(algo="cent"), "--consensus-every 5"), (dict(algo="event", sync_mode="async"), "--consensus-every 5"),
    (dict(algo="spevent", sync_mode="async"), "--consensus-every 5"), (dict(backend="refport"), "--consensus-every 5"),
])
def test_validation_rejects(kw, match):
    with pytest.raises(ValueError, match=match):
        _c(**kw).validate()


@pytest.mark.parametrize("kw", [
    dict(), dict(algo="event"), dict(algo="spevent"), dict(topology="exp"), dict(topology="onepeer-exp"),
    dict(topology="1,3"), dict(algo="event", compress="int8"), dict(gradient_tracking=True),
    dict(exact_diffusion=True), dict(local_steps=4), dict(global_avg_period=3),
    dict(quasi_global_momentum=True, momentum=0.9), dict(slowmo_period=3, momentum=0.9, lr=0.1),
    dict(slowmo_period=3, local_steps=3, lr=0.1), dict(overlap_push=True), dict(double_buffer=True),
    dict(overlap_push=True, ce_push=True), dict(algo="event", file_write=1), dict(dtype="bf16"),
    dict(dtype="tf32"), dict(grad_table=False), dict(algo="event", trigger="drift"), dict(consensus_every=0),
    dict(consensus_every=0, algo="cent"), dict(consensus_every=0, algo="event", sync_mode="async"),
])
def test_validation_accepts(kw):
    _c(**kw).validate()


@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("dev", ["cuda", "cpu"])
@pytest.mark.parametrize("algo,kw", [("decent", {}), ("event", {}), ("decent", dict(topology="exp")),
                                     ("decent", dict(global_avg_period=2))])
def test_resolved_changes_no_default(world, dev, algo, kw):
    a = _c(algo=algo, consensus_every=0, **kw).validate().resolved(dev, world)
    b = _c(algo=algo, consensus_every=3, **kw).validate().resolved(dev, world)
    assert dataclasses.replace(b, consensus_every=0) == a


def test_cli_and_presets():
    assert all(TrainConfig(**p).consensus_every == 0 for p in PRESETS.values())
    assert TrainConfig().consensus_every == 0
    assert parse_cli("cifar_event", ["--consensus-every", "50"]).consensus_every == 50
    assert parse_cli("decent", []).consensus_every == 0
    with pytest.raises(ValueError, match="cent"):
        parse_cli("cent", ["--consensus-every", "1"])
    with pytest.raises(ValueError, match="--consensus-every"):
        parse_cli("mnist_event", ["--consensus-every", "-2"])


def test_p2p_window_layout_unchanged_without_the_flag():
    """The partial buffer is the window's last section and exists only with the flag on and peers to measure."""
    from eventgrad_b200.parallel.p2p import build_layout
    from eventgrad_b200.parallel.topology import Graph
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    for topology in ("ring", "exp"):
        g = None if topology == "ring" else Graph.build(0, 8, topology)
        off = build_layout(t, _c(consensus_every=0, topology=topology).validate().for_world(8), 8, 64, g)
        on = build_layout(t, _c(topology=topology).validate().for_world(8), 8, 64, g)
        assert list(off.sections.items()) == list(on.sections.items())[:len(off.sections)]
        assert list(on.sections)[-1] == "cons_part" and "cons_part" not in off.sections
        assert on.nbytes("cons_part") == t.n_tiles * 8 * 2 * 8
    assert "cons_part" not in build_layout(t, _c().validate(), 1, 64).sections


# ---------------------------------------------------------------------------------------- gloo
_PORT = [38600 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "consensus_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("world,algo,topology,feature", [
    (2, "decent", "ring", "plain"), (3, "event", "ring", "plain"), (4, "spevent", "ring", "plain"),
    (4, "decent", "exp", "plain"), (4, "decent", "onepeer-exp", "local"), (3, "event", "ring", "int8"),
    (3, "decent", "ring", "gt"), (2, "decent", "ring", "ed"), (4, "decent", "exp", "pga"),
    (3, "event", "ring", "qg"), (4, "decent", "ring", "slowmo")])
def test_gloo_matches_simulator(world, algo, topology, feature):
    rc, out = _torchrun(world, "--mode", "sim", "--algo", algo, "--topology", topology, "--feature", feature)
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_csv_results_and_resume(tmp_path):
    rc, out = _torchrun(2, "--mode", "trainer", "--log-dir", str(tmp_path / "log"), "--ckpt-dir", str(tmp_path / "ck"))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
    assert "Consensus distance in epoch 1 - " in out and "Consensus distance in epoch 2 - " in out
