"""Chebyshev-accelerated gossip rounds (--gossip-accel chebyshev, decent on the ring / a static graph): the coefficients
against the graph's spectrum and the Chebyshev bound, the simulator (explicit mixes and combines, P_Q(W), average
preservation in fp32, bytes and messages), the gloo backend against the simulator bit for bit with a resume that
switches the flag (tests/chebyshev_worker.py), and the configuration rules."""
import math
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import TILE, ParamArena, TensorTable
from eventgrad_b200.parallel.topology import chebyshev_coefficients, circulant_spectrum, parse_topology
from eventgrad_b200.parallel.trigger import mix3_, mixk_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPT = dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=True)
CASES = [("ring", 2), ("ring", 3), ("ring", 5), ("ring", 8), ("exp", 4), ("exp", 8), ("1,3", 8)]


def _table():
    return ParamArena(build_model("cnn2"), torch.device("cpu")).table


def _small_table(sizes=(37, 300)):
    w = [torch.nn.Parameter(torch.zeros(n)) for n in sizes]
    return TensorTable.from_named([(f"w{i}", p) for i, p in enumerate(w)], TILE)


def _mask(t, dtype=torch.float32):
    m = torch.zeros(t.n_padded, dtype=dtype)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


def _grads(t, R, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    m = _mask(t, dtype)
    return [torch.randn(t.n_padded, generator=g, dtype=dtype) * 0.05 * m for _ in range(R)]


def _spread(sim, t, seed):
    gen = torch.Generator().manual_seed(seed)
    for th in sim.theta:
        th.add_(torch.randn(t.n_padded, generator=gen, dtype=th.dtype) * _mask(t, th.dtype))


def _plain_w(topology, R):
    t = _small_table()
    return RingSimulator(R, torch.zeros(t.n_padded), t, "decent", serial_skip=False, offsets=topology).mixing_matrix()


def _p_of(topology, R, Q, fp32):
    """P_Q(W) in float64 from the float64 or the fp32-rounded coefficients (the simulator's recurrence)."""
    t = _small_table()
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", serial_skip=False, offsets=topology,
                        gossip_rounds=Q, gossip_accel="chebyshev")
    sim.cheb_coef = chebyshev_coefficients(sim.offsets, R, Q, fp32=fp32)
    return sim.mixing_matrix()


def _dev_norm(M):
    R = M.shape[0]
    return float(torch.linalg.matrix_norm(M - torch.full((R, R), 1.0 / R, dtype=torch.float64), ord=2))


# ---------------------------------------------------------------------------------------- coefficients
@pytest.mark.parametrize("R", [4, 5, 6, 8, 16, 32])
@pytest.mark.parametrize("topology", ["ring", "exp", "1,3"])
def test_spectrum_is_the_plain_graphs(topology, R):
    """(a, b) of circulant_spectrum are the smallest and largest eigenvalues of mixing_matrix()'s W on 1^perp."""
    if topology == "1,3" and R < 6:
        pytest.skip("offset 3 needs R >= 6")
    ev = torch.linalg.eigvalsh(_plain_w(topology, R))
    i1 = int(torch.argmin((ev - 1.0).abs()))
    rest = torch.cat([ev[:i1], ev[i1 + 1:]])
    a, b = circulant_spectrum(parse_topology(topology, R), R)
    assert abs(a - float(rest.min())) < 1e-12 and abs(b - float(rest.max())) < 1e-12


def test_worked_examples():
    """The coefficients quoted in the docs: ring R = 8, Q = 3 and ring R = 5, Q = 2, and the one-point spectra."""
    got = chebyshev_coefficients((1,), 8, 3)
    for (al, om), (wa, wo) in zip(got, [(1.3084, 0.0), (1.8101, 0.3834), (1.6187, 0.2372)]):
        assert abs(al - wa) < 1e-4 and abs(om - wo) < 1e-4
    got = chebyshev_coefficients((1,), 5, 2)
    for (al, om), (wa, wo) in zip(got, [(1.2, 0.0), (4 / 3, 1 / 9)]):
        assert abs(al - wa) < 1e-6 and abs(om - wo) < 1e-6
    assert chebyshev_coefficients((1,), 2, 3) == [(0.75, 0.0)] * 3
    assert chebyshev_coefficients((1,), 3, 2) == [(1.0, 0.0)] * 2
    for al, om in chebyshev_coefficients((1, 2, 4), 32, 5):          # each value is an fp32
        assert torch.tensor(al, dtype=torch.float32).item() == al and torch.tensor(om, dtype=torch.float32).item() == om
    for bad in (0, -1, 1.5, True):
        with pytest.raises(ValueError):
            chebyshev_coefficients((1,), 8, bad)


@pytest.mark.parametrize("topology,R", [("ring", 4), ("ring", 5), ("ring", 8), ("ring", 16), ("ring", 32),
                                        ("exp", 8), ("exp", 32), ("1,3", 8), ("1,3", 16)])
@pytest.mark.parametrize("Q", [1, 2, 3, 4, 5, 6])
def test_contraction_is_one_over_t_q_of_mu(topology, R, Q):
    """float64 coefficients: ||P_Q(W) - 11^T/R||_2 = 1 / T_Q(mu) to 1e-12, never above W^Q's; P_Q(W) is symmetric with
    unit row sums."""
    a, b = circulant_spectrum(parse_topology(topology, R), R)
    c, d = (a + b) / 2, (b - a) / 2
    mu = (1 - c) / d
    P = _p_of(topology, R, Q, fp32=False)
    assert abs(_dev_norm(P) - 1.0 / math.cosh(Q * math.acosh(mu))) < 1e-12
    assert _dev_norm(P) <= _dev_norm(torch.linalg.matrix_power(_plain_w(topology, R), Q)) + 1e-12
    assert float((P - P.T).abs().max()) < 1e-12
    assert float((P.sum(1) - 1).abs().max()) < 1e-12


@pytest.mark.parametrize("topology,R,Q,power,cheb", [
    ("ring", 8, 1, 0.805, 0.745), ("ring", 8, 2, 0.648, 0.383), ("ring", 8, 3, 0.521, 0.177), ("ring", 8, 4, 0.419, 0.079),
    ("ring", 16, 2, 0.901, 0.752), ("ring", 16, 4, 0.812, 0.395), ("ring", 32, 4, 0.950, 0.754),
    ("exp", 8, 1, 0.429, 0.404), ("exp", 8, 2, 0.184, 0.089), ("exp", 32, 2, 0.478, 0.246), ("exp", 32, 3, 0.331, 0.088),
])
def test_the_documented_table(topology, R, Q, power, cheb):
    """The DESIGN table: ||W^Q|| and ||P_Q(W)|| on 1^perp (the simulator's P_Q(W), fp32 coefficients).  exp at R = 32 is
    offsets (1, 2, 4, 8): at most four offsets (degree <= 8)."""
    t = _small_table()
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", serial_skip=False, offsets=topology, gossip_rounds=Q,
                        gossip_accel="chebyshev")
    assert abs(_dev_norm(torch.linalg.matrix_power(_plain_w(topology, R), Q)) - power) < 5e-4
    assert abs(_dev_norm(sim.mixing_matrix()) - cheb) < 5e-4


@pytest.mark.parametrize("R", [2, 3])
def test_one_point_spectra_average_in_one_round(R):
    """Ring at R = 2 and 3: W's spectrum on 1^perp is one point, and one round (Q = 1, lr = 0) gives every rank the
    average to fp32 rounding."""
    t = _small_table()
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", lr=0.0, serial_skip=False, gossip_rounds=1,
                        gossip_accel="chebyshev")
    _spread(sim, t, R)
    avg = torch.stack(sim.theta).double().mean(0)
    sim.step([torch.zeros(t.n_padded) for _ in range(R)])
    for th in sim.theta:
        assert float((th.double() - avg).abs().max()) < 4e-7
    assert _dev_norm(sim.mixing_matrix()) < 1e-7


# ---------------------------------------------------------------------------------------- simulator
@pytest.mark.parametrize("topology,R", CASES)
@pytest.mark.parametrize("Q", [1, 2, 3])
def test_simulator_is_explicit_mixes_and_combines(topology, R, Q):
    """Q explicit rounds -- every rank's mix (mix3_ / mixk_) of everyone's x_{q-1}, then x + alpha (w - x) and, from
    q = 2, + omega (x - x_prev), each a separate rounded op -- followed by the serial SGD step (a simulator whose local
    steps never communicate) equal the Chebyshev step bit for bit: theta, momentum and bytes."""
    t = _table()
    table = torch.linspace(0.05, 0.01, 7)
    kw = dict(serial_skip=False, offsets=topology, lr_table=table, **OPT)
    a = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", gossip_rounds=Q, gossip_accel="chebyshev", **kw)
    b = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", local_steps=1000, **kw)
    _spread(a, t, R * 10 + Q)
    _spread(b, t, R * 10 + Q)
    coef = chebyshev_coefficients(parse_topology(topology, R), R, Q)
    graphs = a.graphs
    for k in range(1, 6):
        g = _grads(t, R, 40 + k)
        prev = None
        for q, (al, om) in enumerate(coef, 1):
            x = [th.clone() for th in b.theta]
            for r in range(R):
                ins = [x[p] for p in graphs[r].slots()]
                w = x[r].clone()
                if len(ins) == 2:
                    mix3_(w, ins[0], ins[1])
                else:
                    mixk_(w, ins)
                y = torch.add(x[r], torch.mul(torch.sub(w, x[r]), al))
                if q >= 2:
                    y = torch.add(y, torch.mul(torch.sub(x[r], prev[r]), om))
                b.theta[r].copy_(y)
            prev = x
        a.step(g)
        b.step(g)
        for r in range(R):
            assert torch.equal(a.theta[r], b.theta[r]) and torch.equal(a.mom[r], b.mom[r]), f"step {k} rank {r}"
            assert a.bytes[r] == k * Q * a.fanout * 4 * t.n_elems


@pytest.mark.parametrize("R,Q", [(8, 3), (32, 4)])
def test_average_is_preserved_in_fp32(R, Q):
    """lr = 0, fp32, unit-normal theta, 500 steps: the rank average moves by at most 1e-5 (the difference form keeps a
    consensus vector fixed whatever the rounding of the coefficients)."""
    t = _small_table((64, 100))
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", lr=0.0, serial_skip=False, gossip_rounds=Q,
                        gossip_accel="chebyshev")
    gen = torch.Generator().manual_seed(R + Q)
    m = _mask(t)
    for th in sim.theta:
        th.copy_(torch.randn(t.n_padded, generator=gen) * m)
    avg0 = torch.stack(sim.theta).double().mean(0)
    zeros = [torch.zeros(t.n_padded) for _ in range(R)]
    for _ in range(500):
        sim.step(zeros)
    assert float((torch.stack(sim.theta).double().mean(0) - avg0).abs().max()) <= 1e-5


@pytest.mark.parametrize("topology,R", [("ring", 8), ("exp", 8), ("1,3", 8)])
@pytest.mark.parametrize("Q", [1, 2, 3])
def test_no_learning_is_p_q_to_the_k(topology, R, Q):
    """lr = 0, float64: theta after K steps is P_Q(W)^K theta_0 to 1e-12."""
    t = _small_table()
    gen = torch.Generator().manual_seed(R * 10 + Q)
    m = _mask(t, torch.float64)
    th = torch.stack([torch.randn(t.n_padded, generator=gen, dtype=torch.float64) * m for _ in range(R)])
    sim = RingSimulator(R, th[0], t, "decent", lr=0.0, serial_skip=False, offsets=topology, gossip_rounds=Q,
                        gossip_accel="chebyshev")
    for r in range(R):
        sim.theta[r].copy_(th[r])
    P = sim.mixing_matrix()
    zeros = [torch.zeros(t.n_padded, dtype=torch.float64) for _ in range(R)]
    K = 4
    for _ in range(K):
        sim.step(zeros)
    assert float((torch.stack(sim.theta) - torch.linalg.matrix_power(P, K) @ th).abs().max()) < 1e-12


@pytest.mark.parametrize("topology", ["ring", "exp", "1,3"])
@pytest.mark.parametrize("Q", [1, 2, 3])
def test_bytes_and_messages_are_those_of_the_rounds(topology, Q):
    R, K = 8, 5
    t = _table()
    kw = dict(serial_skip=False, offsets=topology, gossip_rounds=Q)
    a = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", gossip_accel="chebyshev", **kw)
    b = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", **kw)
    for s in range(K):
        g = _grads(t, R, s)
        a.step(g)
        b.step(g)
    assert a.bytes == b.bytes == [K * Q * a.fanout * 4 * t.n_elems] * R
    assert a.dense_messages() == b.dense_messages()


def test_one_rank_runs_nothing_extra():
    t = _table()
    a = RingSimulator(1, torch.zeros(t.n_padded), t, "decent", gossip_rounds=3, gossip_accel="chebyshev", **OPT)
    b = RingSimulator(1, torch.zeros(t.n_padded), t, "decent", **OPT)
    for k in range(3):
        g = _grads(t, 1, k)
        a.step(g)
        b.step(g)
    assert torch.equal(a.theta[0], b.theta[0]) and a.bytes == b.bytes == [0]


@pytest.mark.parametrize("kw", [
    dict(algo="event"), dict(algo="spevent"), dict(algo="cent"), dict(compress="int8"),
    dict(gradient_tracking=True), dict(exact_diffusion=True), dict(local_steps=2), dict(offsets="onepeer-exp"),
    dict(offsets="random-match"), dict(global_avg_period=2), dict(quasi_global=True, momentum=0.9),
    dict(slowmo_period=2),
])
def test_simulator_rejects_what_validate_rejects(kw):
    t = _table()
    algo = kw.pop("algo", "decent")
    with pytest.raises(ValueError, match="chebyshev gossip"):
        RingSimulator(4, torch.zeros(t.n_padded), t, algo, gossip_accel="chebyshev", **kw)
    with pytest.raises(ValueError, match="gossip_accel"):
        RingSimulator(4, torch.zeros(t.n_padded), t, "decent", gossip_accel="polyak")


# ---------------------------------------------------------------------------------------- configuration
def _ch(**kw):
    base = dict(algo="decent", gossip_rounds=3, gossip_accel="chebyshev")
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("Q", [1, 3])
@pytest.mark.parametrize("kw,match", [
    (dict(algo="cent"), "needs algo decent"),
    (dict(algo="event"), "needs algo decent"),
    (dict(algo="spevent"), "needs algo decent"),
    (dict(topology="onepeer-exp"), "onepeer-exp"),
    (dict(topology="random-match"), "random-match"),
    (dict(compress="int8"), "int8"),
    (dict(gradient_tracking=True), "gradient-tracking"),
    (dict(exact_diffusion=True), "exact-diffusion"),
    (dict(local_steps=2), "local-steps 2"),
    (dict(global_avg_period=4), "global-avg-period"),
    (dict(slowmo_period=4), "slowmo-period"),
    (dict(quasi_global_momentum=True, momentum=0.9), "quasi-global-momentum"),
    (dict(backend="refport"), "refport"),
    (dict(overlap_push=True), "overlap_push"),
    (dict(ce_push=True), "ce_push"),
    (dict(file_write=1), "file_write"),
    (dict(double_buffer=True), "gossip-accel chebyshev does not support double_buffer"),
    (dict(gossip_accel="nesterov"), "gossip-accel must be one of none|chebyshev"),
])
def test_validation_rejects(kw, match, Q):
    """Every combination --gossip-rounds > 1 rejects, also at Q = 1; the time-varying graphs, an explicit double buffer
    and unknown names."""
    with pytest.raises(ValueError, match=match):
        _ch(gossip_rounds=Q, **kw).validate()


def test_validation_rejects_async():
    """async mode: rejected for decent by its lock-step rule, and by the flag for any other algorithm."""
    with pytest.raises(ValueError, match="sync_mode=iter"):
        _ch(sync_mode="async").validate()
    with pytest.raises(ValueError, match="gossip-accel chebyshev needs --sync-mode iter"):
        _ch(algo="event", sync_mode="async", gossip_rounds=1).validate()


def test_validation_accepts():
    for topo in ("ring", "1", "exp", "1,3", "2,3"):
        for Q in (1, 2, 3, 10):
            _ch(topology=topo, gossip_rounds=Q).validate()
    _ch(overlap_push=False, double_buffer=False, ce_push=False, backend="gloo").validate()
    _ch(backend="nccl", momentum=0.9, nesterov=True, weight_decay=5e-4, partition="label", consensus_every=1).validate()
    for algo in ("cent", "decent", "event", "spevent"):
        TrainConfig(algo=algo, gossip_accel="none").validate()          # off restricts nothing


def test_resolved_keeps_the_serial_step_and_no_overlap():
    from eventgrad_b200.parallel.p2p import _rounds_per_step, _wants_dbuf, _wants_rounds
    for Q in (1, 3):
        c = _ch(gossip_rounds=Q).validate().resolved("cuda", 8)
        assert c.overlap_push is False and not _wants_dbuf(c)          # the double-buffer default does not apply
        assert _rounds_per_step(c) == Q and _wants_rounds(c, 8) and not _wants_rounds(c, 1)
    c = _ch(topology="exp").validate().resolved("cuda", 8)
    assert c.overlap_push is False and c.topology == "exp"
    off = TrainConfig(algo="decent", gossip_rounds=3).validate()
    assert _rounds_per_step(off) == 2 and _wants_dbuf(off.resolved("cuda", 8))
    assert _rounds_per_step(TrainConfig(algo="decent").validate()) == 0
    assert TrainConfig(algo="decent", gossip_accel="none").validate().resolved("cuda", 4).overlap_push is True


def test_cli_and_presets():
    c = parse_cli("decent", ["--gossip-rounds", "3", "--gossip-accel", "chebyshev", "--topology", "exp"])
    assert c.gossip_rounds == 3 and c.gossip_accel == "chebyshev" and c.topology == "exp"
    c = parse_cli("decent", ["--gossip-accel", "chebyshev"])
    assert c.gossip_rounds == 1 and c.gossip_accel == "chebyshev"
    assert parse_cli("decent", []).gossip_accel == "none"
    for prog in ("mnist_event", "cent"):
        with pytest.raises(ValueError, match="gossip-accel"):
            parse_cli(prog, ["--gossip-accel", "chebyshev"])
    with pytest.raises(SystemExit):
        parse_cli("decent", ["--gossip-accel", "polyak"])
    assert all(preset(n).gossip_accel == "none" for n in PRESETS)
    assert all("gossip_accel" not in p for p in PRESETS.values())


def test_window_layout():
    """The flag off changes no layout; on, the round sections are appended (also at Q = 1) and the ring's step inboxes
    are single-slot (no double buffer)."""
    from eventgrad_b200.parallel.p2p import build_layout
    from eventgrad_b200.parallel.topology import Graph
    t = _table()
    for topo, g in (("ring", None), ("exp", Graph.build(0, 8, "exp"))):
        for extra in ({}, dict(consensus_every=1)):
            for Q in (1, 3):
                off = build_layout(t, TrainConfig(algo="decent", topology=topo, gossip_rounds=Q, gossip_accel="none",
                                                  **extra).validate(), 8, 528, g)
                dflt = build_layout(t, TrainConfig(algo="decent", topology=topo, gossip_rounds=Q, **extra).validate(),
                                    8, 528, g)
                assert off.sections == dflt.sections and off.size == dflt.size
                on = build_layout(t, _ch(topology=topo, gossip_rounds=Q, **extra).validate(), 8, 528, g)
                n = 2 if g is None else g.n_slots
                rounds = [k for k in on.sections if k.startswith("round_")]
                assert sorted(rounds) == sorted([f"round_inbox_{k}" for k in range(n)]
                                                + [f"round_flag_{k}" for k in range(n)]
                                                + [f"round_ack_{k}" for k in range(n)])
                assert list(on.sections)[-len(rounds):] == rounds
                if g is None:
                    assert on.sections["inbox_l"][1] == t.n_padded * 4      # one slot
            solo = build_layout(t, _ch(topology="ring", **extra).validate(), 1, 528, None)
            assert not any(k.startswith("round_") for k in solo.sections)


def test_checkpoints_gain_no_key():
    from eventgrad_b200.parallel import Ring
    from eventgrad_b200.parallel.collective import CollectiveBackend
    keys = []
    for accel in ("none", "chebyshev"):
        cfg = TrainConfig(algo="decent", device="cpu", backend="gloo", gossip_rounds=2, gossip_accel=accel).validate()
        be = CollectiveBackend(cfg, ParamArena(build_model("cnn2"), torch.device("cpu")), Ring(0, 1))
        keys.append(sorted(be.state_dict()))
    assert keys[0] == keys[1]


# ---------------------------------------------------------------------------------------- gloo
_PORT = [37900 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "chebyshev_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("Q", [1, 3])
@pytest.mark.parametrize("world,topology", [(2, "ring"), (3, "ring"), (4, "ring"), (5, "ring"), (4, "1,2")])
def test_gloo_matches_simulator(world, topology, Q):
    rc, out = _torchrun(world, "--mode", "sim", "--topology", topology, "--gossip-rounds", str(Q))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


@pytest.mark.parametrize("Q,A,Q2,A2", [(3, "chebyshev", 2, "none"), (3, "none", 2, "chebyshev"),
                                       (2, "chebyshev", 3, "chebyshev")])
def test_gloo_resume_switching_the_flag(Q, A, Q2, A2):
    rc, out = _torchrun(5, "--mode", "resume", "--gossip-rounds", str(Q), "--accel", A, "--resume-rounds", str(Q2),
                        "--resume-accel", A2)
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
