"""Several gossip rounds per D-PSGD step (--gossip-rounds Q, decent on the ring / a static graph): the simulator (Q - 1
explicit mixes followed by the unchanged step, W^Q, the lr = 0 spectral identity, bytes and messages), the gloo backend
against the simulator bit for bit, a resume under the same and another Q (tests/gossip_rounds_worker.py), and the
configuration rules."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import TILE, ParamArena, TensorTable
from eventgrad_b200.parallel.trigger import mix3_, mixk_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPT = dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=True)
CASES = [("ring", 2), ("ring", 3), ("ring", 4), ("exp", 4), ("exp", 8), ("1,3", 8)]


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
        th.add_(torch.randn(t.n_padded, generator=gen) * _mask(t))


# ---------------------------------------------------------------------------------------- simulator
@pytest.mark.parametrize("topology,R", CASES)
@pytest.mark.parametrize("Q", [2, 3])
def test_rounds_are_explicit_mixes_then_the_step(topology, R, Q):
    """Q - 1 explicit mixes of every rank's whole theta (mix3_ on the ring, mixk_ on a graph) followed by a plain decent
    step equal the Q-round step bit for bit: theta, momentum and bytes."""
    t = _table()
    table = torch.linspace(0.05, 0.01, 7)
    kw = dict(serial_skip=False, offsets=topology, lr_table=table, **OPT)
    a = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", gossip_rounds=Q, **kw)
    b = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", **kw)
    _spread(a, t, R * 10 + Q)
    _spread(b, t, R * 10 + Q)
    graphs = a.graphs
    for k in range(1, 6):
        g = _grads(t, R, 40 + k)
        for _ in range(Q - 1):
            snap = [x.clone() for x in b.theta]
            for r in range(R):
                ins = [snap[p] for p in graphs[r].slots()]
                if len(ins) == 2:
                    mix3_(b.theta[r], ins[0], ins[1])
                else:
                    mixk_(b.theta[r], ins)
        a.step(g)
        b.step(g)
        for r in range(R):
            assert torch.equal(a.theta[r], b.theta[r]) and torch.equal(a.mom[r], b.mom[r]), f"step {k} rank {r}"
            assert a.bytes[r] == Q * b.bytes[r]
    assert a.dense_messages() == Q * b.dense_messages()


@pytest.mark.parametrize("topology,R", CASES)
@pytest.mark.parametrize("Q", [2, 3])
def test_no_learning_is_w_to_the_qk(topology, R, Q):
    """lr = 0, float64: mixing_matrix() is W^Q and theta after K steps is W^(QK) theta_0 to 1e-12."""
    t = _small_table()
    gen = torch.Generator().manual_seed(R * 10 + Q)
    m = _mask(t, torch.float64)
    th = torch.stack([torch.randn(t.n_padded, generator=gen, dtype=torch.float64) * m for _ in range(R)])
    sim = RingSimulator(R, th[0], t, "decent", lr=0.0, serial_skip=False, offsets=topology, gossip_rounds=Q)
    plain = RingSimulator(R, th[0], t, "decent", lr=0.0, serial_skip=False, offsets=topology)
    for r in range(R):
        sim.theta[r].copy_(th[r])
    W = plain.mixing_matrix()
    assert torch.allclose(sim.mixing_matrix(), torch.linalg.matrix_power(W, Q), rtol=0, atol=1e-15)
    zeros = [torch.zeros(t.n_padded, dtype=torch.float64) for _ in range(R)]
    K = 4
    for _ in range(K):
        sim.step(zeros)
    want = torch.linalg.matrix_power(W, Q * K) @ th
    assert float((torch.stack(sim.theta) - want).abs().max()) < 1e-12


@pytest.mark.parametrize("topology,R", [("ring", 1), ("ring", 4), ("exp", 8)])
def test_one_round_is_the_plain_step(topology, R):
    t = _table()
    kw = dict(serial_skip=False, offsets=topology, **OPT)
    a = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", gossip_rounds=1, **kw)
    b = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", **kw)
    for k in range(4):
        g = _grads(t, R, k)
        a.step(g)
        b.step(g)
    assert all(torch.equal(x, y) for x, y in zip(a.theta, b.theta)) and a.bytes == b.bytes
    assert torch.equal(a.mixing_matrix(), b.mixing_matrix())


def test_one_rank_runs_nothing_extra():
    t = _table()
    a = RingSimulator(1, torch.zeros(t.n_padded), t, "decent", gossip_rounds=3, **OPT)
    b = RingSimulator(1, torch.zeros(t.n_padded), t, "decent", **OPT)
    for k in range(3):
        g = _grads(t, 1, k)
        a.step(g)
        b.step(g)
    assert torch.equal(a.theta[0], b.theta[0]) and a.bytes == b.bytes == [0]


@pytest.mark.parametrize("topology", ["ring", "exp", "1,3"])
@pytest.mark.parametrize("Q", [1, 2, 3])
def test_bytes_and_messages(topology, Q):
    R, K = 8, 5
    t = _table()
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", serial_skip=False, offsets=topology, gossip_rounds=Q)
    for s in range(K):
        sim.step(_grads(t, R, s))
    assert sim.bytes == [K * Q * sim.fanout * 4 * t.n_elems] * R
    assert sim.dense_messages() == Q * sim.fanout * t.n_tensors * K * R


def test_matched_bytes_ring_q3_and_exp_q1():
    """At R = 8 the ring with Q = 3 and the exp graph (offsets 1, 2, 4) with Q = 1 send the same bytes per step."""
    t = _table()
    a = RingSimulator(8, torch.zeros(t.n_padded), t, "decent", serial_skip=False, gossip_rounds=3)
    b = RingSimulator(8, torch.zeros(t.n_padded), t, "decent", serial_skip=False, offsets="exp")
    g = _grads(t, 8, 0)
    a.step(g)
    b.step(g)
    assert a.bytes == b.bytes


@pytest.mark.parametrize("kw", [
    dict(algo="event"), dict(algo="spevent"), dict(algo="cent"), dict(compress="int8"),
    dict(gradient_tracking=True), dict(exact_diffusion=True), dict(local_steps=2), dict(offsets="onepeer-exp"),
    dict(global_avg_period=2), dict(quasi_global=True, momentum=0.9), dict(slowmo_period=2),
])
def test_simulator_rejects_what_validate_rejects(kw):
    t = _table()
    algo = kw.pop("algo", "decent")
    with pytest.raises(ValueError, match="gossip rounds"):
        RingSimulator(4, torch.zeros(t.n_padded), t, algo, gossip_rounds=2, **kw)
    for bad in (0, -1, 2.5, True):
        with pytest.raises(ValueError, match="gossip_rounds"):
            RingSimulator(4, torch.zeros(t.n_padded), t, "decent", gossip_rounds=bad)


# ---------------------------------------------------------------------------------------- configuration
def _gr(**kw):
    base = dict(algo="decent", gossip_rounds=3)
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("kw,match", [
    (dict(algo="cent"), "gossip-rounds 3 needs algo decent"),
    (dict(algo="event"), "gossip-rounds 3 needs algo decent.*trigger"),
    (dict(algo="spevent"), "gossip-rounds 3 needs algo decent.*trigger"),
    (dict(topology="onepeer-exp"), "gossip-rounds.*onepeer-exp"),
    (dict(compress="int8"), "gossip-rounds.*int8"),
    (dict(gradient_tracking=True), "gossip-rounds.*gradient-tracking"),
    (dict(exact_diffusion=True), "gossip-rounds.*exact-diffusion"),
    (dict(local_steps=2), "gossip-rounds.*local-steps 2"),
    (dict(global_avg_period=4), "gossip-rounds.*global-avg-period"),
    (dict(slowmo_period=4), "gossip-rounds.*slowmo-period"),
    (dict(quasi_global_momentum=True, momentum=0.9), "gossip-rounds.*quasi-global-momentum.*overwritten"),
    (dict(backend="refport"), "gossip-rounds.*refport"),
    (dict(overlap_push=True), "gossip-rounds.*overlap_push.*backward"),
    (dict(ce_push=True), "gossip-rounds.*ce_push"),
    (dict(file_write=1), "gossip-rounds.*file_write"),
    (dict(gossip_rounds=0), "gossip-rounds must be an integer >= 1"),
    (dict(gossip_rounds=-2), "gossip-rounds must be"),
    (dict(gossip_rounds=2.0), "gossip-rounds must be"),
    (dict(gossip_rounds=True), "gossip-rounds must be"),
])
def test_validation_rejects(kw, match):
    with pytest.raises(ValueError, match=match):
        _gr(**kw).validate()


def test_validation_accepts():
    for topo in ("ring", "1", "exp", "1,3", "2,3"):
        for Q in (1, 2, 3, 10):
            _gr(topology=topo, gossip_rounds=Q).validate()
    _gr(overlap_push=False, double_buffer=True, ce_push=False, backend="gloo", local_steps=1).validate()
    _gr(double_buffer=False, backend="nccl", momentum=0.9, nesterov=True, weight_decay=5e-4, partition="label",
        consensus_every=1).validate()
    for algo in ("cent", "decent", "event", "spevent"):
        TrainConfig(algo=algo, gossip_rounds=1).validate()           # Q = 1 restricts nothing


def test_resolved_keeps_the_fused_step_and_no_overlap():
    from eventgrad_b200.parallel.p2p import _wants_dbuf
    c = _gr().validate().resolved("cuda", 8)
    assert c.overlap_push is False and _wants_dbuf(c)              # the rounds run ahead of the double-buffered step
    assert not _wants_dbuf(_gr(double_buffer=False).validate().resolved("cuda", 8))
    c = _gr(topology="exp").validate().resolved("cuda", 8)
    assert c.overlap_push is False and c.topology == "exp"
    assert TrainConfig(algo="decent").validate().resolved("cuda", 4).overlap_push is True
    assert TrainConfig(algo="decent", gossip_rounds=1).validate().resolved("cuda", 4).overlap_push is True


def test_cli_and_presets():
    c = parse_cli("decent", ["--gossip-rounds", "3", "--topology", "exp"])
    assert c.gossip_rounds == 3 and c.topology == "exp"
    assert parse_cli("decent", []).gossip_rounds == 1
    for prog in ("mnist_event", "cent"):
        with pytest.raises(ValueError, match="gossip-rounds"):
            parse_cli(prog, ["--gossip-rounds", "2"])
    with pytest.raises(SystemExit):
        parse_cli("decent", ["--gossip-rounds", "2.5"])
    assert all(preset(n).gossip_rounds == 1 for n in PRESETS)
    assert all("gossip_rounds" not in p for p in PRESETS.values())


def test_window_layout_is_unchanged_without_rounds():
    """Q = 1 adds no window section; Q > 1 appends its sections after every existing one."""
    from eventgrad_b200.parallel.p2p import build_layout
    from eventgrad_b200.parallel.topology import Graph
    t = _table()
    for topo, g in (("ring", None), ("exp", Graph.build(0, 8, "exp"))):
        for extra in ({}, dict(consensus_every=1)):
            base = build_layout(t, _gr(topology=topo, gossip_rounds=1, **extra).validate(), 8, 528, g)
            one = build_layout(t, TrainConfig(algo="decent", topology=topo, **extra).validate(), 8, 528, g)
            assert base.sections == one.sections and base.size == one.size
            more = build_layout(t, _gr(topology=topo, **extra).validate(), 8, 528, g)
            n = 2 if g is None else g.n_slots
            assert list(more.sections)[:len(base.sections)] == list(base.sections)
            assert all(more.sections[k] == v for k, v in base.sections.items())
            added = list(more.sections)[len(base.sections):]
            assert sorted(added) == sorted([f"round_inbox_{k}" for k in range(n)] + [f"round_flag_{k}" for k in range(n)]
                                           + [f"round_ack_{k}" for k in range(n)])
            # one rank: nothing is allocated
            solo = build_layout(t, _gr(topology="ring", **extra).validate(), 1, 528, None)
            assert not any(k.startswith("round_") for k in solo.sections)


def test_checkpoints_gain_no_key():
    from eventgrad_b200.parallel import Ring
    from eventgrad_b200.parallel.collective import CollectiveBackend
    keys = []
    for Q in (1, 3):
        cfg = TrainConfig(algo="decent", device="cpu", backend="gloo", gossip_rounds=Q).validate()
        be = CollectiveBackend(cfg, ParamArena(build_model("cnn2"), torch.device("cpu")), Ring(0, 1))
        keys.append(sorted(be.state_dict()))
    assert keys[0] == keys[1]


# ---------------------------------------------------------------------------------------- gloo
_PORT = [37300 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "gossip_rounds_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("Q", [2, 3])
@pytest.mark.parametrize("world,topology", [(2, "ring"), (3, "ring"), (4, "ring"), (4, "1,2")])
def test_gloo_matches_simulator(world, topology, Q):
    rc, out = _torchrun(world, "--mode", "sim", "--topology", topology, "--gossip-rounds", str(Q))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


@pytest.mark.parametrize("Q,Q2", [(3, 3), (3, 2), (2, 1)])
def test_gloo_resume_is_exact_also_under_another_q(Q, Q2):
    rc, out = _torchrun(3, "--mode", "resume", "--gossip-rounds", str(Q), "--resume-rounds", str(Q2))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
