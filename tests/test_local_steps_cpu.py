"""Periodic gossip (--local-steps H, decent): the simulator (H = 1 is the plain simulator bit for bit; without learning
theta follows the product of the rounds' mixing matrices and the one-peer graph reaches the exact average after tau * H
steps; the local steps are each rank's serial SGD; bytes count at the rounds only), the gloo backend against the
simulator bit for bit and a mid-cycle Trainer resume (tests/local_steps_worker.py), and the configuration rules."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import TILE, ParamArena, TensorTable
from eventgrad_b200.parallel.base import check_local_steps_state
from eventgrad_b200.parallel.trigger import sgd_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOPOLOGIES = ["ring", "exp", "onepeer-exp"]


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


OPT = dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=True)


# ---------------------------------------------------------------------------------------- simulator
@pytest.mark.parametrize("topology", TOPOLOGIES)
@pytest.mark.parametrize("R", [4, 5])
def test_h1_is_the_plain_simulator(topology, R):
    t = _table()
    theta0 = torch.randn(t.n_padded, generator=torch.Generator().manual_seed(1)) * _mask(t)
    table = torch.linspace(0.05, 0.01, 7)
    a = RingSimulator(R, theta0, t, "decent", serial_skip=False, offsets=topology, lr_table=table, **OPT)
    b = RingSimulator(R, theta0, t, "decent", serial_skip=False, offsets=topology, lr_table=table, local_steps=1, **OPT)
    for s in range(9):
        assert torch.equal(a.mixing_matrix(), b.mixing_matrix())
        g = _grads(t, R, 10 + s)
        a.step(g)
        b.step(g)
        for r in range(R):
            assert torch.equal(a.theta[r], b.theta[r]) and torch.equal(a.mom[r], b.mom[r])
            for x, y in zip(a.inbox[r], b.inbox[r]):
                assert torch.equal(x, y)
    assert a.bytes == b.bytes and a.dense_messages() == b.dense_messages()


@pytest.mark.parametrize("H", [2, 3, 4])
@pytest.mark.parametrize("topology,R", [("ring", 3), ("ring", 5), ("exp", 8), ("1,3", 8), ("onepeer-exp", 4),
                                        ("onepeer-exp", 6), ("onepeer-exp", 8)])
def test_no_learning_follows_the_product_of_round_matrices(topology, R, H):
    """lr = 0, float64: theta_K = W_K ... W_1 theta_0 with W = I at local steps and the round's matrix at the others."""
    t = _small_table()
    gen = torch.Generator().manual_seed(R * 10 + H)
    m = _mask(t, torch.float64)
    th = torch.stack([torch.randn(t.n_padded, generator=gen, dtype=torch.float64) * m for _ in range(R)])
    sim = RingSimulator(R, th[0], t, "decent", lr=0.0, serial_skip=False, offsets=topology, local_steps=H)
    for r in range(R):
        sim.theta[r].copy_(th[r])
    P = torch.eye(R, dtype=torch.float64)
    zeros = [torch.zeros(t.n_padded, dtype=torch.float64) for _ in range(R)]
    for k in range(1, 4 * H + 2):
        W = sim.mixing_matrix()
        assert torch.equal(W, torch.eye(R, dtype=torch.float64)) == (k % H != 0), k
        assert torch.allclose(W.sum(1), torch.ones(R, dtype=torch.float64))
        P = W @ P
        sim.step(zeros)
        want = P @ th
        got = torch.stack(sim.theta)
        assert float((got - want).abs().max()) < 1e-12, f"step {k}"


@pytest.mark.parametrize("H", [1, 2, 3])
@pytest.mark.parametrize("R", [4, 8])
def test_onepeer_exact_average_after_tau_rounds(R, H):
    """Integer theta, no learning: the one-peer graph (slot indexed by round) holds the exact mean after tau * H steps,
    and not one step earlier."""
    t = _small_table()
    tau = (R - 1).bit_length()
    m = _mask(t, torch.float64)
    gen = torch.Generator().manual_seed(R + H)
    th = [torch.randint(-64, 64, (t.n_padded,), generator=gen).double() * m for _ in range(R)]
    sim = RingSimulator(R, th[0], t, "decent", lr=0.0, serial_skip=False, offsets="onepeer-exp", local_steps=H)
    for r in range(R):
        sim.theta[r].copy_(th[r])
    mean = torch.stack(th).mean(0)
    zeros = [torch.zeros(t.n_padded, dtype=torch.float64) for _ in range(R)]
    for k in range(1, tau * H + 1):
        sim.step(zeros)
        same = all(torch.equal(x, mean) for x in sim.theta)
        assert same == (k == tau * H), f"step {k}"


@pytest.mark.parametrize("topology", TOPOLOGIES)
def test_local_steps_are_serial_sgd(topology):
    """Between rounds each rank runs sgd_ on its own theta and momentum; the inboxes keep the last round's values."""
    R, H = 4, 3
    t = _table()
    theta0 = torch.randn(t.n_padded, generator=torch.Generator().manual_seed(3)) * _mask(t)
    table = torch.linspace(0.05, 0.02, 12)
    sim = RingSimulator(R, theta0, t, "decent", serial_skip=False, offsets=topology, local_steps=H, lr_table=table,
                        **OPT)
    for k in range(1, 10):
        g = _grads(t, R, 50 + k)
        before = [(x.clone(), mo.clone()) for x, mo in zip(sim.theta, sim.mom)]
        inb = [[x.clone() for x in ib] for ib in sim.inbox]
        sim.step(g)
        if k % H == 0:
            continue
        for r in range(R):
            th, mo = before[r]
            sgd_(th, g[r], mo, float(table[k - 1]), OPT["momentum"], OPT["weight_decay"], OPT["nesterov"])
            assert torch.equal(sim.theta[r], th) and torch.equal(sim.mom[r], mo), f"step {k} rank {r}"
            assert all(torch.equal(x, y) for x, y in zip(sim.inbox[r], inb[r]))


@pytest.mark.parametrize("topology", TOPOLOGIES)
@pytest.mark.parametrize("H", [1, 2, 3, 8])
def test_bytes_count_the_rounds_only(topology, H):
    R, K = 4, 13
    t = _table()
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", serial_skip=False, offsets=topology, local_steps=H)
    for s in range(K):
        sim.step(_grads(t, R, s))
    assert sim.bytes == [(K // H) * sim.fanout * 4 * t.n_elems] * R
    assert sim.dense_messages() == sim.fanout * t.n_tensors * K * R        # per-step definition, unchanged


@pytest.mark.parametrize("kw", [dict(algo="event"), dict(algo="spevent"), dict(algo="cent"), dict(compress="int8"),
                                dict(gradient_tracking=True)])
def test_simulator_rejects_what_validate_rejects(kw):
    t = _table()
    algo = kw.pop("algo", "decent")
    with pytest.raises(ValueError, match="local steps"):
        RingSimulator(4, torch.zeros(t.n_padded), t, algo, local_steps=2, **kw)
    for bad in (0, -1, 1.5):
        with pytest.raises(ValueError, match="local_steps"):
            RingSimulator(4, torch.zeros(t.n_padded), t, "decent", local_steps=bad)


# ---------------------------------------------------------------------------------------- configuration
def _ls(**kw):
    base = dict(algo="decent", local_steps=4)
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("kw,match", [
    (dict(algo="cent"), "all-reduce"),
    (dict(algo="event"), "trigger"),
    (dict(algo="spevent"), "trigger"),
    (dict(gradient_tracking=True), "gradient-tracking"),
    (dict(compress="int8"), "int8"),
    (dict(backend="refport"), "refport"),
    (dict(overlap_push=True), "overlap_push"),
    (dict(double_buffer=True), "double_buffer"),
    (dict(ce_push=True), "ce_push"),
    (dict(file_write=1), "file_write"),
    (dict(local_steps=0), "local-steps"),
    (dict(local_steps=-2), "local-steps"),
    (dict(local_steps=2.5), "local-steps"),
])
def test_validation_rejects(kw, match):
    with pytest.raises(ValueError, match=match):
        _ls(**kw).validate()


def test_validation_accepts():
    for topo in ("ring", "exp", "1,3", "onepeer-exp"):
        _ls(topology=topo).validate()
    _ls(overlap_push=False, double_buffer=False, ce_push=False, backend="gloo").validate()
    for algo in ("cent", "decent", "event", "spevent"):
        TrainConfig(algo=algo, local_steps=1).validate()      # H = 1 restricts nothing


def test_resolved_keeps_the_fused_single_slot_step():
    from eventgrad_b200.parallel.p2p import _wants_dbuf
    for topo in ("ring", "exp", "onepeer-exp"):
        c = _ls(topology=topo).validate().resolved("cuda", 8)
        assert c.overlap_push is False and not _wants_dbuf(c)
    c = TrainConfig(algo="decent", local_steps=1).validate().resolved("cuda", 4)
    assert c.overlap_push is True
    assert _wants_dbuf(TrainConfig(algo="decent", overlap_push=False, local_steps=1).validate())


def test_cli_and_presets():
    c = parse_cli("decent", ["--local-steps", "4", "--topology", "onepeer-exp"])
    assert c.local_steps == 4 and c.topology == "onepeer-exp"
    assert parse_cli("decent", []).local_steps == 1
    with pytest.raises(ValueError, match="local-steps"):
        parse_cli("mnist_event", ["--local-steps", "2"])
    with pytest.raises(ValueError, match="local-steps"):
        parse_cli("cent", ["--local-steps", "2"])
    assert all(preset(n).local_steps == 1 for n in PRESETS)


def test_check_local_steps_state():
    check_local_steps_state({}, 1, "decent")                     # no key: every step gossiped
    check_local_steps_state({"local_steps": 4}, 4, "decent")
    check_local_steps_state({}, 4, "event")                      # only decent carries the period
    with pytest.raises(ValueError, match="local-steps"):
        check_local_steps_state({}, 4, "decent")
    with pytest.raises(ValueError, match="local-steps 4"):
        check_local_steps_state({"local_steps": 4}, 2, "decent")


# ---------------------------------------------------------------------------------------- gloo
_PORT = [35300 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "local_steps_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("H", [2, 3])
@pytest.mark.parametrize("world,topology", [(2, "ring"), (3, "ring"), (4, "ring"), (4, "exp"), (4, "onepeer-exp")])
def test_gloo_matches_simulator(world, topology, H):
    rc, out = _torchrun(world, "--mode", "sim", "--topology", topology, "--local-steps", str(H))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_resume_mid_cycle_is_exact_and_refuses_other_h(tmp_path):
    rc, out = _torchrun(3, "--mode", "resume", "--ckpt-dir", str(tmp_path))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
