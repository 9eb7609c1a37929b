"""Circulant gossip graphs beyond the ring (parallel/topology.py): offsets and their validation, the mixing matrix,
the simulator against the ring and against float64 W @ theta, configuration / CLI limits, and the gloo backend
against the simulator bit for bit (tests/topology_worker.py), including an exact checkpoint resume."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.parallel.arena import TensorTable
from eventgrad_b200.parallel.topology import Graph, Ring, parse_topology
from eventgrad_b200.parallel.trigger import TriggerConfig, mix3_, mixk_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------- offsets
def _exp(R):
    out, o = [], 1
    while o <= max(1, R // 2) and len(out) < 4:
        out.append(o)
        o *= 2
    return tuple(out)


@pytest.mark.parametrize("R", range(1, 17))
def test_offsets_of_ring_exp_and_explicit_sets(R):
    assert parse_topology("ring", R) == (1,)
    assert parse_topology("exp", R) == _exp(R)
    assert (parse_topology("exp", R) == (1,)) == (R <= 3)
    assert Graph.build(0, R, "exp").is_ring == (R <= 3)
    half = R // 2
    if half >= 1:
        assert parse_topology(str(half), R) == (half,)
        assert parse_topology("1", R) == (1,)
    if half >= 3:
        assert parse_topology("1,3", R) == (1, 3)
    # out of range, duplicated, unsorted, too many, malformed (a single rank accepts the ring's "1" only)
    for bad in ([f"{half + 1}"] if R > 1 else ["2"]) + ["0", "1,1", "2,1", "1,2,3,4,5", "x", "1,,2", "-1"]:
        with pytest.raises(ValueError):
            parse_topology(bad, R)


def test_exp_names():
    assert parse_topology("exp", 8) == (1, 2, 4)
    assert parse_topology("exp", 16) == (1, 2, 4, 8)
    assert parse_topology("exp", 64) == (1, 2, 4, 8)          # at most 4 offsets: degree <= 8
    assert parse_topology("exp", 5) == (1, 2)
    assert parse_topology("EXP", 4) == (1, 2) and parse_topology(" ring ", 9) == (1,)


@pytest.mark.parametrize("R", range(1, 17))
def test_slots_and_out_slots_are_consistent(R):
    for spec in ("ring", "exp", "2", "1,3"):
        try:
            offs = parse_topology(spec, R)
        except ValueError:
            continue
        gs = [Graph(r, R, offs) for r in range(R)]
        for r, g in enumerate(gs):
            assert g.n_slots == 2 * len(offs) == len(g.slots()) == len(g.out_slots())
            for j, (p, k) in enumerate(g.out_slots()):
                assert k == j and gs[p].slots()[k] == r          # my out-slot j is the peer's slot j, fed by me
            for k, o in enumerate(offs):
                assert g.slots()[2 * k] == (r - o) % R and g.slots()[2 * k + 1] == (r + o) % R


def test_ring_graph_matches_ring():
    for R in range(1, 9):
        for r in range(R):
            g, ring = Graph.build(r, R, "ring"), Ring(r, R)
            assert (g.left, g.right, g.degenerate_pair, g.serial) == (ring.left, ring.right, ring.degenerate_pair,
                                                                     ring.serial)
            assert g.mixing_row() == ring.mixing_row() and g.slots() == ring.slots()
            assert g.out_slots() == ring.out_slots()
    with pytest.raises(AttributeError):
        Graph.build(0, 8, "exp").left


@pytest.mark.parametrize("R", range(2, 17))
def test_mixing_matrix_is_symmetric_and_doubly_stochastic(R):
    for spec in ("ring", "exp", "1,3", str(R // 2)):
        try:
            offs = parse_topology(spec, R)
        except ValueError:
            continue
        W = torch.tensor([Graph(r, R, offs).mixing_row() for r in range(R)], dtype=torch.float64)
        assert torch.allclose(W, W.T, atol=0, rtol=0)
        assert torch.allclose(W.sum(0), torch.ones(R, dtype=torch.float64), atol=1e-12)
        assert torch.allclose(W.sum(1), torch.ones(R, dtype=torch.float64), atol=1e-12)
        assert (W >= 0).all()
        if R % 2 == 0 and R // 2 in offs:                       # aliased offset: that peer counts twice
            assert W[0, R // 2] == pytest.approx(2.0 / (2 * len(offs) + 1))


# ---------------------------------------------------------------------------------------- simulator
def _table():
    shapes = [(37,), (5, 7), (3000,), (11, 13)]
    return TensorTable.from_named([(f"p{i}", torch.zeros(s)) for i, s in enumerate(shapes)], 2048)


def _mask(t):
    m = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


def test_mixk_equals_mix3():
    g = torch.Generator().manual_seed(4)
    th, L, R = (torch.randn(5000, generator=g) for _ in range(3))
    assert torch.equal(mix3_(th.clone(), L, R), mixk_(th.clone(), [L, R]))


@pytest.mark.parametrize("algo", ["decent", "event"])
@pytest.mark.parametrize("R", [1, 2, 3, 5])
def test_simulator_default_ring_is_unchanged(algo, R):
    t = _table()
    g = torch.Generator().manual_seed(1)
    th0 = torch.randn(t.n_padded, generator=g)
    tc = TriggerConfig(initial_comm_passes=2)
    a = RingSimulator(R, th0, t, algo, tc, lr=0.05, momentum=0.9, serial_skip=False)
    b = RingSimulator(R, th0, t, algo, tc, lr=0.05, momentum=0.9, serial_skip=False, offsets=(1,))
    c = RingSimulator(R, th0, t, algo, tc, lr=0.05, momentum=0.9, serial_skip=False, offsets="exp" if R <= 3 else (1,))
    for s in range(8):
        grads = [torch.randn(t.n_padded, generator=g) * 0.1 for _ in range(R)]
        for sim in (a, b, c):
            sim.step(grads)
    for sim in (b, c):
        assert all(torch.equal(x, y) for x, y in zip(a.theta, sim.theta))
        assert sim.events == a.events and sim.bytes == a.bytes and sim.dense_messages() == a.dense_messages()
    # the ring path itself: (theta + L + R) / 3 with L/R the neighbours' pre-step theta
    th = [torch.randn(t.n_padded, generator=g) * _mask(t) for _ in range(R)]      # tile padding is never pushed
    sim = RingSimulator(R, th0, t, "decent", lr=0.0, serial_skip=False)
    sim.theta = [x.clone() for x in th]
    sim.step([torch.zeros(t.n_padded)] * R)
    for r in range(R):
        want = th[r].clone().add_(th[(r - 1) % R]).add_(th[(r + 1) % R]).div_(3)
        assert torch.equal(sim.theta[r], want)


@pytest.mark.parametrize("R,spec", [(4, "exp"), (5, "exp"), (5, "2"), (8, "exp"), (8, "1,3"), (16, "exp"), (6, "3")])
def test_simulator_decent_step_is_W_theta(R, spec):
    t = _table()
    g = torch.Generator().manual_seed(7)
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", lr=0.0, serial_skip=False, offsets=spec)
    th = torch.randn(R, t.n_padded, generator=g, dtype=torch.float64) * _mask(t)
    sim.theta = [th[r].float().clone() for r in range(R)]
    sim.step([torch.zeros(t.n_padded)] * R)
    want = sim.mixing_matrix() @ th.float().double()
    got = torch.stack(sim.theta).double()
    assert torch.allclose(got, want, rtol=0, atol=2e-6), (got - want).abs().max()
    n = 2 * len(parse_topology(spec, R))
    assert sim.dense_messages() == n * t.n_tensors * R
    assert sim.bytes == [n * t.n_elems * 4] * R


def test_simulator_event_counters_scale_with_slots():
    t = _table()
    R = 8
    sim = RingSimulator(R, torch.randn(t.n_padded), t, "event", TriggerConfig(initial_comm_passes=3), lr=0.01,
                        serial_skip=False, offsets="exp")
    for s in range(2):                                         # steps 1, 2 < initial_comm_passes: every tensor fires
        sim.step([torch.randn(t.n_padded) * 0.1 for _ in range(R)])
    assert sim.events == [6 * t.n_tensors * 2] * R and sim.total_events() == sim.dense_messages()


def test_simulator_rejects_spevent_and_cent_graphs():
    t = _table()
    for algo in ("spevent", "cent"):
        with pytest.raises(ValueError):
            RingSimulator(8, torch.zeros(t.n_padded), t, algo, offsets="exp")


# ---------------------------------------------------------------------------------------- config / CLI
def test_config_rejects_unsupported_combinations():
    ok = dict(algo="event", topology="exp")
    TrainConfig(**ok).validate()
    TrainConfig(algo="decent", topology="1,3", sync_mode="iter", backend="nccl").validate()
    TrainConfig(algo="event", topology="2", sync_mode="async", backend="p2p", overlap_push=False).validate()
    bad = [dict(algo="spevent"), dict(algo="cent"), dict(backend="refport"), dict(overlap_push=True),
           dict(double_buffer=True), dict(ce_push=True), dict(file_write=1)]
    for b in bad:
        with pytest.raises(ValueError):
            TrainConfig(**{**ok, **b}).validate()
    for spec in ("2,1", "1,1", "0", "1,2,3,4,5", "star", ""):
        with pytest.raises(ValueError):
            TrainConfig(topology=spec).validate()
    # the ring keeps every option
    TrainConfig(algo="spevent", topology="ring", file_write=1, overlap_push=True).validate()
    TrainConfig(algo="decent", topology="1", double_buffer=True).validate()


def test_resolved_turns_auto_overlap_off_for_graphs():
    c = TrainConfig(algo="decent", topology="exp").validate().resolved("cuda", 8)
    assert c.overlap_push is False
    r = TrainConfig(algo="decent").validate().resolved("cuda", 8)
    assert r.overlap_push is True
    from eventgrad_b200.parallel.p2p import _wants_dbuf
    assert _wants_dbuf(TrainConfig(algo="decent", overlap_push=False))
    assert not _wants_dbuf(TrainConfig(algo="decent", overlap_push=False, topology="exp"))


def test_names_that_resolve_to_the_ring_get_the_ring_defaults():
    from eventgrad_b200.parallel.p2p import _wants_dbuf
    for R in (1, 2, 3):
        for algo in ("decent", "event"):
            ring = TrainConfig(algo=algo).validate()
            for spec in ("exp", "1"):
                c = TrainConfig(algo=algo, topology=spec).validate()
                for dev in ("cuda", "cpu"):
                    got = c.resolved(dev, R)
                    assert got.ring_topology and got.replace(topology="ring") == ring.resolved(dev, R)
                assert c.for_world(R).ring_topology
                assert _wants_dbuf(c.resolved("cuda", R).replace(overlap_push=False)) == (algo == "decent")
    assert TrainConfig(algo="decent", topology="exp").validate().for_world(2).topology == "ring"
    assert TrainConfig(algo="decent", topology="exp").validate().for_world(4).topology == "exp"
    with pytest.raises(ValueError):
        TrainConfig(algo="decent", topology="3").validate().resolved("cuda", 4)        # 3 > R/2


def test_cli_topology_flag():
    assert parse_cli("cifar_event", ["0", "1", "1.0", "--topology", "exp"]).topology == "exp"
    assert parse_cli("decent", ["0", "--topology", "1,3"]).topology == "1,3"
    assert parse_cli("mnist_event", ["0"]).topology == "ring"
    for name in ("cent", "decent", "mnist_event", "cifar_event", "cifar_spevent"):
        assert preset(name).topology == "ring"
    with pytest.raises(ValueError):
        parse_cli("cifar_spevent", ["0", "1", "1.0", "5", "--topology", "exp"])
    with pytest.raises(ValueError):
        parse_cli("cent", ["--topology", "exp"])
    with pytest.raises(ValueError):
        parse_cli("mnist_event", ["1", "--topology", "exp"])           # file_write=1
    with pytest.raises(ValueError):
        parse_cli("cifar_event", ["0", "1", "1.0", "--topology", "exp", "--overlap-push"])


def test_trainer_rejects_offsets_out_of_range_for_the_world():
    from eventgrad_b200.data import synthetic_source
    from eventgrad_b200.engine.trainer import Trainer
    from eventgrad_b200.utils.dist import DistEnv
    cfg = preset("mnist_event", device="cpu", backend="gloo", topology="2", quiet=True, train_samples=64)
    with pytest.raises(ValueError):
        Trainer(cfg, DistEnv(0, 1, 0, torch.device("cpu"), "none"), train_source=synthetic_source("mnist", 64))


# ---------------------------------------------------------------------------------------- gloo
_PORT = [32700 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "topology_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("algo", ["decent", "event"])
@pytest.mark.parametrize("world,topology", [(4, "exp"), (5, "exp"), (5, "2")])
def test_gloo_graph_matches_simulator(algo, world, topology):
    rc, out = _torchrun(world, "--mode", "sim", "--algo", algo, "--topology", topology, "--steps", "10")
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_graph_resume_is_exact_and_refuses_the_ring(tmp_path):
    rc, out = _torchrun(4, "--mode", "resume", "--topology", "exp", "--ckpt-dir", str(tmp_path))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
