"""The time-varying one-peer exponential graph (parallel/topology.py OnePeerExp, --topology onepeer-exp): the name and
its limits, the mixing matrices in exact fractions, exact consensus in the simulator, and the gloo backend against the
simulator bit for bit (tests/onepeer_worker.py), including a checkpoint resume at a step inside the cycle."""
import os
import subprocess
import sys
from fractions import Fraction

import pytest
import torch

from eventgrad_b200.config import TrainConfig, parse_cli
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import ParamArena
from eventgrad_b200.parallel.topology import Graph, OnePeerExp, parse_topology
from eventgrad_b200.parallel.trigger import TriggerConfig, mix2_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "onepeer-exp"


def _table():
    return ParamArena(build_model("cnn2"), torch.device("cpu")).table


def _mask(t):
    m = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


# ---------------------------------------------------------------------------------------- the graph
@pytest.mark.parametrize("R", range(2, 18))
def test_period_offsets_and_peers(R):
    tau = (R - 1).bit_length()
    assert 2 ** (tau - 1) < R <= 2 ** tau
    for r in range(R):
        g = Graph.build(r, R, NAME)
        assert isinstance(g, OnePeerExp) and not g.is_ring and g.fanout == 1
        assert g.period == g.n_slots == tau and g.offsets == tuple(2 ** m for m in range(tau))
        assert all(o < R for o in g.offsets)
        for k in range(1, 3 * tau + 1):
            m = (k - 1) % tau
            assert g.active(k) == m
            assert g.out_peer(k) == (r + 2 ** m) % R and g.in_peer(k) == (r - 2 ** m) % R
            # the sender of my active slot pushes into exactly that slot at the same step
            src = Graph.build(g.in_peer(k), R, NAME)
            assert src.out_slots()[m] == (r, m) and src.out_peer(k) == r
        assert g.slots() == [g.in_peer(m + 1) for m in range(tau)]


def test_three_ranks_and_two_ranks():
    g = Graph.build(0, 3, NAME)
    assert g.offsets == (1, 2) and g.period == 2
    assert [g.out_peer(k) for k in (1, 2, 3)] == [1, 2, 1]
    g2 = Graph.build(1, 2, NAME)
    assert g2.period == 1 and g2.mixing_row(1) == [0.5, 0.5]      # (theta + theta_peer) / 2, not the ring's 1/3, 2/3


def test_single_rank_and_static_offsets():
    assert parse_topology(NAME, 1) == (1,)
    assert Graph.build(0, 1, NAME).is_ring
    for R in (2, 3, 8):
        with pytest.raises(ValueError):
            parse_topology(NAME, R)          # time-varying: no static offsets
    with pytest.raises(ValueError):
        Graph.build(0, 257, NAME)            # period 9 > the kernel's 8 slots
    with pytest.raises(ValueError):
        Graph.build(0, 4, NAME).active(0)    # steps are 1-based


def _W(R, k):
    return [[Fraction(x) for x in Graph.build(r, R, NAME).mixing_row(k)] for r in range(R)]


def _matmul(A, B):
    n = len(A)
    return [[sum(A[i][j] * B[j][c] for j in range(n)) for c in range(n)] for i in range(n)]


@pytest.mark.parametrize("R", [2, 3, 4, 5, 8, 16])
def test_every_W_is_doubly_stochastic_and_directed(R):
    tau = Graph.build(0, R, NAME).period
    for k in range(1, tau + 1):
        W = _W(R, k)
        assert all(sum(row) == 1 for row in W)
        assert all(sum(W[i][j] for i in range(R)) == 1 for j in range(R))
        assert all(x >= 0 for row in W for x in row)
        symmetric = all(W[i][j] == W[j][i] for i in range(R) for j in range(R))
        assert symmetric == (2 ** (k - 1) * 2 == R)       # directed unless the offset is R/2 (then r+o == r-o)


@pytest.mark.parametrize("R", [2, 4, 8, 16])
def test_product_over_one_period_is_the_exact_average(R):
    tau = Graph.build(0, R, NAME).period
    P = _W(R, 1)
    for k in range(2, tau + 1):
        P = _matmul(_W(R, k), P)                 # W_tau ... W_1
    assert P == [[Fraction(1, R)] * R for _ in range(R)]


@pytest.mark.parametrize("R", [3, 5, 6])
def test_product_is_not_exact_when_R_is_not_a_power_of_two(R):
    tau = Graph.build(0, R, NAME).period
    P = _W(R, 1)
    for k in range(2, tau + 1):
        P = _matmul(_W(R, k), P)
    assert P != [[Fraction(1, R)] * R for _ in range(R)]
    assert all(sum(row) == 1 for row in P)


# ---------------------------------------------------------------------------------------- simulator
def test_mix2_rounding():
    a = torch.tensor([1.0, 3.0, 1e-45, 3.4e38, 0.1])
    b = torch.tensor([2.0, 4.0, 0.0, 3.4e38, 0.2])
    want = (a + b) / 2
    assert torch.equal(mix2_(a.clone(), b), want)


@pytest.mark.parametrize("R", [4, 8])
def test_simulator_reaches_exact_consensus_in_one_period(R):
    t = _table()
    m = _mask(t)
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", lr=0.0, serial_skip=False, offsets=NAME)
    g = torch.Generator().manual_seed(R)
    sim.theta = [torch.randint(-64, 64, (t.n_padded,), generator=g).float() * m for _ in range(R)]
    mean = torch.stack(sim.theta).double().mean(0)
    assert torch.equal(mean.float().double(), mean)          # the mean is exact in fp32
    for _ in range(sim.period - 1):
        sim.step([torch.zeros(t.n_padded)] * R)
    assert not all(torch.equal(th, mean.float()) for th in sim.theta)
    sim.step([torch.zeros(t.n_padded)] * R)
    for r in range(R):
        assert torch.equal(sim.theta[r], mean.float()), r


@pytest.mark.parametrize("R", [3, 4, 5])
def test_simulator_step_is_W_k_theta(R):
    t = _table()
    m = _mask(t)
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", lr=0.0, serial_skip=False, offsets=NAME)
    g = torch.Generator().manual_seed(1)
    th = torch.randn(R, t.n_padded, generator=g, dtype=torch.float64) * m
    sim.theta = [th[r].float().clone() for r in range(R)]
    x = torch.stack(sim.theta).double()
    for k in range(1, 2 * sim.period + 2):
        W = sim.mixing_matrix()
        assert torch.equal(W, sim.mixing_matrix(k))
        x = W @ x
        sim.step([torch.zeros(t.n_padded)] * R)
        assert torch.allclose(torch.stack(sim.theta).double(), x, rtol=1e-6, atol=1e-7)


def test_simulator_event_accounting():
    R = 4
    t = _table()
    tc = TriggerConfig(thres_type=1, horizon=1.0, initial_comm_passes=3)
    sim = RingSimulator(R, torch.randn(t.n_padded) * _mask(t), t, "event", tc, lr=0.05, serial_skip=False,
                        offsets=NAME)
    for s in range(2):                                  # steps 1, 2 < initial_comm_passes: every tensor fires
        sim.step([torch.randn(t.n_padded) * 0.1 for _ in range(R)])
    assert sim.events == [t.n_tensors * 2] * R and sim.total_events() == sim.dense_messages()
    assert sim.bytes == [t.n_elems * 4 * 2] * R
    for algo in ("spevent", "cent"):
        with pytest.raises(ValueError):
            RingSimulator(R, torch.zeros(t.n_padded), t, algo, offsets=NAME)


def test_event_slot_keeps_the_last_arrival():
    """A slot holds what last arrived from its sender, possibly from tau or more steps back."""
    R = 4
    t = _table()
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "event", TriggerConfig(), lr=0.0, serial_skip=False,
                        offsets=NAME)
    th = [torch.full((t.n_padded,), float(r + 1)) * _mask(t) for r in range(R)]
    sim.theta = [x.clone() for x in th]
    fire_all = [torch.ones(t.n_tensors, dtype=torch.bool)] * R
    fire_none = [torch.zeros(t.n_tensors, dtype=torch.bool)] * R
    sim.step([torch.zeros(t.n_padded)] * R, fires=fire_all)     # step 1: slot 0 of r holds theta of r-1
    for r in range(R):
        assert torch.equal(sim.inbox[r][0], th[(r - 1) % R])
        assert torch.equal(sim.theta[r], (th[r] + th[(r - 1) % R]) / 2)
    snap = [x.clone() for x in sim.theta]
    sim.step([torch.zeros(t.n_padded)] * R, fires=fire_none)    # step 2: nothing sent, slot 1 still zero
    for r in range(R):
        assert torch.equal(sim.theta[r], snap[r] / 2)
    snap = [x.clone() for x in sim.theta]
    sim.step([torch.zeros(t.n_padded)] * R, fires=fire_none)    # step 3: slot 0 again, its value is from step 1
    for r in range(R):
        assert torch.equal(sim.theta[r], (snap[r] + th[(r - 1) % R]) / 2)
    assert sim.events == [t.n_tensors] * R


# ---------------------------------------------------------------------------------------- config / CLI
def test_config_name_limits_and_resolution():
    ok = dict(algo="event", topology=NAME)
    TrainConfig(**ok).validate()
    TrainConfig(algo="decent", topology=NAME, backend="nccl").validate()
    TrainConfig(algo="event", topology=NAME, sync_mode="async", backend="p2p", overlap_push=False).validate()
    bad = [dict(algo="spevent"), dict(algo="cent"), dict(backend="refport"), dict(overlap_push=True),
           dict(double_buffer=True), dict(ce_push=True), dict(file_write=1)]
    for b in bad:
        with pytest.raises(ValueError):
            TrainConfig(**{**ok, **b}).validate()
    c = TrainConfig(**ok).validate()
    assert not c.ring_topology
    assert c.for_world(1).topology == "ring"
    assert c.resolved("cuda", 1) == TrainConfig(algo="event").validate().resolved("cuda", 1)
    for R in (2, 3, 4, 8):
        assert c.for_world(R).topology == NAME
        r = TrainConfig(algo="decent", topology=NAME).validate().resolved("cuda", R)
        assert r.overlap_push is False and r.topology == NAME
        from eventgrad_b200.parallel.p2p import _wants_dbuf
        assert not _wants_dbuf(r)


def test_cli_topology_flag():
    assert parse_cli("cifar_event", ["0", "1", "1.0", "--topology", NAME]).topology == NAME
    assert parse_cli("decent", ["0", "--topology", NAME]).topology == NAME
    with pytest.raises(ValueError):
        parse_cli("cifar_spevent", ["0", "1", "1.0", "5", "--topology", NAME])
    with pytest.raises(ValueError):
        parse_cli("mnist_event", ["1", "--topology", NAME])            # file_write=1
    with pytest.raises(ValueError):
        parse_cli("cifar_event", ["0", "1", "1.0", "--topology", NAME, "--double-buffer"])


def test_checkpoint_state_is_tagged_with_the_name():
    from eventgrad_b200.parallel.base import check_topology_state
    one = Graph.build(0, 4, NAME)
    stat = Graph.build(0, 4, "exp")
    assert one.offsets == stat.offsets == (1, 2)            # same offsets: the name must tell them apart
    sd = {"topology": one.kind, "topology_offsets": list(one.offsets)}
    check_topology_state(sd, one, "event")
    for other in (stat, Graph.build(0, 4, "ring")):
        with pytest.raises(ValueError):
            check_topology_state(sd, other, "event")
    with pytest.raises(ValueError):
        check_topology_state({"topology_offsets": [1, 2]}, one, "decent")
    with pytest.raises(ValueError):
        check_topology_state({}, one, "decent")


# ---------------------------------------------------------------------------------------- gloo, multi-process
_PORT = [34700 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "onepeer_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("algo", ["decent", "event"])
def test_gloo_onepeer_matches_simulator_every_step(algo, world):
    rc, out = _torchrun(world, "--mode", "sim", "--algo", algo)
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_resume_inside_the_cycle_is_exact_and_refuses_other_graphs(tmp_path):
    rc, out = _torchrun(4, "--mode", "resume", "--ckpt-dir", str(tmp_path))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
