"""Periodic global averaging (--global-avg-period P, decent): the simulator (an averaging step is the rank-ordered mean
followed by each rank's SGD step, gossip steps are plain decent's bit for bit, the mixing matrices and the byte count),
the gloo backend against the simulator bit for bit and a Trainer resume one step before an average
(tests/global_avg_worker.py), and the configuration rules."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import TILE, ParamArena, TensorTable
from eventgrad_b200.parallel.base import check_global_avg_state
from eventgrad_b200.parallel.trigger import rank_mean, sgd_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPT = dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=True)


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
    """Give every rank a different theta (ranks start from one theta_0; the first average would hide nothing)."""
    gen = torch.Generator().manual_seed(seed)
    for th in sim.theta:
        th.add_(torch.randn(t.n_padded, generator=gen) * _mask(t))


# ---------------------------------------------------------------------------------------- simulator
def test_rank_mean_is_rank_ordered_adds_then_one_division():
    gen = torch.Generator().manual_seed(0)
    xs = [torch.randn(4096, generator=gen) * 10 ** e for e in (0, 3, -3, 1, 2)]
    want = xs[0].clone()
    for x in xs[1:]:
        want = want + x
    want = want / torch.tensor(5.0)
    assert torch.equal(rank_mean(xs), want)
    assert all(torch.equal(a, b) for a, b in zip(xs, [x.clone() for x in xs]))      # inputs untouched
    # the order matters in fp32: a differently ordered sum is not always the same bits
    other = (((xs[4] + xs[3]) + xs[2]) + xs[1] + xs[0]) / 5
    assert not torch.equal(other, want)


@pytest.mark.parametrize("topology,R", [("ring", 3), ("ring", 4), ("exp", 8), ("1,3", 8)])
@pytest.mark.parametrize("P", [2, 3])
def test_average_step_is_the_rank_mean_then_sgd(topology, R, P):
    t = _table()
    table = torch.linspace(0.05, 0.01, 11)
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", serial_skip=False, offsets=topology,
                        global_avg_period=P, lr_table=table, **OPT)
    _spread(sim, t, R * 10 + P)
    for k in range(1, 2 * P + 2):
        g = _grads(t, R, 70 + k)
        before = [(x.clone(), mo.clone()) for x, mo in zip(sim.theta, sim.mom)]
        inb = [[x.clone() for x in ib] for ib in sim.inbox]
        by = list(sim.bytes)
        sim.step(g)
        if k % P:
            continue
        avg = rank_mean([th for th, _ in before])
        for r in range(R):
            th, mo = avg.clone(), before[r][1]
            sgd_(th, g[r], mo, float(table[k - 1]), OPT["momentum"], OPT["weight_decay"], OPT["nesterov"])
            assert torch.equal(sim.theta[r], th) and torch.equal(sim.mom[r], mo), f"step {k} rank {r}"
            assert all(torch.equal(x, y) for x, y in zip(sim.inbox[r], inb[r])), "an average touched an inbox"
            assert sim.bytes[r] - by[r] == t.n_elems * 4


@pytest.mark.parametrize("topology,R", [("ring", 2), ("ring", 5), ("exp", 8)])
def test_zero_gradients_leave_every_rank_bit_identical_after_an_average(topology, R):
    t = _table()
    # no weight decay: with it the momentum buffers would carry each rank's own wd * theta past the average
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", serial_skip=False, offsets=topology,
                        global_avg_period=3, lr=0.05, momentum=0.9, nesterov=True)
    _spread(sim, t, R)
    zeros = [torch.zeros(t.n_padded) for _ in range(R)]
    for k in range(1, 7):
        sim.step(zeros)
        same = all(torch.equal(sim.theta[0], x) for x in sim.theta[1:])
        if k % 3 == 0:
            assert same, f"step {k}"
        elif k == 1:
            assert not same


@pytest.mark.parametrize("topology,R", [("ring", 2), ("ring", 4), ("exp", 8), ("1,3", 8)])
@pytest.mark.parametrize("P", [2, 3, 5])
def test_gossip_steps_equal_plain_decent(topology, R, P):
    """Restart a plain decent simulator from the P-run's state after each average: the P - 1 gossip steps that follow
    are plain decent steps bit for bit (theta, momentum, inboxes, bytes)."""
    t = _table()
    table = torch.linspace(0.05, 0.01, 3 * P)
    kw = dict(serial_skip=False, offsets=topology, lr_table=table, **OPT)
    a = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", global_avg_period=P, **kw)
    _spread(a, t, P)
    for k in range(1, 3 * P):
        if k % P == 1 or k == 1:
            b = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", **kw)
            b.pass_num = a.pass_num
            for r in range(R):
                b.theta[r].copy_(a.theta[r])
                b.mom[r].copy_(a.mom[r])
                for x, y in zip(b.inbox[r], a.inbox[r]):
                    x.copy_(y)
            b.bytes = list(a.bytes)
        g = _grads(t, R, 300 + k)
        a.step(g)
        if k % P == 0:
            continue
        b.step(g)
        for r in range(R):
            assert torch.equal(a.theta[r], b.theta[r]) and torch.equal(a.mom[r], b.mom[r]), f"step {k} rank {r}"
            assert all(torch.equal(x, y) for x, y in zip(a.inbox[r], b.inbox[r]))
        assert a.bytes == b.bytes


@pytest.mark.parametrize("topology,R", [("ring", 3), ("ring", 6), ("exp", 8), ("1,3", 8)])
@pytest.mark.parametrize("P", [2, 3])
def test_mixing_matrices_and_no_learning(topology, R, P):
    """lr = 0, float64: W = 11^T / R at averaging steps and the graph's W otherwise, and theta_K = W_K ... W_1 theta_0."""
    t = _small_table()
    gen = torch.Generator().manual_seed(R * 10 + P)
    m = _mask(t, torch.float64)
    th = torch.stack([torch.randn(t.n_padded, generator=gen, dtype=torch.float64) * m for _ in range(R)])
    sim = RingSimulator(R, th[0], t, "decent", lr=0.0, serial_skip=False, offsets=topology, global_avg_period=P)
    plain = RingSimulator(R, th[0], t, "decent", lr=0.0, serial_skip=False, offsets=topology)
    for r in range(R):
        sim.theta[r].copy_(th[r])
    J = torch.full((R, R), 1.0 / R, dtype=torch.float64)
    Pm = torch.eye(R, dtype=torch.float64)
    zeros = [torch.zeros(t.n_padded, dtype=torch.float64) for _ in range(R)]
    for k in range(1, 3 * P + 2):
        W = sim.mixing_matrix()
        assert torch.equal(sim.mixing_matrix(k), W)
        assert torch.equal(W, J if k % P == 0 else plain.mixing_matrix(k)), k
        Pm = W @ Pm
        sim.step(zeros)
        assert float((torch.stack(sim.theta) - Pm @ th).abs().max()) < 1e-12, f"step {k}"


@pytest.mark.parametrize("topology", ["ring", "exp", "1,3"])
@pytest.mark.parametrize("P", [2, 3, 7])
def test_bytes(topology, P):
    R, K = 8, 15
    t = _table()
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", serial_skip=False, offsets=topology,
                        global_avg_period=P)
    for s in range(K):
        sim.step(_grads(t, R, s))
    avgs = K // P
    assert sim.bytes == [(avgs + (K - avgs) * sim.fanout) * 4 * t.n_elems] * R
    assert sim.dense_messages() == sim.fanout * t.n_tensors * K * R        # per-step definition, unchanged


@pytest.mark.parametrize("kw,match", [
    (dict(algo="event"), "global averaging"), (dict(algo="spevent"), "global averaging"),
    (dict(algo="cent"), "global averaging"), (dict(compress="int8"), "global averaging"),
    (dict(gradient_tracking=True), "global averaging"), (dict(exact_diffusion=True), "global averaging"),
    (dict(local_steps=2), "global averaging"), (dict(offsets="onepeer-exp"), "global averaging"),
])
def test_simulator_rejects_what_validate_rejects(kw, match):
    t = _table()
    algo = kw.pop("algo", "decent")
    with pytest.raises(ValueError, match=match):
        RingSimulator(4, torch.zeros(t.n_padded), t, algo, global_avg_period=2, **kw)
    with pytest.raises(ValueError, match="cent"):
        RingSimulator(4, torch.zeros(t.n_padded), t, "decent", global_avg_period=1)
    for bad in (-1, 2.5, True):
        with pytest.raises(ValueError, match="global_avg_period"):
            RingSimulator(4, torch.zeros(t.n_padded), t, "decent", global_avg_period=bad)


# ---------------------------------------------------------------------------------------- configuration
def _ga(**kw):
    base = dict(algo="decent", global_avg_period=4)
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("kw,match", [
    (dict(algo="cent"), "global-avg-period 4 needs algo decent"),
    (dict(algo="event"), "global-avg-period 4 needs algo decent"),
    (dict(algo="spevent"), "global-avg-period 4 needs algo decent"),
    (dict(topology="onepeer-exp"), "onepeer-exp"),
    (dict(gradient_tracking=True), "global-avg-period.*gradient-tracking"),
    (dict(exact_diffusion=True), "exact-diffusion"),
    (dict(compress="int8"), "global-avg-period.*int8"),
    (dict(local_steps=2), "global-avg-period.*local-steps 2"),
    (dict(backend="refport"), "global-avg-period.*refport"),
    (dict(overlap_push=True), "global-avg-period.*overlap_push"),
    (dict(double_buffer=True), "global-avg-period.*double_buffer"),
    (dict(ce_push=True), "global-avg-period.*ce_push"),
    (dict(file_write=1), "global-avg-period.*file_write"),
    (dict(global_avg_period=1), "global-avg-period 1.*cent"),
    (dict(global_avg_period=-2), "global-avg-period"),
    (dict(global_avg_period=2.5), "global-avg-period"),
    (dict(global_avg_period=True), "global-avg-period"),
])
def test_validation_rejects(kw, match):
    with pytest.raises(ValueError, match=match):
        _ga(**kw).validate()


def test_validation_accepts():
    for topo in ("ring", "1", "exp", "1,3", "2,3"):
        for P in (2, 3, 100):
            _ga(topology=topo, global_avg_period=P).validate()
    _ga(overlap_push=False, double_buffer=False, ce_push=False, backend="gloo", local_steps=1).validate()
    _ga(backend="nccl", momentum=0.9, nesterov=True, weight_decay=5e-4, partition="label").validate()
    for algo in ("cent", "decent", "event", "spevent"):
        TrainConfig(algo=algo, global_avg_period=0).validate()      # P = 0 restricts nothing


def test_resolved_keeps_the_fused_single_slot_step():
    from eventgrad_b200.parallel.p2p import _wants_dbuf
    for topo in ("ring", "exp"):
        c = _ga(topology=topo).validate().resolved("cuda", 8)
        assert c.overlap_push is False and not _wants_dbuf(c)
    assert _wants_dbuf(TrainConfig(algo="decent", overlap_push=False).validate())
    assert TrainConfig(algo="decent").validate().resolved("cuda", 4).overlap_push is True


def test_cli_and_presets():
    c = parse_cli("decent", ["--global-avg-period", "4", "--topology", "exp"])
    assert c.global_avg_period == 4 and c.topology == "exp"
    assert parse_cli("decent", []).global_avg_period == 0
    for prog in ("mnist_event", "cent"):
        with pytest.raises(ValueError, match="global-avg-period"):
            parse_cli(prog, ["--global-avg-period", "2"])
    with pytest.raises(ValueError, match="cent"):
        parse_cli("decent", ["--global-avg-period", "1"])
    assert all(preset(n).global_avg_period == 0 for n in PRESETS)


def test_check_global_avg_state():
    check_global_avg_state({}, 0, "decent")                      # no key: never averaged
    check_global_avg_state({"global_avg_period": 4}, 4, "decent")
    check_global_avg_state({}, 4, "event")                       # only decent carries the period
    with pytest.raises(ValueError, match="global-avg-period 0"):
        check_global_avg_state({}, 4, "decent")
    with pytest.raises(ValueError, match="global-avg-period 4"):
        check_global_avg_state({"global_avg_period": 4}, 2, "decent")


def test_plain_checkpoints_keep_their_keys():
    """P = 0 writes no global_avg_period key, so a run without the feature saves what it saved before."""
    import torch.distributed as dist
    from eventgrad_b200.parallel import Ring
    from eventgrad_b200.parallel.collective import CollectiveBackend
    assert not dist.is_initialized()
    for P in (0, 3):
        cfg = TrainConfig(algo="decent", device="cpu", backend="gloo", global_avg_period=P).validate()
        be = CollectiveBackend(cfg, ParamArena(build_model("cnn2"), torch.device("cpu")), Ring(0, 1))
        assert ("global_avg_period" in be.state_dict()) == (P > 0)


# ---------------------------------------------------------------------------------------- gloo
_PORT = [36300 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "global_avg_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("P", [2, 3])
@pytest.mark.parametrize("world,topology", [(2, "ring"), (3, "ring"), (4, "ring"), (4, "exp")])
def test_gloo_matches_simulator(world, topology, P):
    rc, out = _torchrun(world, "--mode", "sim", "--topology", topology, "--global-avg-period", str(P))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_resume_before_an_average_is_exact_and_refuses_other_p(tmp_path):
    rc, out = _torchrun(3, "--mode", "resume", "--ckpt-dir", str(tmp_path))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
