"""Gradient tracking (--gradient-tracking, decent on the ring) and label-sorted shards (--partition label): the simulator
in float64 on heterogeneous quadratics (y_1 = g_1, sum y = sum g, exact consensus at the minimiser where plain decent
stays biased), the unchanged non-tracking path, the gloo backend against the simulator bit for bit and a checkpoint
resume (tests/tracking_worker.py), the configuration rules and the sampler."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.data.sampler import ShardSampler
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import TILE, ParamArena, TensorTable
from eventgrad_b200.parallel.base import check_tracking_state
from eventgrad_b200.parallel.trigger import mix3_, sgd_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------- heterogeneous quadratics
class Quadratics:
    """f_r(theta) = 1/2 (theta - c_r)^T A_r (theta - c_r), A_r diagonal, on a two-tensor table (float64).  The global
    minimiser of sum_r f_r is theta* = (sum A_r)^-1 sum A_r c_r; the padding lanes have A = 0 and stay zero."""

    def __init__(self, R, sizes=(37, 300), seed=0, dtype=torch.float64):
        w = [torch.nn.Parameter(torch.zeros(n)) for n in sizes]
        self.table = TensorTable.from_named([(f"w{i}", p) for i, p in enumerate(w)], TILE)
        t = self.table
        self.mask = torch.zeros(t.n_padded, dtype=dtype)
        for o, n in zip(t.offsets, t.numels):
            self.mask[o:o + n] = 1
        g = torch.Generator().manual_seed(seed)
        self.A = [(0.5 + 1.5 * torch.rand(t.n_padded, generator=g, dtype=dtype)) * self.mask for _ in range(R)]
        self.c = [(torch.randn(t.n_padded, generator=g, dtype=dtype) * 2.0 + r) * self.mask for r in range(R)]
        sa = torch.stack(self.A).sum(0)
        self.opt = torch.where(self.mask > 0, torch.stack([a * c for a, c in zip(self.A, self.c)]).sum(0)
                               / torch.where(sa > 0, sa, torch.ones_like(sa)), torch.zeros_like(sa))
        self.dtype = dtype

    def grads(self, thetas):
        return [a * (th - c) for a, c, th in zip(self.A, self.c, thetas)]

    def sim(self, R, tracking, lr=0.1, **kw):
        return RingSimulator(R, torch.zeros(self.table.n_padded, dtype=self.dtype), self.table, "decent", lr=lr,
                             momentum=kw.pop("momentum", 0.0), serial_skip=False, gradient_tracking=tracking, **kw)


def _err(sim, q):
    return max(float((th - q.opt).abs().max()) for th in sim.theta)


@pytest.mark.parametrize("R", [2, 3, 4, 5])
def test_first_y_is_the_gradient_and_y_tracks_the_gradient_sum(R):
    q = Quadratics(R)
    sim = q.sim(R, True)
    for k in range(1, 61):
        g = q.grads(sim.theta)
        sim.step(g)
        if k == 1:
            assert all(torch.equal(y, gr) for y, gr in zip(sim.y, g)), "y_1 must be g_1"
        dev = float((torch.stack(sim.y).sum(0) - torch.stack(g).sum(0)).abs().max())
        assert dev < 1e-12, f"step {k}: |sum y - sum g| = {dev:.3e}"
        assert all(torch.equal(gp, gr) for gp, gr in zip(sim.g_prev, g))


@pytest.mark.parametrize("R", [2, 4, 6])
def test_tracking_reaches_the_global_minimiser_where_decent_does_not(R):
    q = Quadratics(R, seed=R)
    gt, dp = q.sim(R, True), q.sim(R, False)
    for _ in range(600):
        gt.step(q.grads(gt.theta))
        dp.step(q.grads(dp.theta))
    assert _err(gt, q) < 1e-10, _err(gt, q)
    assert _err(dp, q) > 1e-2, _err(dp, q)          # constant-lr D-PSGD settles at a biased point
    assert all(bool((th[q.mask == 0] == 0).all()) for th in gt.theta)


def test_tracking_with_momentum_weight_decay_and_nesterov_converges():
    """The optimizer sees y_k where it saw g_k: with heavy-ball momentum the fixed point is the minimiser of
    sum f_r + wd/2 ||theta||^2 (weight decay is the same on every rank, so it is not tracked)."""
    R, wd = 4, 0.05
    q = Quadratics(R, seed=9)
    sim = q.sim(R, True, lr=0.02, momentum=0.9, weight_decay=wd, nesterov=True)
    for _ in range(1500):
        sim.step(q.grads(sim.theta))
    sa = torch.stack(q.A).sum(0)
    want = torch.stack([a * c for a, c in zip(q.A, q.c)]).sum(0) / torch.where(q.mask > 0, sa + R * wd, 1.0)
    assert max(float((th - want).abs().max()) for th in sim.theta) < 1e-10


def test_r1_is_plain_sgd():
    q = Quadratics(1)
    a, b = q.sim(1, True), q.sim(1, False)
    for _ in range(5):
        a.step(q.grads(a.theta))
        b.step(q.grads(b.theta))
    assert torch.equal(a.theta[0], b.theta[0]) and not a.gt


def test_tracking_off_is_the_plain_simulator():
    """gradient_tracking=False computes exactly what mix3_ + sgd_ compute per rank (the simulator before tracking)."""
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    m = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    g = torch.Generator().manual_seed(2)
    theta0 = torch.randn(t.n_padded, generator=g) * m
    R = 3
    a = RingSimulator(R, theta0, t, "decent", lr=0.05, momentum=0.9, serial_skip=False)
    b = RingSimulator(R, theta0, t, "decent", lr=0.05, momentum=0.9, serial_skip=False, gradient_tracking=False)
    th = [theta0.clone() for _ in range(R)]
    mom = [torch.zeros_like(theta0) for _ in range(R)]
    for s in range(5):
        gr = [torch.randn(t.n_padded, generator=g) * m for _ in range(R)]
        a.step(gr)
        b.step(gr)
        snap = [x.clone() for x in th]
        for r in range(R):
            mix3_(th[r], snap[(r - 1) % R], snap[(r + 1) % R])
            sgd_(th[r], gr[r], mom[r], 0.05, 0.9)
    for r in range(R):
        assert torch.equal(a.theta[r], th[r]) and torch.equal(b.theta[r], th[r])
    assert a.bytes == b.bytes == [5 * 2 * t.n_elems * 4] * R
    assert not hasattr(b, "y")


def test_tracking_bytes_are_two_payloads():
    q = Quadratics(3)
    sim = q.sim(3, True)
    for _ in range(4):
        sim.step(q.grads(sim.theta))
    assert sim.bytes == [4 * 2 * 2 * q.table.n_elems * 4] * 3


@pytest.mark.parametrize("kw", [dict(algo="event"), dict(algo="spevent"), dict(algo="cent"), dict(offsets=(1, 2)),
                                dict(offsets="onepeer-exp"), dict(compress="int8")])
def test_simulator_rejects_what_validate_rejects(kw):
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    algo = kw.pop("algo", "decent")
    with pytest.raises(ValueError, match="tracking"):
        RingSimulator(5, torch.zeros(t.n_padded), t, algo, gradient_tracking=True, **kw)


# ---------------------------------------------------------------------------------------- configuration
def _gt(**kw):
    base = dict(algo="decent", gradient_tracking=True)
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("kw,match", [
    (dict(algo="event"), "stale y"),
    (dict(algo="spevent"), "stale y"),
    (dict(algo="cent"), "decent"),
    (dict(topology="exp"), "ring"),
    (dict(topology="1,2"), "ring"),
    (dict(topology="onepeer-exp"), "ring"),
    (dict(backend="refport"), "refport"),
    (dict(overlap_push=True), "overlap_push"),
    (dict(double_buffer=True), "double_buffer"),
    (dict(ce_push=True), "ce_push"),
    (dict(compress="int8"), "int8"),
    (dict(file_write=1), "file_write"),
])
def test_validation_rejects(kw, match):
    with pytest.raises(ValueError, match=match):
        _gt(**kw).validate()


def test_validation_accepts_and_partition_rules():
    _gt().validate()
    _gt(overlap_push=False, double_buffer=False, ce_push=False, backend="gloo").validate()
    for algo in ("cent", "decent", "event", "spevent"):
        TrainConfig(algo=algo, partition="label").validate()
    with pytest.raises(ValueError, match="partition"):
        TrainConfig(partition="dirichlet").validate()


def test_resolved_keeps_the_fused_single_slot_step():
    from eventgrad_b200.parallel.p2p import _wants_dbuf, _wants_gt
    c = _gt().validate().resolved("cuda", 4)
    assert c.overlap_push is False and not _wants_dbuf(c) and _wants_gt(c, 4)
    assert not _wants_gt(c, 1)
    assert TrainConfig(algo="decent").validate().resolved("cuda", 4).overlap_push is True
    assert _wants_dbuf(TrainConfig(algo="decent", overlap_push=False).validate())


def test_cli_and_presets():
    for prog in ("decent", "mnist_event", "cifar_event", "cent"):
        c = parse_cli(prog, ["--partition", "label"])
        assert c.partition == "label" and not c.gradient_tracking
    c = parse_cli("decent", ["--gradient-tracking"])
    assert c.gradient_tracking and c.partition == "iid"
    with pytest.raises(ValueError, match="decent"):
        parse_cli("mnist_event", ["--gradient-tracking"])
    assert all(not preset(n).gradient_tracking and preset(n).partition == "iid" for n in PRESETS)


def test_check_tracking_state():
    check_tracking_state({}, False, "decent")
    check_tracking_state({"gradient_tracking": True}, True, "decent")
    check_tracking_state({}, True, "event")                 # only decent carries tracking state
    with pytest.raises(ValueError, match="gradient-tracking"):
        check_tracking_state({}, True, "decent")
    with pytest.raises(ValueError, match="gradient-tracking"):
        check_tracking_state({"gradient_tracking": True}, False, "decent")


# ---------------------------------------------------------------------------------------- label shards
def _labels(n, classes=10, seed=5):
    return torch.randint(0, classes, (n,), generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("size,world", [(103, 4), (600, 3), (64, 8), (50, 1)])
def test_label_shards_are_disjoint_equal_identical_and_sorted(size, world):
    lab = _labels(size)
    local = size // world
    shards = []
    for r in range(world):
        s = ShardSampler(size, world, r, "sequential", seed=3, partition="label", labels=lab)
        other = ShardSampler(size, world, r, "sequential", seed=3, partition="label", labels=lab.clone())
        assert torch.equal(s.indices(), other.indices())           # every rank computes the same order
        shards.append(s.indices())
        assert len(shards[-1]) == local and s.local_size == local
    cat = torch.cat(shards)
    assert len(set(cat.tolist())) == world * local               # disjoint
    assert bool((lab[cat][1:] >= lab[cat][:-1]).all())           # sorted by class across the ranks
    # random mode permutes inside the same shard; reshuffling changes the permutation with the epoch
    for r in range(world):
        a = ShardSampler(size, world, r, "random", seed=3, partition="label", labels=lab)
        b = ShardSampler(size, world, r, "random", seed=3, partition="label", labels=lab, reshuffle=True)
        i0 = a.indices()
        assert sorted(i0.tolist()) == sorted(shards[r].tolist())
        a.set_epoch(1)
        assert torch.equal(a.indices(), i0)
        assert torch.equal(b.indices(), i0)
        b.set_epoch(1)
        i1 = b.indices()
        assert sorted(i1.tolist()) == sorted(i0.tolist())
        if local > 4:
            assert not torch.equal(i1, i0)


def test_label_shards_are_skewed():
    lab = _labels(1000)
    for r in range(4):
        s = ShardSampler(1000, 4, r, "random", partition="label", labels=lab)
        assert len(set(lab[s.indices()].tolist())) <= 4           # 10 classes over 4 ranks: at most 4 per rank


@pytest.mark.parametrize("mode", ["random", "sequential"])
def test_iid_indices_are_unchanged(mode):
    size, world = 103, 4
    for r in range(world):
        for reshuffle in (False, True):
            s = ShardSampler(size, world, r, mode, seed=7, reshuffle=reshuffle)
            t = ShardSampler(size, world, r, mode, seed=7, reshuffle=reshuffle, partition="iid", labels=_labels(size))
            for ep in (0, 1, 2):
                s.set_epoch(ep)
                t.set_epoch(ep)
                b, e = r * (size // world), (r + 1) * (size // world)
                if mode == "sequential":
                    want = torch.arange(b, e)
                else:
                    want = torch.randperm(size, generator=torch.Generator().manual_seed(7 + (ep if reshuffle else 0)))
                    want = want[b:e]
                assert torch.equal(s.indices(), want) and torch.equal(t.indices(), want)


def test_label_partition_needs_labels():
    with pytest.raises(ValueError, match="label"):
        ShardSampler(10, 2, 0, partition="label")


# ---------------------------------------------------------------------------------------- gloo
_PORT = [34300 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "tracking_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("world", [2, 3, 4])
def test_gloo_matches_simulator(world):
    rc, out = _torchrun(world, "--mode", "sim", "--steps", "9")
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_resume_is_exact_and_refuses_plain(tmp_path):
    rc, out = _torchrun(3, "--mode", "resume", "--ckpt-dir", str(tmp_path))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
