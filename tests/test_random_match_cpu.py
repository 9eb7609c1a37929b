"""Random pairwise matchings (parallel/topology.py RandomMatch, --topology random-match): the matching function against
literal pairs and its statistics, W_k and its expected contraction, the simulator's step, bytes, every rejection, the
CLI and the window layout, and the gloo backend against the simulator bit for bit (tests/random_match_worker.py),
including a checkpoint resume mid-run under the same seed and a refused resume under another."""
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
from eventgrad_b200.parallel.topology import (Graph, RandomMatch, match_pairs, match_partner, match_perm,
                                              parse_topology)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "random-match"


def _table():
    return ParamArena(build_model("cnn2"), torch.device("cpu")).table


def _mask(t):
    m = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


# ---------------------------------------------------------------------------------------- the matching
def test_golden_pairs():
    """Literal pairs of the definition (splitmix64 from (seed << 32) ^ k, Fisher-Yates, consecutive pairs)."""
    assert [match_pairs(0, 8, k) for k in range(1, 5)] == [
        [(4, 3), (2, 7), (5, 6), (0, 1)],
        [(5, 2), (7, 4), (1, 3), (0, 6)],
        [(7, 0), (1, 4), (2, 6), (3, 5)],
        [(6, 0), (5, 1), (7, 3), (4, 2)],
    ]
    assert [match_perm(7, 5, k) for k in range(1, 4)] == [[3, 4, 0, 1, 2], [1, 3, 4, 2, 0], [1, 0, 3, 4, 2]]
    assert [match_pairs(7, 5, k) for k in range(1, 4)] == [[(3, 4), (0, 1)], [(1, 3), (4, 2)], [(1, 0), (3, 4)]]
    assert match_partner(7, 5, 1, 2) is None and match_partner(7, 5, 2, 0) is None and match_partner(7, 5, 1, 4) == 3


@pytest.mark.parametrize("R", [2, 3, 4, 5, 6, 7, 8, 16, 33])
def test_every_step_is_a_perfect_matching(R):
    for seed in (0, 1, 2 ** 31 - 1):
        for k in range(1, 60):
            pairs = match_pairs(seed, R, k)
            seen = [x for p in pairs for x in p]
            assert len(pairs) == R // 2 and len(set(seen)) == len(seen) == 2 * (R // 2)
            idle = set(range(R)) - set(seen)
            assert len(idle) == R % 2
            for a, b in pairs:
                assert match_partner(seed, R, k, a) == b and match_partner(seed, R, k, b) == a
            for r in idle:
                assert match_partner(seed, R, k, r) is None


@pytest.mark.parametrize("R", [4, 5, 8])
def test_pair_frequencies_are_uniform(R):
    """Each of the R(R-1)/2 pairs is equally likely: chi^2 over 20 000 steps below the 0.999 quantile."""
    from scipy.stats import chi2
    n, cnt = 20000, {}
    for k in range(1, n + 1):
        for a, b in match_pairs(5, R, k):
            key = (min(a, b), max(a, b))
            cnt[key] = cnt.get(key, 0) + 1
    cells = R * (R - 1) // 2
    expect = n * (R // 2) / cells
    stat = sum((cnt.get((a, b), 0) - expect) ** 2 / expect for a in range(R) for b in range(a + 1, R))
    assert stat < chi2.ppf(0.999, cells - 1), stat


def test_topology_object_and_resolution():
    for R in (2, 3, 8):
        g = Graph.build(1, R, NAME, seed=9)
        assert isinstance(g, RandomMatch) and g.kind == NAME and not g.is_ring and g.fanout == 1 and g.seed == 9
        for k in range(1, 10):
            assert g.partner(k) == match_partner(9, R, k, 1)
    assert Graph.build(0, 1, NAME).is_ring and parse_topology(NAME, 1) == (1,)
    with pytest.raises(ValueError):
        parse_topology(NAME, 4)
    for bad in (-1, 2 ** 31, True, 1.5):
        with pytest.raises(ValueError):
            RandomMatch(0, 4, bad)
    with pytest.raises(ValueError):
        RandomMatch(0, 1025, 0)
    with pytest.raises(ValueError):
        RandomMatch(0, 4, 0).partner(0)           # steps are 1-based


# ---------------------------------------------------------------------------------------- W_k and contraction
def _W(R, seed, k):
    return [[Fraction(x) for x in RandomMatch(r, R, seed).mixing_row(k)] for r in range(R)]


@pytest.mark.parametrize("R", [2, 3, 4, 5, 8])
def test_W_is_symmetric_doubly_stochastic_and_idempotent(R):
    for k in range(1, 12):
        W = _W(R, 3, k)
        assert all(W[i][j] == W[j][i] for i in range(R) for j in range(R))
        assert all(sum(row) == 1 for row in W) and all(x >= 0 for row in W for x in row)
        W2 = [[sum(W[i][j] * W[j][c] for j in range(R)) for c in range(R)] for i in range(R)]
        assert W2 == W


@pytest.mark.parametrize("R", [4, 5, 6, 8])
def test_average_is_kept_in_float64_at_lr_zero(R):
    t = _table()
    sim = RingSimulator(R, torch.zeros(t.n_padded, dtype=torch.float64), t, "decent", lr=0.0, serial_skip=False,
                        offsets=NAME, topology_seed=4)
    g = torch.Generator().manual_seed(R)
    sim.theta = [torch.randn(t.n_padded, generator=g, dtype=torch.float64) * _mask(t) for _ in range(R)]
    mean0 = torch.stack(sim.theta).mean(0)
    for _ in range(25):
        sim.step([torch.zeros(t.n_padded, dtype=torch.float64)] * R)
        assert (torch.stack(sim.theta).mean(0) - mean0).abs().max() < 1e-12


@pytest.mark.parametrize("R", [4, 5, 6, 8])
def test_mean_contraction_matches_lambda2(R):
    """W_k is a projection, so ||W_k x||^2 = x^T W_k x, and its mean over the matchings is x^T E[W] x: for zero-mean x
    exactly lambda_2(E[W]) ||x||^2, (R-2)/(2(R-1)) for even R and 1/2 for odd R (E[W] has one eigenvalue on the
    zero-mean space).  The ratio over many steps must match it."""
    lam = (R - 2) / (2 * (R - 1)) if R % 2 == 0 else 0.5
    gen = torch.Generator().manual_seed(0)
    ratios = []
    for k in range(1, 4001):
        W = torch.tensor([RandomMatch(r, R, 1).mixing_row(k) for r in range(R)], dtype=torch.float64)
        x = torch.randn(R, generator=gen, dtype=torch.float64)
        x -= x.mean()
        ratios.append(float(((W @ x) ** 2).sum() / (x ** 2).sum()))
    mean = sum(ratios) / len(ratios)
    assert abs(mean - lam) < 0.02, (mean, lam)


# ---------------------------------------------------------------------------------------- simulator
def _sim(R, t, dtype=torch.float32, **kw):
    return RingSimulator(R, torch.zeros(t.n_padded, dtype=dtype), t, "decent", serial_skip=False, offsets=NAME,
                         topology_seed=kw.pop("seed", 2), **kw)


@pytest.mark.parametrize("R", [2, 3, 4, 5])
def test_partners_are_bitwise_equal_after_the_mix(R):
    t = _table()
    sim = _sim(R, t, lr=0.0)
    g = torch.Generator().manual_seed(1)
    sim.theta = [torch.randn(t.n_padded, generator=g) * _mask(t) for _ in range(R)]
    for k in range(1, 8):
        sim.step([torch.zeros(t.n_padded)] * R)
        for a, b in match_pairs(2, R, k):
            assert torch.equal(sim.theta[a], sim.theta[b])


def test_two_ranks_equal_onepeer_exp_bit_for_bit():
    t = _table()
    g = torch.Generator().manual_seed(3)
    th0 = torch.randn(t.n_padded, generator=g) * _mask(t)
    kw = dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=True)
    a = _sim(2, t, **kw)
    b = RingSimulator(2, th0, t, "decent", serial_skip=False, offsets="onepeer-exp", **kw)
    a.theta = [th0.clone(), (th0 * 0.5).clone()]
    b.theta = [th0.clone(), (th0 * 0.5).clone()]
    for s in range(6):
        grads = [torch.randn(t.n_padded, generator=g) * 0.1 * _mask(t) for _ in range(2)]
        a.step(grads)
        b.step(grads)
        for r in range(2):
            assert torch.equal(a.theta[r], b.theta[r]) and torch.equal(a.mom[r], b.mom[r])
    assert a.bytes == b.bytes


@pytest.mark.parametrize("R", [3, 4, 5])
def test_simulator_equals_explicit_mixes_plus_sgd(R):
    t = _table()
    kw = dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=True)
    sim = _sim(R, t, seed=6, **kw)
    g = torch.Generator().manual_seed(R)
    theta = [torch.randn(t.n_padded, generator=g) * _mask(t) for _ in range(R)]
    mom = [torch.zeros(t.n_padded) for _ in range(R)]
    sim.theta = [x.clone() for x in theta]
    from eventgrad_b200.parallel.trigger import sgd_
    for k in range(1, 7):
        grads = [torch.randn(t.n_padded, generator=g) * 0.1 * _mask(t) for _ in range(R)]
        snap = [x.clone() for x in theta]
        for r in range(R):
            p = match_partner(6, R, k, r)
            if p is not None:
                theta[r] = (theta[r] + snap[p]) / 2
            sgd_(theta[r], grads[r], mom[r], 0.05, 0.9, 5e-4, True)
        sim.step(grads)
        for r in range(R):
            assert torch.equal(sim.theta[r], theta[r]) and torch.equal(sim.mom[r], mom[r])
        W = sim.mixing_matrix(k)
        assert torch.equal(W, torch.tensor([RandomMatch(r, R, 6).mixing_row(k) for r in range(R)],
                                           dtype=torch.float64))


@pytest.mark.parametrize("R", [4, 5])
def test_bytes_events_and_dense_messages(R):
    t = _table()
    sim = _sim(R, t, lr=0.01)
    for k in range(1, 6):
        sim.step([torch.zeros(t.n_padded)] * R)
    for r in range(R):
        matched = sum(match_partner(2, R, k, r) is not None for k in range(1, 6))
        assert sim.bytes[r] == matched * t.n_elems * 4
    assert sim.events == [0] * R                       # decent counts no trigger events, on every topology
    assert sim.dense_messages() == t.n_tensors * 5 * R
    for bad in (dict(algo="event"), dict(compress="int8"), dict(gradient_tracking=True), dict(local_steps=2),
                dict(global_avg_period=2), dict(gossip_rounds=2), dict(exact_diffusion=True)):
        kw = dict(algo="decent")
        kw.update(bad)
        algo = kw.pop("algo")
        with pytest.raises(ValueError):
            RingSimulator(R, torch.zeros(t.n_padded), t, algo, offsets=NAME, **kw)


# ---------------------------------------------------------------------------------------- config / CLI / layout
def _ok(**kw):
    base = dict(algo="decent", topology=NAME)
    base.update(kw)
    return TrainConfig(**base).validate()


def test_allowed_combinations():
    _ok()
    _ok(topology_seed=2 ** 31 - 1, momentum=0.9, nesterov=True, weight_decay=1e-4, lr_schedule="cosine")
    _ok(cuda_graph=True, partition="label", consensus_every=5, grad_table=False)
    _ok(backend="gloo")
    _ok(backend="nccl")


@pytest.mark.parametrize("bad", [
    dict(algo="event"), dict(algo="spevent"), dict(algo="cent"), dict(algo="event", sync_mode="async"),
    dict(local_steps=2), dict(global_avg_period=2), dict(slowmo_period=2), dict(gossip_rounds=2),
    dict(compress="int8"), dict(compress="sign"), dict(compress="int8", choco_gamma=0.5), dict(gradient_tracking=True),
    dict(exact_diffusion=True), dict(quasi_global_momentum=True, momentum=0.9), dict(backend="refport"),
    dict(overlap_push=True), dict(double_buffer=True), dict(ce_push=True), dict(file_write=1),
    dict(topology_seed=-1), dict(topology_seed=2 ** 31), dict(topology_seed=True), dict(topology_seed=1.0)])
def test_rejections(bad):
    with pytest.raises(ValueError):
        _ok(**bad)


def test_async_decent_is_rejected_with_its_reason():
    c = TrainConfig(algo="decent", topology=NAME)
    object.__setattr__(c, "sync_mode", "async")
    with pytest.raises(ValueError):
        c.validate()


def test_resolution_and_cli():
    c = _ok(topology_seed=4)
    assert c.for_world(1).topology == "ring"
    for R in (2, 3, 8):
        r = c.resolved("cuda", R)
        assert r.topology == NAME and r.overlap_push is False and r.topology_seed == 4
        from eventgrad_b200.parallel.p2p import _wants_dbuf
        assert not _wants_dbuf(r)
    c = parse_cli("decent", ["0", "--topology", NAME, "--topology-seed", "17"])
    assert c.topology == NAME and c.topology_seed == 17
    assert parse_cli("decent", ["0"]).topology_seed == 0
    with pytest.raises(ValueError):
        parse_cli("decent", ["0", "--topology", NAME, "--topology-seed", "-3"])
    with pytest.raises(ValueError):
        parse_cli("cifar_event", ["0", "1", "1.0", "--topology", NAME])


def test_window_layout():
    from eventgrad_b200.parallel.p2p import build_layout
    t = _table()
    for R in (2, 3, 8):
        g = Graph.build(0, R, NAME)
        lay = build_layout(t, _ok(), R, 64, g)
        names = list(lay.sections)
        assert names[:5] == ["theta", "grad", "match_inbox", "match_flag", "match_done"], names
        assert not any(n.startswith(("inbox_", "flag_from_", "ack_from_")) for n in names)
        lay_c = build_layout(t, _ok(consensus_every=2), R, 64, g)
        names_c = list(lay_c.sections)
        assert names_c[-1] == "cons_part"


def test_checkpoint_state_carries_the_name_and_the_seed():
    from eventgrad_b200.parallel.base import check_topology_state
    m = Graph.build(0, 4, NAME, seed=3)
    sd = {"topology": NAME, "topology_seed": 3, "topology_offsets": []}
    check_topology_state(sd, m, "decent")
    for other in (Graph.build(0, 4, NAME, seed=4), Graph.build(0, 4, "ring"), Graph.build(0, 4, "onepeer-exp")):
        with pytest.raises(ValueError):
            check_topology_state(sd, other, "decent")
    with pytest.raises(ValueError):
        check_topology_state({}, m, "decent")


# ---------------------------------------------------------------------------------------- gloo, multi-process
_PORT = [35300 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "random_match_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("world", [2, 3, 4, 5])
def test_gloo_random_match_matches_simulator_every_step(world):
    rc, out = _torchrun(world, "--mode", "sim")
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_resume_continues_the_matchings_and_refuses_another_seed(tmp_path):
    rc, out = _torchrun(4, "--mode", "resume", "--ckpt-dir", str(tmp_path))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
