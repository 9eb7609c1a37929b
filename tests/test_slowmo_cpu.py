"""SlowMo (--slowmo-period tau, decent): the slowmo_sync_ oracle against an op-by-op numpy float32 update, the simulator
(beta = 0, alpha = 1 is Gossip-PGA or local SGD with periodic averaging; ranks agree after a sync; x and u agree across
ranks; the slow momentum accelerates an ill-conditioned quadratic; bytes), the configuration rules, the checkpoint keys,
and the gloo backend against the simulator bit for bit plus Trainer resumes (tests/slowmo_worker.py)."""
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
from eventgrad_b200.parallel.base import check_slowmo_state
from eventgrad_b200.parallel.trigger import rank_mean, sgd_, slowmo_sync_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPT = dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=True)
f32 = np.float32


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
    """Give every rank a different theta (ranks start from one theta_0; the first sync would hide nothing)."""
    gen = torch.Generator().manual_seed(seed)
    for th in sim.theta:
        th.add_(torch.randn(t.n_padded, generator=gen, dtype=th.dtype) * _mask(t, th.dtype))


# ---------------------------------------------------------------------------------------- the oracle
def _np_slowmo(x, u, avg, lr, beta, alpha):
    """slowmo_sync_kernel of csrc/allreduce.cu, one rounded float32 op at a time (fma through float64, exact for fp32
    inputs)."""
    fma = lambda a, b, c: f32(np.float64(a) * np.float64(b) + np.float64(c))
    lr, beta, alpha = f32(lr), f32(beta), f32(alpha)
    if lr == 0:
        return avg, u
    q = f32(f32(x - avg) / lr)
    u = f32(f32(beta * u) + q)
    c = f32(alpha * lr)
    return fma(u, -c, x), u


@pytest.mark.parametrize("beta,alpha", [(0.5, 1.0), (0.0, 1.0), (0.9, 0.7), (0.3, 1.3)])
@pytest.mark.parametrize("lr", [0.05, 0.0123, 0.0])
def test_slowmo_sync_matches_numpy_float32(beta, alpha, lr):
    gen = torch.Generator().manual_seed(3)
    n = 4096
    x = torch.randn(n, generator=gen)
    avg = x + torch.randn(n, generator=gen) * 1e-2          # the cycle moved the average a little
    u = torch.randn(n, generator=gen) * 0.3
    want_x, want_u = np.empty(n, f32), np.empty(n, f32)
    for i in range(n):
        want_x[i], want_u[i] = _np_slowmo(x[i].numpy(), u[i].numpy(), avg[i].numpy(), lr, beta, alpha)
    xx, uu = x.clone(), u.clone()
    slowmo_sync_(xx, uu, avg, lr, beta, alpha)
    assert np.array_equal(xx.numpy(), want_x) and np.array_equal(uu.numpy(), want_u)
    if lr == 0.0:
        assert torch.equal(uu, u) and torch.equal(xx, avg)    # lr = 0: u kept, x = theta_bar


def test_beta_zero_alpha_one_lands_on_the_average_up_to_rounding():
    gen = torch.Generator().manual_seed(4)
    x = torch.randn(4096, generator=gen, dtype=torch.float64)
    avg = x + torch.randn(4096, generator=gen, dtype=torch.float64) * 1e-2
    u = torch.randn(4096, generator=gen, dtype=torch.float64)
    slowmo_sync_(x, u, avg, 0.05, 0.0, 1.0)
    assert float((x - avg).abs().max()) < 1e-15


# ---------------------------------------------------------------------------------------- simulator
def _slowmo_sim(R, t, tau, H=1, topology="ring", dtype=torch.float32, beta=0.5, alpha=1.0, **kw):
    kw = {**dict(serial_skip=False, **OPT), **kw}
    return RingSimulator(R, torch.zeros(t.n_padded, dtype=dtype), t, "decent", offsets=topology, local_steps=H,
                         slowmo_period=tau, slowmo_beta=beta, slowmo_lr=alpha, **kw)


@pytest.mark.parametrize("topology,R", [("ring", 3), ("exp", 8), ("1,3", 8)])
@pytest.mark.parametrize("tau,H", [(2, 1), (3, 1), (3, 3)])
def test_sync_step_is_the_outer_update_then_sgd(topology, R, tau, H):
    t = _table()
    table = torch.linspace(0.05, 0.01, 11)
    sim = _slowmo_sim(R, t, tau, H, topology, beta=0.6, alpha=1.2, lr_table=table)
    _spread(sim, t, R * 10 + tau)
    for k in range(1, 3 * tau + 2):
        g = _grads(t, R, 70 + k)
        before = [(x.clone(), mo.clone()) for x, mo in zip(sim.theta, sim.mom)]
        xu = [(x.clone(), u.clone()) for x, u in zip(sim.slowmo_x, sim.slowmo_u)]
        inb = [[x.clone() for x in ib] for ib in sim.inbox]
        by = list(sim.bytes)
        sim.step(g)
        if k % tau:
            assert all(torch.equal(a, b[0]) and torch.equal(c, b[1])
                       for a, c, b in zip(sim.slowmo_x, sim.slowmo_u, xu)), "x or u changed off a sync step"
            if H == tau:                                   # local SGD base: the serial step, no bytes
                for r in range(R):
                    th, mo = before[r][0].clone(), before[r][1].clone()
                    sgd_(th, g[r], mo, float(table[k - 1]), OPT["momentum"], OPT["weight_decay"], OPT["nesterov"])
                    assert torch.equal(sim.theta[r], th) and sim.bytes[r] == by[r]
            continue
        avg = rank_mean([th for th, _ in before])
        for r in range(R):
            x, u = xu[r]
            slowmo_sync_(x, u, avg, float(table[k - 1]), 0.6, 1.2)
            th, mo = x.clone(), before[r][1]
            sgd_(th, g[r], mo, float(table[k - 1]), OPT["momentum"], OPT["weight_decay"], OPT["nesterov"])
            assert torch.equal(sim.slowmo_x[r], x) and torch.equal(sim.slowmo_u[r], u), f"step {k} rank {r}"
            assert torch.equal(sim.theta[r], th) and torch.equal(sim.mom[r], mo), f"step {k} rank {r}"
            assert all(torch.equal(a, b) for a, b in zip(sim.inbox[r], inb[r])), "a sync touched an inbox"
            assert sim.bytes[r] - by[r] == t.n_elems * 4


@pytest.mark.parametrize("topology,R", [("ring", 4), ("exp", 8), ("1,3", 8)])
@pytest.mark.parametrize("tau", [2, 3, 5])
def test_beta_zero_alpha_one_is_gossip_pga_with_gossip_base(topology, R, tau):
    """float64: SlowMo with beta = 0, alpha = 1 and local_steps 1 equals Gossip-PGA at P = tau to 1e-12."""
    t = _small_table()
    table = torch.linspace(0.05, 0.01, 4 * tau)
    kw = dict(serial_skip=False, offsets=topology, lr_table=table, **OPT)
    a = _slowmo_sim(R, t, tau, 1, topology, torch.float64, beta=0.0, alpha=1.0, lr_table=table)
    b = RingSimulator(R, torch.zeros(t.n_padded, dtype=torch.float64), t, "decent", global_avg_period=tau, **kw)
    for s in (a, b):
        _spread(s, t, 5)
    for k in range(1, 4 * tau + 1):
        g = _grads(t, R, 500 + k, torch.float64)
        a.step(g)
        b.step(g)
        for r in range(R):
            assert float((a.theta[r] - b.theta[r]).abs().max()) < 1e-12, f"step {k} rank {r}"
            assert float((a.mom[r] - b.mom[r]).abs().max()) < 1e-12
    assert a.bytes == b.bytes


@pytest.mark.parametrize("topology,R", [("ring", 4), ("exp", 8)])
@pytest.mark.parametrize("tau", [2, 4])
def test_beta_zero_alpha_one_is_local_sgd_with_averaging(topology, R, tau):
    """float64: SlowMo with beta = 0, alpha = 1 and local_steps tau equals hand-written local SGD whose ranks average
    their parameters at every tau-th step before the SGD step, to 1e-12."""
    t = _small_table()
    table = torch.linspace(0.05, 0.01, 4 * tau)
    sim = _slowmo_sim(R, t, tau, tau, topology, torch.float64, beta=0.0, alpha=1.0, lr_table=table)
    _spread(sim, t, 9)
    th = [x.clone() for x in sim.theta]
    mo = [torch.zeros_like(x) for x in th]
    for k in range(1, 4 * tau + 1):
        g = _grads(t, R, 900 + k, torch.float64)
        sim.step(g)
        if k % tau == 0:
            avg = torch.stack(th).mean(0)
            th = [avg.clone() for _ in range(R)]
        for r in range(R):
            sgd_(th[r], g[r], mo[r], float(table[k - 1]), OPT["momentum"], OPT["weight_decay"], OPT["nesterov"])
            assert float((sim.theta[r] - th[r]).abs().max()) < 1e-12, f"step {k} rank {r}"
    assert sim.bytes == [(4 * tau // tau) * t.n_elems * 4] * R


@pytest.mark.parametrize("topology,R,H", [("ring", 2, 1), ("ring", 5, 1), ("exp", 8, 1), ("ring", 4, 3)])
def test_zero_gradients_leave_every_rank_bit_identical_after_a_sync(topology, R, H):
    t = _table()
    # no weight decay: with it the momentum buffers would carry each rank's own wd * theta past the sync
    sim = _slowmo_sim(R, t, 3, H, topology, lr=0.05, momentum=0.9, nesterov=True, weight_decay=0.0)
    _spread(sim, t, R)
    zeros = [torch.zeros(t.n_padded) for _ in range(R)]
    for k in range(1, 10):
        sim.step(zeros)
        same = all(torch.equal(sim.theta[0], x) for x in sim.theta[1:])
        if k % 3 == 0:
            assert same, f"step {k}"
        elif k == 1:
            assert not same


@pytest.mark.parametrize("topology,R,tau,H", [("ring", 3, 2, 1), ("exp", 8, 3, 3), ("1,3", 8, 4, 1)])
def test_x_and_u_are_identical_on_every_rank(topology, R, tau, H):
    t = _table()
    sim = _slowmo_sim(R, t, tau, H, topology, beta=0.7)
    _spread(sim, t, 3)
    for k in range(1, 3 * tau + 1):
        sim.step(_grads(t, R, 40 + k))
        for r in range(1, R):
            assert torch.equal(sim.slowmo_x[0], sim.slowmo_x[r]) and torch.equal(sim.slowmo_u[0], sim.slowmo_u[r])
        if k % tau == 0:
            assert bool(sim.slowmo_u[0].abs().max() > 0)


def test_one_rank_is_an_outer_heavy_ball_on_its_own_trajectory():
    """R = 1: a sync step still applies the outer update, with theta_bar = theta_k, and counts no bytes."""
    t = _small_table()
    sim = _slowmo_sim(1, t, 3, 1, beta=0.5, lr=0.05, momentum=0.0, weight_decay=0.0, nesterov=False, serial_skip=True)
    th = sim.theta[0].clone()
    x, u = th.clone(), torch.zeros_like(th)
    for k in range(1, 10):
        g = _grads(t, 1, 60 + k)[0]
        sim.step([g])
        if k % 3 == 0:
            slowmo_sync_(x, u, th, 0.05, 0.5, 1.0)
            th.copy_(x)
        sgd_(th, g, None, 0.05, 0.0)
        assert torch.equal(sim.theta[0], th), f"step {k}"
    assert sim.bytes == [0] and bool(u.abs().max() > 0)


def _quadratic_run(beta, R=4, tau=8, lr=0.01, cycles=60, dim=16, H=1):
    """Ill-conditioned separable quadratic, float64: f_r(x) = sum_i c_i (x_i - b_ri)^2 / 2, curvatures c_i from 0.05 to
    5, each rank's optimum b_r shifted.  Returns the distance of the rank average to the global minimiser mean_r b_r."""
    t = TensorTable.from_named([("x", torch.nn.Parameter(torch.zeros(dim)))], TILE)
    c = torch.logspace(np.log10(0.05), np.log10(5.0), dim, dtype=torch.float64)
    gen = torch.Generator().manual_seed(1)
    b = [10.0 + torch.randn(dim, generator=gen, dtype=torch.float64) * 2 + r for r in range(R)]
    xstar = torch.stack(b).mean(0)
    sim = RingSimulator(R, torch.zeros(t.n_padded, dtype=torch.float64), t, "decent", lr=lr, momentum=0.0,
                        serial_skip=False, local_steps=H, slowmo_period=tau, slowmo_beta=beta, slowmo_lr=1.0)
    for _ in range(cycles * tau):
        grads = []
        for r in range(R):
            gr = torch.zeros(t.n_padded, dtype=torch.float64)
            gr[:dim] = c * (sim.theta[r][:dim] - b[r])
            grads.append(gr)
        sim.step(grads)
    return float((torch.stack([th[:dim] for th in sim.theta]).mean(0) - xstar).norm())


@pytest.mark.parametrize("H", [1, 8])
def test_slow_momentum_accelerates_an_ill_conditioned_quadratic(H):
    # the simulator gives 4.18 (beta = 0.8) against 17.09 (beta = 0) after 60 cycles, over either base
    d0, d8 = _quadratic_run(0.0, H=H), _quadratic_run(0.8, H=H)
    assert d8 < 0.3 * d0, (d8, d0)


@pytest.mark.parametrize("topology", ["ring", "exp", "1,3"])
@pytest.mark.parametrize("tau,H", [(2, 1), (3, 1), (7, 1), (3, 3)])
def test_bytes(topology, tau, H):
    R, K = 8, 15
    t = _table()
    sim = _slowmo_sim(R, t, tau, H, topology)
    for s in range(K):
        sim.step(_grads(t, R, s))
    syncs = K // tau
    per = 0 if H == tau else sim.fanout
    assert sim.bytes == [(syncs + (K - syncs) * per) * 4 * t.n_elems] * R
    assert sim.dense_messages() == sim.fanout * t.n_tensors * K * R        # per-step definition, unchanged


@pytest.mark.parametrize("kw", [
    dict(algo="event"), dict(algo="spevent"), dict(algo="cent"), dict(compress="int8"),
    dict(gradient_tracking=True), dict(exact_diffusion=True), dict(local_steps=2), dict(offsets="onepeer-exp"),
    dict(global_avg_period=2), dict(quasi_global=True, momentum=0.9), dict(slowmo_beta=1.0), dict(slowmo_beta=-0.1),
    dict(slowmo_lr=0.0), dict(lr=0.0),
])
def test_simulator_rejects_what_validate_rejects(kw):
    t = _table()
    algo = kw.pop("algo", "decent")
    with pytest.raises(ValueError, match="slowmo"):
        RingSimulator(4, torch.zeros(t.n_padded), t, algo, slowmo_period=3, **kw)
    for bad in (1, -1, 2.5, True):
        with pytest.raises(ValueError, match="slowmo_period"):
            RingSimulator(4, torch.zeros(t.n_padded), t, "decent", slowmo_period=bad)


# ---------------------------------------------------------------------------------------- configuration
def _sm(**kw):
    base = dict(algo="decent", slowmo_period=4)
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("kw,match", [
    (dict(slowmo_period=1), "slowmo-period 1.*cent"),
    (dict(slowmo_period=-2), "slowmo-period"),
    (dict(slowmo_period=2.5), "slowmo-period"),
    (dict(slowmo_period=True), "slowmo-period"),
    (dict(slowmo_beta=1.0), "slowmo-beta"),
    (dict(slowmo_beta=-0.5), "slowmo-beta"),
    (dict(slowmo_lr=0.0), "slowmo-lr"),
    (dict(slowmo_lr=-1.0), "slowmo-lr"),
    (dict(lr=0.0), "slowmo-period 4 needs --lr > 0"),
    (dict(algo="cent"), "slowmo-period 4 needs algo decent.*cent"),
    (dict(algo="event"), "slowmo-period 4 needs algo decent.*event"),
    (dict(algo="spevent"), "slowmo-period 4 needs algo decent.*spevent"),
    (dict(topology="onepeer-exp"), "slowmo-period.*onepeer-exp"),
    (dict(local_steps=2), "slowmo-period 4 needs --local-steps 1.*or 4"),
    (dict(local_steps=8), "slowmo-period 4 needs --local-steps 1.*or 4"),
    (dict(global_avg_period=2), "slowmo-period.*global-avg-period"),
    (dict(gradient_tracking=True), "slowmo-period.*gradient-tracking"),
    (dict(exact_diffusion=True), "slowmo-period.*exact-diffusion"),
    (dict(compress="int8"), "slowmo-period.*int8"),
    (dict(quasi_global_momentum=True, momentum=0.9), "slowmo-period.*quasi-global-momentum"),
    (dict(backend="refport"), "slowmo-period.*refport"),
    (dict(overlap_push=True), "slowmo-period.*overlap_push"),
    (dict(double_buffer=True), "slowmo-period.*double_buffer"),
    (dict(ce_push=True), "slowmo-period.*ce_push"),
    (dict(file_write=1), "slowmo-period.*file_write"),
])
def test_validation_rejects(kw, match):
    with pytest.raises(ValueError, match=match):
        _sm(**kw).validate()


def test_validation_accepts():
    for topo in ("ring", "1", "exp", "1,3", "2,3"):
        for tau in (2, 3, 100):
            for H in (1, tau):
                _sm(topology=topo, slowmo_period=tau, local_steps=H).validate()
    _sm(overlap_push=False, double_buffer=False, ce_push=False, backend="gloo", slowmo_beta=0.0).validate()
    _sm(backend="nccl", momentum=0.9, nesterov=True, weight_decay=5e-4, partition="label", slowmo_lr=2.0).validate()
    for algo in ("cent", "decent", "event", "spevent"):
        TrainConfig(algo=algo, slowmo_period=0, slowmo_beta=5.0, slowmo_lr=-1.0).validate()    # off restricts nothing


def test_resolved_keeps_the_fused_single_slot_step():
    from eventgrad_b200.parallel.p2p import _wants_dbuf
    for topo in ("ring", "exp"):
        for H in (1, 4):
            c = _sm(topology=topo, local_steps=H).validate().resolved("cuda", 8)
            assert c.overlap_push is False and not _wants_dbuf(c)
    assert TrainConfig(algo="decent").validate().resolved("cuda", 4).overlap_push is True


def test_cli_and_presets():
    c = parse_cli("decent", ["--slowmo-period", "4", "--slowmo-beta", "0.7", "--slowmo-lr", "1.5", "--local-steps",
                             "4", "--topology", "exp"])
    assert (c.slowmo_period, c.slowmo_beta, c.slowmo_lr, c.local_steps) == (4, 0.7, 1.5, 4)
    d = parse_cli("decent", [])
    assert (d.slowmo_period, d.slowmo_beta, d.slowmo_lr) == (0, 0.5, 1.0)
    for prog in ("mnist_event", "cent"):
        with pytest.raises(ValueError, match="slowmo-period"):
            parse_cli(prog, ["--slowmo-period", "2"])
    with pytest.raises(ValueError, match="cent"):
        parse_cli("decent", ["--slowmo-period", "1"])
    with pytest.raises(ValueError, match="slowmo-beta"):
        parse_cli("decent", ["--slowmo-period", "2", "--slowmo-beta", "1"])
    assert all(preset(n).slowmo_period == 0 for n in PRESETS)


def test_check_slowmo_state():
    check_slowmo_state({}, 0, 0.5, 1.0, "decent")                  # no key: never ran SlowMo
    sd = {"slowmo_period": 4, "slowmo_beta": 0.7, "slowmo_lr": 1.5}
    check_slowmo_state(sd, 4, 0.7, 1.5, "decent")
    check_slowmo_state({}, 4, 0.7, 1.5, "event")                   # only decent carries it
    with pytest.raises(ValueError, match="slowmo-period 0"):
        check_slowmo_state({}, 4, 0.7, 1.5, "decent")
    for run in ((0, 0.5, 1.0), (2, 0.7, 1.5), (4, 0.5, 1.5), (4, 0.7, 1.0)):
        with pytest.raises(ValueError, match="slowmo-period 4"):
            check_slowmo_state(sd, *run, "decent")


def test_checkpoint_keys_only_when_on():
    import torch.distributed as dist
    from eventgrad_b200.parallel import Ring
    from eventgrad_b200.parallel.collective import CollectiveBackend
    assert not dist.is_initialized()
    keys = {"slowmo_period", "slowmo_beta", "slowmo_lr", "slowmo_x", "slowmo_u"}
    for tau in (0, 3):
        cfg = TrainConfig(algo="decent", device="cpu", backend="gloo", slowmo_period=tau).validate()
        be = CollectiveBackend(cfg, ParamArena(build_model("cnn2"), torch.device("cpu")), Ring(0, 1))
        sd = be.state_dict()
        assert (keys & set(sd)) == (keys if tau else set())
        if tau:
            assert torch.equal(sd["slowmo_x"], be.arena.theta) and not bool(sd["slowmo_u"].any())


# ---------------------------------------------------------------------------------------- gloo
_PORT = [38300 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "slowmo_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("tau,H", [(2, 1), (3, 3)])
@pytest.mark.parametrize("world,topology", [(2, "ring"), (3, "ring"), (4, "ring"), (4, "exp")])
def test_gloo_matches_simulator(world, topology, tau, H):
    rc, out = _torchrun(world, "--mode", "sim", "--topology", topology, "--slowmo-period", str(tau), "--local-steps",
                        str(H), "--slowmo-beta", "0.7", "--slowmo-lr", "1.2")
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


@pytest.mark.parametrize("tau,H", [(3, 1), (5, 5)])
def test_gloo_trainer_resume_is_exact_and_refuses_other_settings(tmp_path, tau, H):
    """Checkpoint at step 5: one step before a sync (tau = 3, gossip base) and at a sync (tau = 5, local SGD base)."""
    rc, out = _torchrun(3, "--mode", "resume", "--ckpt-dir", str(tmp_path), "--slowmo-period", str(tau),
                        "--local-steps", str(H))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
