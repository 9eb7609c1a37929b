"""Quasi-global momentum (--quasi-global-momentum): the qg_sgd_ oracle against an op-by-op numpy float32 update, the
simulator's fixed points on heterogeneous quadratics (QG settles where plain D-PSGD at lr does, heavy ball where plain
D-PSGD at lr / (1 - mu) does), the configuration rules, the checkpoint key, and the gloo backend against the simulator
bit for bit plus a Trainer resume (tests/qg_momentum_worker.py)."""
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
from eventgrad_b200.parallel.base import check_qg_state
from eventgrad_b200.parallel.trigger import qg_sgd_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


# ---------------------------------------------------------------------------------------- the oracle
def _np_qg(theta, theta_k, g, mh, lr, mu, wd, nesterov):
    """qg_sgd_elem of csrc/common.cuh, one rounded float32 op at a time (fma through float64, exact for fp32 inputs)."""
    fma = lambda x, y, z: f32(np.float64(x) * np.float64(y) + np.float64(z))
    lr, mu, wd = f32(lr), f32(mu), f32(wd)
    a = f32(mh * mu)
    d = fma(theta, wd, g) if wd != 0 else g
    m = f32(a + d)
    s = fma(m, mu, d) if nesterov else m
    out = fma(s, -lr, theta)
    if lr != 0:
        q = f32(f32(f32(theta_k - theta) / lr) + s)
        mh = f32(a + f32(f32(f32(1) - mu) * q))
    return out, mh


@pytest.mark.parametrize("wd,nesterov", [(0.0, False), (5e-4, False), (0.0, True), (5e-4, True)])
@pytest.mark.parametrize("lr", [0.05, 0.0123, 0.0])
def test_qg_sgd_matches_numpy_float32(wd, nesterov, lr):
    gen = torch.Generator().manual_seed(3)
    n = 4096
    th_k = torch.randn(n, generator=gen)
    th = th_k + torch.randn(n, generator=gen) * 1e-2        # the mix moved theta a little
    g = torch.randn(n, generator=gen) * 0.1
    mh = torch.randn(n, generator=gen) * 0.3
    want_th, want_m = np.empty(n, f32), np.empty(n, f32)
    for i in range(n):
        want_th[i], want_m[i] = _np_qg(th[i].numpy(), th_k[i].numpy(), g[i].numpy(), mh[i].numpy(), lr, 0.9, wd,
                                       nesterov)
    t, m = th.clone(), mh.clone()
    qg_sgd_(t, th_k, g, m, lr, 0.9, wd, nesterov)
    assert np.array_equal(t.numpy(), want_th) and np.array_equal(m.numpy(), want_m)
    if lr == 0.0:
        assert torch.equal(m, mh)                           # lr = 0: m_hat unchanged


def test_step_without_mix_is_an_ema_of_the_step_direction():
    gen = torch.Generator().manual_seed(5)
    th = torch.randn(2048, generator=gen)
    g = torch.randn(2048, generator=gen)
    mh = torch.randn(2048, generator=gen)
    mu = 0.9
    t, m = th.clone(), mh.clone()
    qg_sgd_(t, th, g, m, 0.05, mu, 0.0, False)
    s = mh * mu + g
    c = float(torch.tensor(1.0).sub_(mu))
    assert torch.equal(m, (mh * mu).add_(s.mul(c)))          # m_hat = mu m_hat + (1 - mu) s exactly


# ---------------------------------------------------------------------------------------- quadratics, float64
def _quadratic(R, dim=5, seed=0):
    """Heterogeneous least squares: f_r(x) = |A_r x - b_r|^2 / 2, shifted targets per rank."""
    gen = torch.Generator().manual_seed(seed)
    A = [torch.eye(dim, dtype=torch.float64) + 0.3 * torch.randn(dim, dim, generator=gen, dtype=torch.float64)
         for _ in range(R)]
    b = [torch.randn(dim, generator=gen, dtype=torch.float64) * 2 + 3 * r for r in range(R)]
    return A, b


def _fixed_point(W, A, b, lr):
    """Plain D-PSGD at `lr`: x = W x - lr grad(x), solved directly."""
    R, dim = len(A), A[0].shape[0]
    M = torch.eye(R * dim, dtype=torch.float64) - torch.kron(W, torch.eye(dim, dtype=torch.float64))
    rhs = torch.zeros(R * dim, dtype=torch.float64)
    for r in range(R):
        M[r * dim:(r + 1) * dim, r * dim:(r + 1) * dim] += lr * A[r].T @ A[r]
        rhs[r * dim:(r + 1) * dim] = lr * A[r].T @ b[r]
    return torch.linalg.solve(M, rhs).view(R, dim)


def _run_quadratic(R, topology, steps, lr, mu, quasi_global, nesterov=False, dtype=torch.float64):
    dim = 5
    A, b = _quadratic(R, dim)
    t = TensorTable.from_named([("x", torch.nn.Parameter(torch.zeros(dim)))], TILE)
    sim = RingSimulator(R, torch.zeros(t.n_padded, dtype=dtype), t, "decent", lr=lr, momentum=mu, nesterov=nesterov,
                        serial_skip=False, offsets=topology, quasi_global=quasi_global)
    Ad = [x.to(dtype) for x in A]
    bd = [x.to(dtype) for x in b]
    for _ in range(steps):
        grads = []
        for r in range(R):
            gr = torch.zeros(t.n_padded, dtype=dtype)
            x = sim.theta[r][:dim]
            gr[:dim] = Ad[r].T @ (Ad[r] @ x - bd[r])
            grads.append(gr)
        sim.step(grads)
    return sim, torch.stack([th[:dim] for th in sim.theta]), A, b


@pytest.mark.parametrize("R,topology", [(4, "ring"), (8, "exp")])
def test_fixed_points_on_heterogeneous_quadratics(R, topology):
    lr, mu, steps = 0.02, 0.9, 6000
    sim, x_qg, A, b = _run_quadratic(R, topology, steps, lr, mu, True)
    W = sim.mixing_matrix()
    _, x_qgn, _, _ = _run_quadratic(R, topology, steps, lr, mu, True, nesterov=True)
    _, x_hb, _, _ = _run_quadratic(R, topology, steps, lr, mu, False)
    assert float((x_qg - _fixed_point(W, A, b, lr)).abs().max()) < 1e-9
    assert float((x_qgn - _fixed_point(W, A, b, lr * (1 + mu))).abs().max()) < 1e-9
    assert float((x_hb - _fixed_point(W, A, b, lr / (1 - mu))).abs().max()) < 1e-9
    AtA = sum(a.T @ a for a in A)
    xstar = torch.linalg.solve(AtA, sum(a.T @ bb for a, bb in zip(A, b)))
    d_qg = float((x_qg - xstar).norm(dim=1).max())
    d_hb = float((x_hb - xstar).norm(dim=1).max())
    assert d_qg < d_hb, (d_qg, d_hb)


# ---------------------------------------------------------------------------------------- simulator and configuration
def test_simulator_rejects_what_validate_rejects():
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    z = torch.zeros(t.n_padded)
    for algo, kw in (("cent", dict(momentum=0.9)), ("decent", dict(momentum=0.0)),
                     ("decent", dict(momentum=0.9, compress="int8")), ("decent", dict(momentum=0.9,
                                                                                     gradient_tracking=True)),
                     ("decent", dict(momentum=0.9, exact_diffusion=True)),
                     ("decent", dict(momentum=0.9, global_avg_period=2))):
        with pytest.raises(ValueError, match="quasi-global"):
            RingSimulator(4, z, t, algo, quasi_global=True, **kw)


def _qg(**kw):
    base = dict(algo="decent", momentum=0.9, quasi_global_momentum=True)
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("kw,match", [
    (dict(momentum=0.0), "quasi-global-momentum needs --momentum"),
    (dict(algo="cent"), "quasi-global-momentum.*cent"),
    (dict(algo="event", sync_mode="async"), "quasi-global-momentum needs --sync-mode iter"),
    (dict(compress="int8"), "quasi-global-momentum.*int8"),
    (dict(gradient_tracking=True), "quasi-global-momentum.*gradient-tracking"),
    (dict(exact_diffusion=True), "quasi-global-momentum.*exact-diffusion"),
    (dict(global_avg_period=2), "quasi-global-momentum.*global-avg-period"),
    (dict(backend="refport"), "quasi-global-momentum.*refport"),
    (dict(ce_push=True), "quasi-global-momentum.*ce_push"),
])
def test_validation_rejects(kw, match):
    with pytest.raises(ValueError, match=match):
        _qg(**kw).validate()


def test_validation_accepts():
    for algo in ("decent", "event", "spevent"):
        _qg(algo=algo).validate()
    for topo in ("ring", "exp", "1,3", "onepeer-exp"):
        for algo in ("decent", "event"):
            _qg(algo=algo, topology=topo).validate()
    _qg(local_steps=2, nesterov=True, weight_decay=5e-4).validate()
    _qg(overlap_push=True, file_write=1).validate()
    _qg(double_buffer=True, backend="gloo").validate()
    _qg(algo="event", trigger="drift").validate()
    for algo in ("cent", "decent", "event", "spevent"):
        TrainConfig(algo=algo, momentum=0.0).validate()                 # off restricts nothing


def test_cli_and_presets():
    c = parse_cli("cifar_event", ["--quasi-global-momentum"])
    assert c.quasi_global_momentum and c.momentum == 0.9
    assert not parse_cli("cifar_event", []).quasi_global_momentum
    with pytest.raises(ValueError, match="quasi-global-momentum needs --momentum"):
        parse_cli("decent", ["--quasi-global-momentum"])               # the decent preset has momentum 0
    assert parse_cli("decent", ["--quasi-global-momentum", "--momentum", "0.9"]).quasi_global_momentum
    assert all(not preset(n).quasi_global_momentum for n in PRESETS)


def test_check_qg_state():
    check_qg_state({}, False, "decent")
    check_qg_state({"quasi_global_momentum": True}, True, "event")
    check_qg_state({}, True, "cent")                                     # only gossip algorithms carry it
    with pytest.raises(ValueError, match="quasi-global-momentum"):
        check_qg_state({}, True, "decent")
    with pytest.raises(ValueError, match="quasi-global-momentum"):
        check_qg_state({"quasi_global_momentum": True}, False, "spevent")


def test_checkpoint_key_only_when_on():
    import torch.distributed as dist
    from eventgrad_b200.parallel import Ring
    from eventgrad_b200.parallel.collective import CollectiveBackend
    assert not dist.is_initialized()
    for algo in ("decent", "event", "spevent"):
        for qg in (False, True):
            cfg = TrainConfig(algo=algo, device="cpu", backend="gloo", momentum=0.9,
                              quasi_global_momentum=qg).validate()
            be = CollectiveBackend(cfg, ParamArena(build_model("cnn2"), torch.device("cpu")), Ring(0, 1))
            assert ("quasi_global_momentum" in be.state_dict()) == qg


# ---------------------------------------------------------------------------------------- gloo
_PORT = [37300 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "qg_momentum_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("world,algo,topology,extra", [
    (2, "decent", "ring", []), (3, "decent", "ring", []), (4, "decent", "exp", []),
    (4, "decent", "onepeer-exp", []), (3, "decent", "ring", ["--local-steps", "2"]),
    (4, "decent", "exp", ["--local-steps", "2"]),
    (2, "event", "ring", []), (3, "event", "ring", ["--trigger", "drift"]), (4, "event", "exp", []),
    (4, "event", "onepeer-exp", ["--trigger", "drift"]),
    (3, "spevent", "ring", []), (4, "spevent", "ring", ["--trigger", "drift"]),
])
def test_gloo_matches_simulator(world, algo, topology, extra):
    rc, out = _torchrun(world, "--mode", "sim", "--algo", algo, "--topology", topology, *extra)
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_trainer_resume_is_exact_and_refuses_the_other_setting(tmp_path):
    rc, out = _torchrun(3, "--mode", "resume", "--ckpt-dir", str(tmp_path))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]
