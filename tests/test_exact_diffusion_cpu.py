"""Exact diffusion (--exact-diffusion, decent on the ring): the simulator in float64 on heterogeneous quadratics
(phi_1 = sgd(theta_0), sum theta = sum psi, exact consensus at the minimiser where plain decent stays biased, also with
momentum, weight decay and Nesterov), the unchanged plain path, the gloo backend against the simulator bit for bit and a
checkpoint resume (tests/exact_diffusion_worker.py), and the configuration rules."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import TILE, ParamArena, TensorTable
from eventgrad_b200.parallel.base import check_exact_diffusion_state
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

    def sim(self, R, ed, lr=0.1, **kw):
        return RingSimulator(R, torch.zeros(self.table.n_padded, dtype=self.dtype), self.table, "decent", lr=lr,
                             momentum=kw.pop("momentum", 0.0), serial_skip=False, exact_diffusion=ed, **kw)


def _err(sim, want):
    return max(float((th - want).abs().max()) for th in sim.theta)


@pytest.mark.parametrize("R", [2, 3, 4, 5, 6])
def test_first_phi_is_sgd_and_sum_theta_equals_sum_psi(R):
    q = Quadratics(R)
    sim = q.sim(R, True)
    theta0 = sim.theta[0].clone()
    for k in range(1, 61):
        g = q.grads(sim.theta)
        sim.step(g)
        if k == 1:
            # psi = theta_0, so phi_1 = p_1 = sgd(theta_0): the adapt-then-combine step, and the inboxes hold it
            for r in range(R):
                p = theta0.clone()
                sgd_(p, g[r], None, 0.1, 0.0)
                assert torch.equal(sim.psi[r], p), f"rank {r}: phi_1 must be sgd(theta_0)"
                assert torch.equal(sim.inbox_r[(r - 1) % R], p) and torch.equal(sim.inbox_l[(r + 1) % R], p)
        dev = float((torch.stack(sim.theta).sum(0) - torch.stack(sim.psi).sum(0)).abs().max())
        assert dev < 1e-12, f"step {k}: |sum theta - sum psi| = {dev:.3e}"


@pytest.mark.parametrize("R", [2, 3, 4, 5, 6])
def test_exact_diffusion_reaches_the_global_minimiser_where_decent_does_not(R):
    q = Quadratics(R, seed=R)
    ed, dp = q.sim(R, True), q.sim(R, False)
    for _ in range(1500):
        ed.step(q.grads(ed.theta))
        dp.step(q.grads(dp.theta))
    assert _err(ed, q.opt) < 1e-10, _err(ed, q.opt)
    assert _err(dp, q.opt) > 1e-2, _err(dp, q.opt)          # constant-lr D-PSGD settles at a biased point
    for buf in ed.theta + ed.psi:
        assert bool((buf[q.mask == 0] == 0).all()), "padding lanes must stay zero"


@pytest.mark.parametrize("R", [2, 4, 5])
def test_exact_diffusion_with_momentum_weight_decay_and_nesterov_converges(R):
    """The optimizer is unchanged (weight decay, heavy-ball Nesterov momentum, all local): the fixed point is the
    minimiser of sum f_r + R wd/2 ||theta||^2."""
    wd = 0.05
    q = Quadratics(R, seed=9)
    sim = q.sim(R, True, lr=0.02, momentum=0.9, weight_decay=wd, nesterov=True)
    for _ in range(3000):
        sim.step(q.grads(sim.theta))
    sa = torch.stack(q.A).sum(0)
    want = torch.stack([a * c for a, c in zip(q.A, q.c)]).sum(0) / torch.where(q.mask > 0, sa + R * wd, 1.0)
    assert _err(sim, want) < 1e-10, _err(sim, want)
    assert all(bool((th[q.mask == 0] == 0).all()) for th in sim.theta)


def test_r1_is_plain_sgd():
    q = Quadratics(1)
    a, b = q.sim(1, True), q.sim(1, False)
    for _ in range(5):
        a.step(q.grads(a.theta))
        b.step(q.grads(b.theta))
    assert torch.equal(a.theta[0], b.theta[0]) and not a.ed
    assert not hasattr(a, "psi")


def test_exact_diffusion_off_is_the_plain_simulator():
    """exact_diffusion=False computes exactly what mix3_ + sgd_ compute per rank (the simulator before exact
    diffusion)."""
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    m = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    g = torch.Generator().manual_seed(2)
    theta0 = torch.randn(t.n_padded, generator=g) * m
    R = 3
    a = RingSimulator(R, theta0, t, "decent", lr=0.05, momentum=0.9, serial_skip=False)
    b = RingSimulator(R, theta0, t, "decent", lr=0.05, momentum=0.9, serial_skip=False, exact_diffusion=False)
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
    assert not hasattr(b, "psi") and not b.ed


def test_exact_diffusion_step_is_the_spec_and_costs_decents_bytes():
    """One step op for op as the spec writes it (fp32, momentum, R = 4), and decent's byte count."""
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    g = torch.Generator().manual_seed(5)
    R = 4
    theta0 = torch.randn(t.n_padded, generator=g)
    sim = RingSimulator(R, theta0, t, "decent", lr=0.05, momentum=0.9, serial_skip=False, exact_diffusion=True)
    th = [theta0.clone() for _ in range(R)]
    psi = [theta0.clone() for _ in range(R)]
    mom = [torch.zeros_like(theta0) for _ in range(R)]
    for s in range(4):
        gr = [torch.randn(t.n_padded, generator=g) for _ in range(R)]
        sim.step(gr)
        phi = []
        for r in range(R):
            p = th[r].clone()
            sgd_(p, gr[r], mom[r], 0.05, 0.9)
            phi.append(p.add(th[r].sub(psi[r])))
            psi[r] = p
        for r in range(R):
            tm = phi[r].clone().add_(phi[(r - 1) % R]).add_(phi[(r + 1) % R]).div_(3)
            th[r] = phi[r].add(tm).div_(2)
    for r in range(R):
        assert torch.equal(sim.theta[r], th[r]) and torch.equal(sim.psi[r], psi[r]) and torch.equal(sim.mom[r], mom[r])
    assert sim.bytes == [4 * 2 * t.n_elems * 4] * R
    assert sim.dense_messages() == 2 * t.n_tensors * 4 * R


@pytest.mark.parametrize("kw", [dict(algo="event"), dict(algo="spevent"), dict(algo="cent"), dict(offsets=(1, 2)),
                                dict(offsets="onepeer-exp"), dict(compress="int8"), dict(gradient_tracking=True),
                                dict(local_steps=2)])
def test_simulator_rejects_what_validate_rejects(kw):
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    algo = kw.pop("algo", "decent")
    with pytest.raises(ValueError, match="exact diffusion"):
        RingSimulator(5, torch.zeros(t.n_padded), t, algo, exact_diffusion=True, **kw)


# ---------------------------------------------------------------------------------------- configuration
def _ed(**kw):
    base = dict(algo="decent", exact_diffusion=True)
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("kw,match", [
    (dict(algo="event"), "stale phi"),
    (dict(algo="spevent"), "stale phi"),
    (dict(algo="cent"), "decent"),
    (dict(topology="exp"), "ring"),
    (dict(topology="1,2"), "ring"),
    (dict(topology="onepeer-exp"), "ring"),
    (dict(backend="refport"), "refport"),
    (dict(overlap_push=True), "overlap_push"),
    (dict(double_buffer=True), "double_buffer"),
    (dict(ce_push=True), "ce_push"),
    (dict(compress="int8"), "int8"),
    (dict(gradient_tracking=True), "gradient-tracking"),
    (dict(local_steps=2), "local-steps"),
    (dict(file_write=1), "file_write"),
])
def test_validation_rejects(kw, match):
    with pytest.raises(ValueError, match=match):
        _ed(**kw).validate()


def test_validation_accepts():
    _ed().validate()
    _ed(overlap_push=False, double_buffer=False, ce_push=False, backend="gloo", partition="label").validate()
    _ed(backend="nccl", weight_decay=1e-4, momentum=0.9, nesterov=True).validate()


def test_resolved_keeps_the_fused_single_slot_step():
    from eventgrad_b200.parallel.p2p import _wants_dbuf, _wants_ed, _wants_gt
    c = _ed().validate().resolved("cuda", 4)
    assert c.overlap_push is False and not _wants_dbuf(c) and _wants_ed(c, 4) and not _wants_gt(c, 4)
    assert not _wants_ed(c, 1)
    assert not _wants_ed(TrainConfig(algo="decent").validate(), 4)
    assert TrainConfig(algo="decent").validate().resolved("cuda", 4).overlap_push is True
    assert _wants_dbuf(TrainConfig(algo="decent", overlap_push=False).validate())


def test_layout_holds_psi_only_under_exact_diffusion():
    from eventgrad_b200.parallel.p2p import build_layout
    t = ParamArena(build_model("cnn2"), torch.device("cpu")).table
    on = build_layout(t, _ed(overlap_push=False).validate(), 4, 16)
    off = build_layout(t, TrainConfig(algo="decent", overlap_push=False, double_buffer=False).validate(), 4, 16)
    one = build_layout(t, _ed(overlap_push=False).validate(), 1, 16)
    assert on.sections["psi"][1] == t.n_padded * 4
    assert "psi" not in off.sections and "psi" not in one.sections
    assert on.sections["inbox_l"][1] == off.sections["inbox_l"][1] == t.n_padded * 4      # one slot: no double buffer


def test_cli_and_presets():
    c = parse_cli("decent", ["--exact-diffusion"])
    assert c.exact_diffusion and not c.gradient_tracking and c.local_steps == 1
    assert not parse_cli("decent", []).exact_diffusion
    with pytest.raises(ValueError, match="decent"):
        parse_cli("mnist_event", ["--exact-diffusion"])
    with pytest.raises(ValueError, match="gradient-tracking"):
        parse_cli("decent", ["--exact-diffusion", "--gradient-tracking"])
    assert all(not preset(n).exact_diffusion for n in PRESETS)


def test_check_exact_diffusion_state():
    check_exact_diffusion_state({}, False, "decent")
    check_exact_diffusion_state({"exact_diffusion": True}, True, "decent")
    check_exact_diffusion_state({}, True, "event")                 # only decent carries exact-diffusion state
    with pytest.raises(ValueError, match="exact-diffusion"):
        check_exact_diffusion_state({}, True, "decent")
    with pytest.raises(ValueError, match="exact-diffusion"):
        check_exact_diffusion_state({"exact_diffusion": True}, False, "decent")


# ---------------------------------------------------------------------------------------- gloo
_PORT = [34900 + (os.getpid() % 50) * 10]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "exact_diffusion_worker.py"), *args]
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
