"""The drift trigger (--trigger drift: a tensor fires when ||theta - sent|| >= thres, sent = what its receivers hold):
the oracle FSM, the simulator's invariants on the ring, a circulant graph and the one-peer graph, the gloo backend
against the simulator bit for bit (tests/drift_worker.py), checkpoint resume, and the configuration rules."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import ParamArena
from eventgrad_b200.parallel.base import check_trigger_state
from eventgrad_b200.parallel.trigger import TriggerConfig, TriggerState, drift_norms, trigger_step

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _table():
    return ParamArena(build_model("cnn2"), torch.device("cpu")).table


def _mask(t):
    m = torch.zeros(t.n_padded)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


# ---------------------------------------------------------------------------------------- the oracle FSM
def _norm_rule_reference(state, curr_norm, pass_num, cfg):
    """The norm-difference FSM step as it was before the drift metric existed (event.cpp:300-365), kept here to pin
    the default rule bit for bit."""
    curr = curr_norm.to(torch.float32)
    value_diff = (curr - state.last_norm).abs()
    iter_diff = torch.tensor(float(pass_num), dtype=torch.float32) - state.last_iter
    if cfg.thres_type == 1:
        state.thres.mul_(float(torch.tensor(cfg.horizon, dtype=torch.float32)))
    else:
        state.thres.fill_(float(torch.tensor(cfg.constant, dtype=torch.float32)))
    fire = value_diff >= state.thres
    if pass_num < cfg.initial_comm_passes:
        fire = torch.ones_like(fire)
    new_slope = value_diff / iter_diff
    shifted = torch.cat([state.slopes[:, 1:], new_slope[:, None]], dim=1)
    avg = shifted.double().sum(dim=1) / float(cfg.sent_history)
    state.slopes.copy_(torch.where(fire[:, None], shifted, state.slopes))
    if cfg.thres_type == 1:
        state.thres.copy_(torch.where(fire, avg.float(), state.thres))
    state.last_norm.copy_(torch.where(fire, curr, state.last_norm))
    state.last_iter.copy_(torch.where(fire, torch.full_like(curr, float(pass_num)), state.last_iter))
    return fire


def test_positional_config_and_default_metric():
    c = TriggerConfig(1, 0.9, 0.0, 3, 5)
    assert c.metric == "norm" and c.sent_history == 3 and c.initial_comm_passes == 5
    assert TriggerConfig.from_train(TrainConfig()).metric == "norm"
    assert TriggerConfig.from_train(TrainConfig(trigger="drift")).metric == "drift"


@pytest.mark.parametrize("thres_type", [0, 1])
def test_norm_metric_is_the_reference_rule_bit_for_bit(thres_type):
    g = torch.Generator().manual_seed(7)
    cfg = TriggerConfig(thres_type, 0.95, 0.3, 3, 4)
    assert cfg.metric == "norm"
    a, b = TriggerState(40, 3), TriggerState(40, 3)
    for k in range(1, 60):
        norms = torch.rand(40, generator=g) * (1 + k % 7)
        fa = trigger_step(a, norms, k, cfg)
        fb = _norm_rule_reference(b, norms, k, cfg)
        assert torch.equal(fa, fb)
        for name in ("thres", "last_norm", "last_iter", "slopes"):
            assert torch.equal(getattr(a, name), getattr(b, name)), (k, name)


@pytest.mark.parametrize("change", ["sign", "permute", "rotate"])
def test_norm_preserving_change_fires_only_under_drift(change):
    """A tensor whose norm stays fixed while its values change never fires under the norm rule with a constant
    threshold > 0, and fires under drift."""
    g = torch.Generator().manual_seed(1)
    sent = torch.randn(64, generator=g)
    if change == "sign":
        theta = -sent
    elif change == "permute":
        theta = sent[torch.randperm(64, generator=g)]
    else:     # a 2-D rotation of each pair (exact in norm up to rounding, so compare with the float norm itself)
        theta = torch.stack([-sent[1::2], sent[0::2]], 1).reshape(-1)
    assert float(torch.linalg.vector_norm(theta)) == float(torch.linalg.vector_norm(sent))
    offsets, numels = [0], [64]
    for metric in ("norm", "drift"):
        cfg = TriggerConfig(thres_type=0, constant=0.5, initial_comm_passes=2, metric=metric)
        st = TriggerState(1, cfg.sent_history)
        cur = sent
        fired = []
        for k in range(1, 6):
            val = torch.linalg.vector_norm(cur).reshape(1) if metric == "norm" else drift_norms(cur, sent, offsets, numels)
            fired.append(bool(trigger_step(st, val, k, cfg)[0]))
            cur = theta            # after the first (forced) send of `sent`, the tensor changes to theta and stays
        # step 1 is an initial communication pass; afterwards only the drift rule sees the change
        assert fired[0]
        assert any(fired[1:]) == (metric == "drift"), (metric, fired)


def test_drift_metric_feeds_the_drift_to_the_fsm():
    cfg = TriggerConfig(thres_type=1, horizon=1.0, sent_history=2, initial_comm_passes=1, metric="drift")
    st = TriggerState(3, 2)
    st.thres.fill_(0.5)
    d = torch.tensor([0.4, 0.5, 2.0])
    fire = trigger_step(st, d, 4, cfg)
    assert fire.tolist() == [False, True, True]
    # slope = drift / iter_diff for the fired tensors, threshold = slope history average
    assert torch.equal(st.slopes[:, 1], torch.tensor([0.0, 0.5 / 4, 2.0 / 4]))
    assert torch.equal(st.last_norm, torch.tensor([0.0, 0.5, 2.0]))


# ---------------------------------------------------------------------------------------- simulator invariants
def _constant_sim(R, topology, algo="event", c=0.05):
    torch.manual_seed(0)
    t = _table()
    theta0 = ParamArena(build_model("cnn2"), torch.device("cpu")).theta.clone()
    tcfg = TriggerConfig(thres_type=0, constant=c, initial_comm_passes=2, metric="drift")
    return RingSimulator(R, theta0, t, algo, tcfg, lr=0.05, momentum=0.9, serial_skip=False, offsets=topology), t


@pytest.mark.parametrize("R,topology", [(3, "ring"), (4, "ring"), (4, "exp"), (4, "onepeer-exp")])
def test_simulator_inboxes_hold_sent_and_held_tensors_are_within_threshold(R, topology):
    c = 0.05
    sim, t = _constant_sim(R, topology, c=c)
    assert sim.drift
    m = _mask(t)
    last_fire = [[0] * t.n_tensors for _ in range(R)]     # step of rank r's last firing of tensor i (0: never)
    held = fired = 0
    for s in range(1, 16):
        drift = [sim.trigger_norms(r) for r in range(R)]
        g = torch.Generator().manual_seed(s)
        sim.step([torch.randn(t.n_padded, generator=g) * 0.05 * m for _ in range(R)])
        for r in range(R):
            f = sim.fire_history[-1][r]
            assert bool((drift[r][~f] < c).all()), f"step {s} rank {r}: a held tensor had drift >= c"
            if s >= 2:
                assert bool((drift[r][f] >= c).all())
            held += int((~f).sum())
            fired += int(f.sum())
            gr = sim.graphs[r]
            outs = gr.out_slots()
            for i in range(t.n_tensors):
                if f[i]:
                    last_fire[r][i] = s
                if not last_fire[r][i]:
                    continue
                want = sim._flat(sim.sent[r], i)
                if sim.period:   # one-peer graph: the slot fed at the step of the last firing
                    feeds = [outs[gr.active(last_fire[r][i])]]
                else:
                    feeds = outs
                for p, j in feeds:
                    assert torch.equal(sim._flat(sim.inbox[p][j], i), want), (s, r, i, p, j)
    assert held > 0 and fired > R * t.n_tensors, (held, fired)


def test_simulator_spevent_replicas_equal_prev_under_drift():
    R = 3
    sim, t = _constant_sim(R, "ring", algo="spevent", c=0.02)
    assert sim.drift and sim.sent is sim.prev
    m = _mask(t)
    for s in range(1, 10):
        g = torch.Generator().manual_seed(s)
        sim.step([torch.randn(t.n_padded, generator=g) * 0.05 * m for _ in range(R)])
        for r in range(R):
            assert torch.equal(sim.rep_r[sim.left(r)], sim.prev[r])
            assert torch.equal(sim.rep_l[sim.right(r)], sim.prev[r])


def test_norm_override_still_drives_the_decision():
    R = 3
    sim, t = _constant_sim(R, "ring")
    sim.step([torch.zeros(t.n_padded)] * R)
    big = [torch.full((t.n_tensors,), 10.0)] * R
    sim.step([torch.zeros(t.n_padded)] * R, norms=big)
    assert all(bool(f.all()) for f in sim.fire_history[-1])
    small = [torch.zeros(t.n_tensors)] * R
    sim.step([torch.zeros(t.n_padded)] * R, norms=small)
    assert not any(bool(f.any()) for f in sim.fire_history[-1])


# ---------------------------------------------------------------------------------------- gloo vs the simulator
_PORT = [30400]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "drift_worker.py"), *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("algo,topology,world", [
    ("event", "ring", 2), ("event", "ring", 3), ("event", "ring", 4),
    ("event", "exp", 4), ("event", "exp", 5),
    ("event", "onepeer-exp", 4),
    ("spevent", "ring", 3),
])
def test_gloo_drift_matches_simulator_every_step(algo, topology, world):
    rc, out = _torchrun(world, "--mode", "sim", "--algo", algo, "--topology", topology)
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_gloo_drift_trainer_resume_is_exact_and_refuses_the_norm_trigger(tmp_path):
    rc, out = _torchrun(2, "--mode", "resume", "--ckpt-dir", str(tmp_path))
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


def test_checkpoint_trigger_key():
    check_trigger_state({}, "norm", "event")                       # checkpoints without the key are norm
    check_trigger_state({"trigger": "drift"}, "drift", "spevent")
    check_trigger_state({}, "drift", "decent")                     # no trigger, nothing to check
    with pytest.raises(ValueError, match="trigger"):
        check_trigger_state({}, "drift", "event")
    with pytest.raises(ValueError, match="trigger"):
        check_trigger_state({"trigger": "drift"}, "norm", "spevent")


# ---------------------------------------------------------------------------------------- configuration
def test_every_preset_defaults_to_the_norm_trigger():
    assert TrainConfig().trigger == "norm"
    for name in PRESETS:
        assert preset(name).trigger == "norm"
        assert parse_cli(name, []).trigger == "norm"


@pytest.mark.parametrize("program", ["mnist_event", "cifar_event", "cifar_spevent"])
def test_drift_accepted_for_event_programs(program):
    cfg = parse_cli(program, ["--trigger", "drift"])
    assert cfg.trigger == "drift"
    assert parse_cli(program, ["--trigger", "drift", "--topology", "exp"] if program != "cifar_spevent"
                     else ["--trigger", "drift", "--backend", "gloo"]).trigger == "drift"


@pytest.mark.parametrize("program", ["decent", "cent"])
def test_drift_rejected_without_a_trigger(program):
    with pytest.raises(ValueError, match="trigger"):
        parse_cli(program, ["--trigger", "drift"])


def test_drift_rejected_for_refport_file_write_and_unknown_names():
    with pytest.raises(ValueError, match="refport"):
        parse_cli("cifar_event", ["--trigger", "drift", "--backend", "refport"])
    with pytest.raises(ValueError, match="file_write"):
        parse_cli("mnist_event", ["1", "--trigger", "drift"])
    with pytest.raises(ValueError, match="trigger"):
        TrainConfig(trigger="l2").validate()
    with pytest.raises(SystemExit):
        parse_cli("cifar_event", ["--trigger", "l2"])
