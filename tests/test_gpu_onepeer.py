"""GPU: the time-varying one-peer exponential graph (--topology onepeer-exp) in the fused step kernel
(csrc/gossip_graph.cu with GraphSlots.period > 0), bit for bit against the simulator.  Multi-rank runs use R virtual
ranks on one GPU (ops.local_world.LocalWorld); the torchrun cases at the end need one GPU per rank and skip otherwise."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import TrainConfig
from eventgrad_b200.engine.lr_schedule import lr_table
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.trigger import TriggerConfig, trigger_step

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "onepeer-exp"

SPE = 3          # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=4)


def _cfg(algo, **kw):
    base = dict(algo=algo, dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", horizon=1.0, thres_type=1,
                initial_comm_passes=4, topology=NAME, **OPT)
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    return LocalWorld(cfg, R, lambda: build_model("cnn2"), grid_cap=grid_cap, table_mode=table_mode,
                      timeout_ns=5_000_000_000)


def _mask(t):
    m = torch.zeros(t.n_padded, device="cuda")
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


def _grads(w, R, seed):
    t = w.arenas[0].table
    m = _mask(t)
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(t.n_padded, generator=g, device="cuda") * 0.05 * m for _ in range(R)]


def _sim(cfg, w, R, table):
    return RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, cfg.algo, TriggerConfig.from_train(cfg),
                         lr=cfg.lr, momentum=cfg.momentum, serial_skip=False, weight_decay=cfg.weight_decay,
                         nesterov=cfg.nesterov, lr_table=table, offsets=NAME)


def _steps(R):
    tau = (R - 1).bit_length()
    return max(2 * tau + 1, 9)          # >= 2 periods + 1, and past the schedule's milestone at step 7


def _check_step(w, sim, R, algo, s, fires):
    for r, be in enumerate(w.backends):
        if algo == "event":
            assert torch.equal(fires[r], sim.fire_history[-1][r]), f"step {s} rank {r} fire mask differs"
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} rank {r} theta differs"
        assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s} rank {r} momentum differs"
        assert be.num_events() == (sim.events[r] if algo == "event" else 0), f"step {s} rank {r} events"
        assert be.bytes_sent() == sim.bytes[r], f"step {s} rank {r} bytes"


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("R", [2, 4, 5, 8])
@pytest.mark.parametrize("algo", ["decent", "event"])
def test_onepeer_step_bitwise_vs_simulator(algo, R, mode):
    """Every step: theta, momentum, trigger decisions and counters equal the simulator's.  The simulator runs its own
    trigger FSM on the kernel's norm-on-write results (checked against its own norms to rounding), so the kernel's fire
    masks are checked against the oracle FSM, not copied into it."""
    cfg = _cfg(algo)
    w = _world(cfg, R, table_mode=(mode == "table"))
    tau = (R - 1).bit_length()
    assert all(be.graph is not None and be.graph.period == tau for be in w.backends)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    n_fired, steps = 0, _steps(R)
    for s in range(1, steps + 1):
        norms = fires = None
        if algo == "event":
            fires = [be.fire.clone().bool().cpu() for be in w.backends]      # the kernel's decisions for this step
            norms = [be.cur_norm.clone().cpu() for be in w.backends]         # ... and the norms it took them from
            for r in range(R):
                torch.testing.assert_close(norms[r], sim._norms(sim.theta[r]), rtol=3e-6, atol=1e-7)
            n_fired += sum(int(f.sum()) for f in fires)
        g = _grads(w, R, 40 + s)
        w.step(g)
        sim.step([x.cpu() for x in g], norms=norms)
        torch.cuda.synchronize()
        _check_step(w, sim, R, algo, s, fires)
    for r, be in enumerate(w.backends):
        be.check_status()
        assert int(be.d_pass.item()) == steps
        if algo == "event":          # the decision the kernel already took for the next step
            nxt = trigger_step(sim.state[r].clone(), be.cur_norm.cpu(), sim.pass_num + 1, sim.tcfg)
            assert torch.equal(nxt, be.fire.bool().cpu())
    if algo == "event":
        assert sum(sim.events) == n_fired            # one message per fired tensor
        assert n_fired < steps * R * w.arenas[0].table.n_tensors
    else:
        assert all(b == steps * w.arenas[0].table.n_elems * 4 for b in sim.bytes)
    w.close()


def test_onepeer_exact_consensus_on_device():
    """R = 8, no learning (zero gradients, no momentum or weight decay), integer theta: after tau = 3 steps every rank
    holds the exact mean, bit for bit."""
    R = 8
    cfg = _cfg("decent", momentum=0.0, weight_decay=0.0, nesterov=False, lr_schedule="constant")
    w = _world(cfg, R)
    t = w.arenas[0].table
    m = _mask(t)
    g = torch.Generator(device="cuda").manual_seed(3)
    for r in range(R):
        w.arenas[r].theta.copy_(torch.randint(-64, 64, (t.n_padded,), generator=g, device="cuda").float() * m)
    torch.cuda.synchronize()
    mean = torch.stack([a.theta.double() for a in w.arenas]).mean(0)
    assert torch.equal(mean.float().double(), mean)
    zeros = [torch.zeros(t.n_padded, device="cuda") for _ in range(R)]
    for s in range(3):
        w.step(zeros)
        torch.cuda.synchronize()
        same = all(torch.equal(a.theta, mean.float()) for a in w.arenas)
        assert same == (s == 2), f"step {s + 1}"
    for be in w.backends:
        be.check_status()
    w.close()


@pytest.mark.parametrize("algo", ["decent", "event"])
def test_onepeer_captured_step_replays_the_cycle(algo):
    """Each rank's step captured ONCE in a CUDA graph and replayed 2 tau + 1 times equals the simulator: the active
    slot comes from the device step counter, so the same graph walks through every slot of the cycle."""
    R = 4
    cfg = _cfg(algo)
    w = _world(cfg, R)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    graphs = []
    torch.cuda.synchronize()
    for r in range(R):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            w.backends[r].launch()
        graphs.append(g)
    torch.cuda.synchronize()
    cur = torch.cuda.current_stream()
    for s in range(1, 2 * 2 + 2):
        fires = norms = None
        if algo == "event":
            fires = [be.fire.clone().bool().cpu() for be in w.backends]
            norms = [be.cur_norm.clone().cpu() for be in w.backends]
        gr = _grads(w, R, 20 + s)
        for r in range(R):
            w.arenas[r].grad.copy_(gr[r])
        for st in w.streams:
            st.wait_stream(cur)
        for r in range(R):
            with torch.cuda.stream(w.streams[r]):
                graphs[r].replay()
            w.backends[r].account_step()
        for st in w.streams:
            cur.wait_stream(st)
        torch.cuda.synchronize()
        sim.step([x.cpu() for x in gr], norms=norms)
        _check_step(w, sim, R, algo, s, fires)
    for be in w.backends:
        be.check_status()
    del graphs
    w.close()


@pytest.mark.parametrize("R", [4, 8])
def test_onepeer_async_event_runs_clean(R):
    """async (event only, as on every topology; no flags, reads whatever the slot holds): no bitwise claim, but a
    clean status word and one message per fired tensor."""
    algo = "event"
    cfg = _cfg(algo, sync_mode="async")
    w = _world(cfg, R)
    t = w.arenas[0].table
    fired = [0] * R
    nbytes = [0] * R
    steps = 12
    for s in range(steps):
        for r, be in enumerate(w.backends):
            f = be.fire.clone().bool().cpu()
            fired[r] += int(f.sum())
            nbytes[r] += sum(t.numels[i] * 4 for i in range(t.n_tensors) if f[i])
        w.step(_grads(w, R, 90 + s))
        torch.cuda.synchronize()
    for r, be in enumerate(w.backends):
        be.check_status()
        assert int(be.status.item()) == 0
        assert bool(torch.isfinite(w.arenas[r].theta).all())
        assert int(be.d_pass.item()) == steps
        assert be.num_events() == fired[r]
        assert be.bytes_sent() == nbytes[r]
    w.close()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [29900]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "onepeer_worker.py"), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "WORKER_OK" in out, out[-3000:]


def _need(world):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < world:
        pytest.skip(f"needs {world} GPUs, found {n}")


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("algo", ["decent", "event"])
def test_multigpu_p2p_onepeer_vs_simulator(algo, world):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", "p2p", "--algo", algo, "--steps", "9")


@pytest.mark.multigpu
@pytest.mark.parametrize("algo", ["decent", "event"])
def test_multigpu_nccl_onepeer_vs_simulator(algo):
    _need(4)
    _torchrun(4, "--mode", "sim", "--backend", "nccl", "--algo", algo, "--steps", "9")
