"""GPU: circulant gossip graphs beyond the ring in the fused step kernel (csrc/gossip_graph.cu), bit for bit against
the simulator.  Multi-rank runs use R virtual ranks on one GPU (ops.local_world.LocalWorld); the torchrun cases at the
end need one GPU per rank and skip otherwise."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import TrainConfig
from eventgrad_b200.engine.lr_schedule import lr_table
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.topology import parse_topology
from eventgrad_b200.parallel.trigger import TriggerConfig

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SPE = 3          # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=4)


def _cfg(algo, topology, **kw):
    base = dict(algo=algo, dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", horizon=1.0, thres_type=1,
                initial_comm_passes=4, topology=topology, **OPT)
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    return LocalWorld(cfg, R, lambda: build_model("cnn2"), grid_cap=grid_cap, table_mode=table_mode,
                      timeout_ns=5_000_000_000)


def _grads(w, R, seed):
    t = w.arenas[0].table
    m = torch.zeros(t.n_padded, device="cuda")
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(t.n_padded, generator=g, device="cuda") * 0.05 * m for _ in range(R)]


def _sim(cfg, w, R, table):
    return RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, cfg.algo, TriggerConfig.from_train(cfg),
                         lr=cfg.lr, momentum=cfg.momentum, serial_skip=False, weight_decay=cfg.weight_decay,
                         nesterov=cfg.nesterov, lr_table=table, offsets=cfg.topology)


CASES = [(4, "exp"), (5, "exp"), (8, "exp"), (5, "2")]


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("R,topology", CASES)
@pytest.mark.parametrize("algo", ["decent", "event"])
def test_graph_step_bitwise_vs_simulator(algo, R, topology, mode):
    """Every step: theta, momentum, trigger decisions and counters equal the simulator's.  The simulator runs its own
    trigger FSM on the kernel's norm-on-write results (which must match its own norms to rounding), so the kernel's
    fire masks are checked against the oracle FSM, not copied into it."""
    from eventgrad_b200.parallel.trigger import trigger_step
    cfg = _cfg(algo, topology)
    w = _world(cfg, R, table_mode=(mode == "table"))
    assert all(be.graph is not None and be.graph.offsets == parse_topology(topology, R) for be in w.backends)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    n_fired = 0
    for s in range(10):
        norms = None
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
        for r, be in enumerate(w.backends):
            if algo == "event":
                assert torch.equal(fires[r], sim.fire_history[-1][r]), f"step {s + 1} rank {r} fire mask differs"
            assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s + 1} rank {r} theta differs"
            assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s + 1} rank {r} momentum differs"
            assert be.num_events() == (sim.events[r] if algo == "event" else 0), f"step {s + 1} rank {r} events"
            assert be.bytes_sent() == sim.bytes[r], f"step {s + 1} rank {r} bytes"
    for r, be in enumerate(w.backends):
        be.check_status()
        assert int(be.d_pass.item()) == 10
        if algo == "event":          # the decision the kernel already took for step 11
            nxt = trigger_step(sim.state[r].clone(), be.cur_norm.cpu(), sim.pass_num + 1, sim.tcfg)
            assert torch.equal(nxt, be.fire.bool().cpu())
    if algo == "event":
        n = w.backends[0].graph.n_slots
        assert sum(sim.events) == n * n_fired
        # the trigger really skipped messages after the warm-up (otherwise this is decent with extra steps)
        assert n_fired < 10 * R * w.arenas[0].table.n_tensors
    w.close()


@pytest.mark.parametrize("R", [4, 8])
def test_graph_async_event_runs_clean(R):
    """async (reference RMA semantics: no flags, reads whatever the inboxes hold): no bitwise claim."""
    cfg = _cfg("event", "exp", sync_mode="async")
    w = _world(cfg, R)
    for s in range(20):
        w.step(_grads(w, R, 90 + s))
    torch.cuda.synchronize()
    for r, be in enumerate(w.backends):
        be.check_status()
        assert int(be.status.item()) == 0
        assert bool(torch.isfinite(w.arenas[r].theta).all())
        assert int(be.d_pass.item()) == 20
    w.close()


@pytest.mark.parametrize("R,topology", [(4, "exp"), (5, "2")])
def test_final_average_after_graph_run(R, topology):
    cfg = _cfg("decent", topology)
    w = _world(cfg, R, grid_cap=8)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    for s in range(6):
        g = _grads(w, R, 60 + s)
        w.step(g)
        sim.step([x.cpu() for x in g])
    torch.cuda.synchronize()
    for r in range(R):
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r])
    w.final_average()
    want = sim.final_average()
    for r in range(R):
        got = w.arenas[r].theta.cpu()
        assert torch.allclose(got, want, rtol=1e-6, atol=1e-7), (got - want).abs().max()
    w.close()


@pytest.mark.parametrize("algo", ["decent", "event"])
def test_graph_step_cuda_graph_replay_equals_eager(algo):
    """Each rank's step captured once in a CUDA graph and replayed (the kernel spins on its peers' flags from inside
    the graph; the step counter is device resident) equals eager execution bit for bit."""
    R = 4
    cfg = _cfg(algo, "exp")
    eager, graphed = _world(cfg, R), _world(cfg, R)
    table = lr_table(cfg, SPE)
    for w in (eager, graphed):
        for be in w.backends:
            be.set_lr_table(table)
    graphs = []
    torch.cuda.synchronize()
    for r in range(R):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            graphed.backends[r].launch()
        graphs.append(g)
    torch.cuda.synchronize()
    cur = torch.cuda.current_stream()
    for s in range(8):
        gr = _grads(eager, R, 20 + s)
        eager.step(gr)
        for r in range(R):
            graphed.arenas[r].grad.copy_(gr[r])
        for st in graphed.streams:
            st.wait_stream(cur)
        for r in range(R):
            with torch.cuda.stream(graphed.streams[r]):
                graphs[r].replay()
            graphed.backends[r].account_step()
        for st in graphed.streams:
            cur.wait_stream(st)
        torch.cuda.synchronize()
        for r in range(R):
            assert torch.equal(graphed.arenas[r].theta, eager.arenas[r].theta), f"step {s + 1} rank {r}"
            assert torch.equal(graphed.backends[r].fire, eager.backends[r].fire)
    for r in range(R):
        graphed.backends[r].check_status()
        eager.backends[r].check_status()
        assert graphed.backends[r].num_events() == eager.backends[r].num_events()
    del graphs
    eager.close()
    graphed.close()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [29800]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "topology_worker.py"), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "WORKER_OK" in out, out[-3000:]


def _need(world):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < world:
        pytest.skip(f"needs {world} GPUs, found {n}")


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [4, 8])
@pytest.mark.parametrize("algo", ["decent", "event"])
def test_multigpu_p2p_exp_vs_simulator(algo, world):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", "p2p", "--algo", algo, "--topology", "exp", "--steps", "10")


@pytest.mark.multigpu
@pytest.mark.parametrize("algo", ["decent", "event"])
def test_multigpu_nccl_exp_vs_simulator(algo):
    _need(4)
    _torchrun(4, "--mode", "sim", "--backend", "nccl", "--algo", algo, "--topology", "exp", "--steps", "8")
