"""GPU: SlowMo (--slowmo-period tau, decent) -- the step-gated sync kernel of csrc/allreduce.cu (two-shot average of theta
and the outer update of x and u in one launch) before the fused ring step kernel (csrc/gossip.cu) or the graph step
kernel (csrc/gossip_graph.cu), bit for bit against the simulator.  Multi-rank runs use R virtual ranks on one GPU
(ops.local_world.LocalWorld); the torchrun cases at the end need one GPU per rank and skip otherwise."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import TrainConfig
from eventgrad_b200.engine.lr_schedule import lr_table
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SPE = 3          # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=12)


def _cfg(topology="ring", tau=2, H=1, **kw):
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", topology=topology,
                slowmo_period=tau, local_steps=H, slowmo_beta=0.7, slowmo_lr=1.2, **OPT)
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, model_fn=None, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    w = LocalWorld(cfg, R, model_fn or (lambda: build_model("cnn2")), grid_cap=grid_cap, table_mode=table_mode,
                   timeout_ns=5_000_000_000)
    assert all(be.slowmo_period == cfg.slowmo_period and be.sm is not None and not be.overlap and not be.dbuf
               for be in w.backends)
    assert all(be.slowmo_local == (cfg.local_steps == cfg.slowmo_period) for be in w.backends)
    return w


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
    return RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, "decent", lr=cfg.lr, momentum=cfg.momentum,
                         serial_skip=False, weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table,
                         offsets=w.cfg.topology, local_steps=cfg.local_steps, slowmo_period=cfg.slowmo_period,
                         slowmo_beta=cfg.slowmo_beta, slowmo_lr=cfg.slowmo_lr)


def _inboxes(be):
    """(simulator slot, device buffer) pairs: the graph's slots, or the ring's from-left / from-right inboxes (the
    2-rank ring keeps its single copy in inbox_r)."""
    if be.graph is not None:
        return [(s, be.win.view(f"inbox_{s}", torch.float32)) for s in range(be.graph.n_slots)]
    out = [(1, be.win.view("inbox_r", torch.float32))]
    if not be.wire_dedup:
        out.append((0, be.win.view("inbox_l", torch.float32)))
    return out


def _check(w, sim, s, m):
    for r, be in enumerate(w.backends):
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} rank {r} theta"
        assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s} rank {r} momentum"
        assert torch.equal(be.slowmo_x.cpu(), sim.slowmo_x[r]), f"step {s} rank {r} x"
        assert torch.equal(be.slowmo_u.cpu(), sim.slowmo_u[r]), f"step {s} rank {r} u"
        for slot, buf in _inboxes(be):
            assert torch.equal(buf[:sim.theta[r].numel()].cpu(), sim.inbox[r][slot]), f"step {s} rank {r} slot {slot}"
        assert be.bytes_sent() == sim.bytes[r], f"step {s} rank {r} bytes"
        assert bool((w.arenas[r].theta[m == 0] == 0).all()), f"step {s} rank {r}: padding of theta is not zero"


def _run(cfg, R, table_mode=False, steps=None, model_fn=None, grid_cap=6, grad_seed=40):
    tau = cfg.slowmo_period
    w = _world(cfg, R, model_fn, table_mode, grid_cap)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    m = _mask(w.arenas[0].table)
    steps = steps or max(2 * tau + 1, 9)      # two cycles, and past the schedule's milestone at step 7
    for s in range(1, steps + 1):
        g = _grads(w, R, grad_seed + s)
        w.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        _check(w, sim, s, m)
        # the gate skipped every launch between syncs without touching the sync kernel's launch counter
        assert all(int(be.ar_ctr.item()) == s // tau for be in w.backends), f"step {s}"
    for be in w.backends:
        be.check_status()
        assert int(be.d_pass.item()) == steps
    w.close()


_CASES = [(R, topo) for R in (2, 3, 4, 8) for topo in ("ring", "exp")] + [(8, "1,3")]


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("base", ["gossip", "local"])
@pytest.mark.parametrize("tau", [2, 3, 5])
@pytest.mark.parametrize("R,topology", _CASES)
def test_slowmo_bitwise_vs_simulator(R, topology, tau, base, mode):
    """Every step: theta, momentum, x, u, every inbox and the byte counter equal the simulator's."""
    _run(_cfg(topology, tau, 1 if base == "gossip" else tau), R, table_mode=(mode == "table"))


@pytest.mark.parametrize("base", ["gossip", "local"])
def test_slowmo_one_rank(base):
    """R = 1 (CIFAR: no self-exchange): the sync kernel runs with a world of one and applies the outer update."""
    tau = 3
    cfg = _cfg("ring", tau, 1 if base == "gossip" else tau, dataset="cifar10")
    w = _world(cfg, 1)
    table = lr_table(cfg, SPE)
    w.backends[0].set_lr_table(table)
    sim = RingSimulator(1, w.arenas[0].theta.cpu(), w.arenas[0].table, "decent", lr=cfg.lr, momentum=cfg.momentum,
                        serial_skip=True, weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table,
                        local_steps=cfg.local_steps, slowmo_period=tau, slowmo_beta=cfg.slowmo_beta,
                        slowmo_lr=cfg.slowmo_lr)
    for s in range(1, 2 * tau + 2):
        g = _grads(w, 1, 80 + s)
        w.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        be = w.backends[0]
        assert torch.equal(w.arenas[0].theta.cpu(), sim.theta[0]), f"step {s}"
        assert torch.equal(be.slowmo_x.cpu(), sim.slowmo_x[0]) and torch.equal(be.slowmo_u.cpu(), sim.slowmo_u[0])
        assert be.bytes_sent() == 0 and int(be.ar_ctr.item()) == s // tau
    w.close()


@pytest.mark.parametrize("R,topology,mode,base", [(2, "ring", "flat", "gossip"), (4, "ring", "table", "local"),
                                                  (4, "exp", "flat", "gossip"), (8, "ring", "flat", "local")])
def test_slowmo_resnet18_at_the_full_persistent_grid(R, topology, mode, base):
    """The ResNet-18 `ref` arena (86 tensors, 8 569 tiles) at the co-resident grid of the kernels in use, tau = 3."""
    from eventgrad_b200.ops import ext
    C = ext()
    cfg = _cfg(topology, 3, 1 if base == "gossip" else 3, dataset="cifar10", model="resnet18")
    grid = min(C.gossip_max_grid(0), C.gossip_graph_max_grid(0)) // R
    _run(cfg, R, table_mode=(mode == "table"), steps=7, model_fn=lambda: build_model("resnet18"), grid_cap=grid)


@pytest.mark.parametrize("R,topology,tau,H", [(4, "ring", 3, 1), (8, "exp", 2, 1), (3, "ring", 2, 2),
                                              (4, "exp", 3, 3)])
def test_slowmo_captured_graph_equals_eager(R, topology, tau, H):
    """Each rank's step -- the gated sync kernel and the step kernel -- captured once in a CUDA graph and replayed over
    two cycles equals eager execution: whether a step syncs comes from the device step counter."""
    steps = 2 * tau
    res = []
    for captured in (False, True):
        cfg = _cfg(topology, tau, H)
        w = _world(cfg, R)
        table = lr_table(cfg, SPE)
        for be in w.backends:
            be.set_lr_table(table)
        graphs = []
        if captured:
            torch.cuda.synchronize()
            for r in range(R):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    w.backends[r].launch()
                graphs.append(g)
            torch.cuda.synchronize()
        cur = torch.cuda.current_stream()
        for s in range(1, steps + 1):
            gr = _grads(w, R, 20 + s)
            if not captured:
                w.step(gr)
                continue
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
        for be in w.backends:
            be.check_status()
            assert int(be.d_pass.item()) == steps and int(be.ar_ctr.item()) == 2
        res.append([(a.theta.cpu(), a.mom.cpu(), be.slowmo_x.cpu(), be.slowmo_u.cpu(),
                     [b.cpu() for _, b in _inboxes(be)], be.bytes_sent()) for a, be in zip(w.arenas, w.backends)])
        del graphs
        w.close()
    for r in range(R):
        (t0, m0, x0, u0, i0, b0), (t1, m1, x1, u1, i1, b1) = res[0][r], res[1][r]
        assert torch.equal(t0, t1) and torch.equal(m0, m1) and b0 == b1, f"rank {r}"
        assert torch.equal(x0, x1) and torch.equal(u0, u1), f"rank {r} x / u"
        assert all(torch.equal(x, y) for x, y in zip(i0, i1)), f"rank {r} inboxes"


@pytest.mark.parametrize("at", [2, 3])
@pytest.mark.parametrize("topology,H", [("ring", 1), ("exp", 1), ("ring", 3)])
def test_slowmo_checkpoint_round_trip(topology, H, at):
    """tau = 3: state_dict one step before a sync (step 2) and at a sync (step 3) carries the SlowMo settings, x and u;
    a fresh world loaded from it continues bit for bit over two more cycles, and worlds with another period or beta
    refuse it."""
    R, tau = 4, 3
    cfg = _cfg(topology, tau, H)
    a = _world(cfg, R)
    for s in range(at):
        a.step(_grads(a, R, 400 + s))
    torch.cuda.synchronize()
    sds = [be.state_dict() for be in a.backends]
    arenas = [ar.state_dict() for ar in a.arenas]
    assert all(sd["slowmo_period"] == tau and sd["pass_num"] == at and "slowmo_x" in sd and "slowmo_u" in sd
               for sd in sds)
    b = _world(cfg, R)
    for ar, be, asd, sd in zip(b.arenas, b.backends, arenas, sds):
        ar.load_state_dict(asd)
        be.load_state_dict(sd)
    for s in range(at, at + 2 * tau):
        g = _grads(a, R, 400 + s)
        a.step(g)
        b.step(g)
    torch.cuda.synchronize()
    for r in range(R):
        assert torch.equal(a.arenas[r].theta, b.arenas[r].theta) and torch.equal(a.arenas[r].mom, b.arenas[r].mom)
        assert torch.equal(a.backends[r].slowmo_x, b.backends[r].slowmo_x)
        assert torch.equal(a.backends[r].slowmo_u, b.backends[r].slowmo_u)
        for (_, x), (_, y) in zip(_inboxes(a.backends[r]), _inboxes(b.backends[r])):
            assert torch.equal(x, y), f"rank {r}"
        a.backends[r].check_status()
        b.backends[r].check_status()
        assert a.backends[r].bytes_sent() == b.backends[r].bytes_sent()
    b.close()
    for other in (_cfg(topology, 2, 1 if H == 1 else 2), _cfg(topology, tau, H, slowmo_beta=0.5)):
        n = _world(other, R)
        with pytest.raises(ValueError, match="slowmo|local-steps"):
            n.backends[0].load_state_dict(sds[0])
        n.close()
    a.close()


def test_slowmo_launcher_rejects_what_it_does_not_run():
    """The sync kernel's launcher refuses a gate below 2 or without its pass counter, one-shot mode, a mode other than
    0, a null x or u, beta outside [0, 1) and alpha <= 0, before anything is enqueued."""
    s = torch.cuda.current_stream().cuda_stream
    w = _world(_cfg("ring", 2), 3)
    be = w.backends[0]
    good = {"gate_period": 2, "gate_pass": be.d_pass.data_ptr(), "two_shot": 1, "mode": 0,
            "x": be.slowmo_x.data_ptr(), "u": be.slowmo_u.data_ptr(), "beta": 0.7, "alpha": 1.2}
    bads = [{"gate_period": 1}, {"gate_period": 0}, {"gate_period": -2}, {"gate_pass": 0}, {"two_shot": 0},
            {"mode": 1}, {"x": 0}, {"u": 0}, {"beta": 1.0}, {"beta": -0.1}, {"alpha": 0.0}, {"alpha": -1.0}]
    for bad in bads:
        be.sm.update(bad)
        with pytest.raises(RuntimeError, match="slowmo_sync"):
            be.C.slowmo_sync(be.sm, be.grid, s)
        be.sm.update(good)
    torch.cuda.synchronize()
    for b in w.backends:
        b.check_status()
        assert int(b.ar_ctr.item()) == 0
    w.close()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [30580]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "slowmo_worker.py"), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "WORKER_OK" in out, out[-3000:]


def _need(world):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < world:
        pytest.skip(f"needs {world} GPUs, found {n}")


@pytest.mark.multigpu
@pytest.mark.parametrize("world,topology,H", [(2, "ring", 1), (4, "ring", 3), (8, "exp", 1)])
@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_multigpu_slowmo_vs_simulator(world, topology, H, backend):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", backend, "--topology", topology, "--slowmo-period", "3",
              "--local-steps", str(H))
