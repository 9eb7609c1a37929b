"""GPU: Chebyshev-accelerated gossip rounds (--gossip-accel chebyshev, decent) -- Q launches of the Chebyshev round
kernel (csrc/gossip_rounds.cu) and then the serial step kernel, bit for bit against the simulator.  Multi-rank runs use
R virtual ranks on one GPU (ops.local_world.LocalWorld); the torchrun cases at the end need one GPU per rank and skip
otherwise."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import TrainConfig
from eventgrad_b200.engine.lr_schedule import lr_table
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.topology import chebyshev_coefficients
from eventgrad_b200.parallel.trigger import consensus_stats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SPE = 3          # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=12)


def _cfg(topology="ring", Q=2, accel="chebyshev", **kw):
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", topology=topology,
                gossip_rounds=Q, gossip_accel=accel, overlap_push=False, **OPT)
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, model_fn=None, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    w = LocalWorld(cfg, R, model_fn or (lambda: build_model("cnn2")), grid_cap=grid_cap, table_mode=table_mode,
                   timeout_ns=5_000_000_000)
    on = R > 1 and cfg.gossip_accel == "chebyshev"
    for be in w.backends:
        assert (be.cs is not None) == on and not be.overlap
        assert not (on and be.dbuf)                 # no double-buffered step after the rounds
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


def _sim(cfg, w, R, table, **kw):
    return RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, "decent", lr=cfg.lr, momentum=cfg.momentum,
                         serial_skip=False, weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table,
                         offsets=w.cfg.topology, gossip_rounds=cfg.gossip_rounds, gossip_accel=cfg.gossip_accel, **kw)


def _check(w, sim, s, m):
    for r, be in enumerate(w.backends):
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} rank {r} theta"
        assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s} rank {r} momentum"
        assert be.bytes_sent() == sim.bytes[r], f"step {s} rank {r} bytes"
        assert bool((w.arenas[r].theta[m == 0] == 0).all()), f"step {s} rank {r}: padding of theta is not zero"


def _run(cfg, R, table_mode=False, steps=9, model_fn=None, grid_cap=6, grad_seed=40):
    w = _world(cfg, R, model_fn, table_mode, grid_cap)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    m = _mask(w.arenas[0].table)
    for s in range(1, steps + 1):
        g = _grads(w, R, grad_seed + s)
        w.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        _check(w, sim, s, m)
    Q = cfg.gossip_rounds
    for be in w.backends:
        be.check_status()
        assert int(be.status.item()) == 0 and int(be.d_pass.item()) == steps
        # Q round launches per step: every round acked every slot with the last counter h = Q * steps
        for k in range(be.ring.n_slots):
            assert int(be.win.view(f"round_ack_{k}", torch.int32)[0].item()) == Q * steps
    assert all(b == steps * Q * sim.fanout * 4 * w.arenas[0].table.n_elems for b in sim.bytes)
    w.close()


_RING = [2, 3, 4, 5, 8]
_GRAPH = [(8, "exp"), (8, "1,3")]


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("Q", [1, 2, 3])
@pytest.mark.parametrize("R", _RING)
def test_cheb_ring_bitwise_vs_simulator(R, Q, mode):
    """theta, momentum and bytes at every step on the ring, R = 2 and 3 (one-point spectra) included."""
    _run(_cfg("ring", Q), R, table_mode=(mode == "table"))


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("Q", [1, 2, 3])
@pytest.mark.parametrize("R,topology", _GRAPH)
def test_cheb_graph_bitwise_vs_simulator(R, topology, Q, mode):
    _run(_cfg(topology, Q), R, table_mode=(mode == "table"))


@pytest.mark.parametrize("R,topology", [(2, "ring"), (4, "ring"), (8, "exp")])
def test_cheb_resnet18_at_the_full_persistent_grid(R, topology):
    """The ResNet-18 `ref` arena at the co-resident grid of the kernels in use, Q = 3."""
    from eventgrad_b200.ops import ext
    C = ext()
    cfg = _cfg(topology, 3, dataset="cifar10", model="resnet18")
    grid = min(C.gossip_max_grid(0), C.gossip_graph_max_grid(0), C.gossip_rounds_max_grid(0)) // R
    _run(cfg, R, steps=4, model_fn=lambda: build_model("resnet18"), grid_cap=grid)


@pytest.mark.parametrize("R,topology,Q", [(4, "ring", 3), (3, "ring", 2), (8, "exp", 2), (5, "ring", 1)])
def test_cheb_captured_graph_equals_eager(R, topology, Q):
    """Each rank's step -- the Q Chebyshev round launches and the serial step kernel -- captured once in a CUDA graph
    and replayed equals eager execution: the handshake counter comes from the device step counter."""
    steps, res = 5, []
    for captured in (False, True):
        cfg = _cfg(topology, Q)
        w = _world(cfg, R)
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
            assert int(be.d_pass.item()) == steps
        res.append([(a.theta.cpu(), a.mom.cpu(), be.bytes_sent()) for a, be in zip(w.arenas, w.backends)])
        del graphs
        w.close()
    for r in range(R):
        (t0, m0, b0), (t1, m1, b1) = res[0][r], res[1][r]
        assert torch.equal(t0, t1) and torch.equal(m0, m1) and b0 == b1, f"rank {r}"


@pytest.mark.parametrize("R,topology,Q", [(4, "ring", 2), (3, "ring", 1), (8, "exp", 2)])
def test_cheb_with_consensus_every_step(R, topology, Q):
    """--consensus-every 1 leaves training bit for bit unchanged, and every measurement is the simulator's within the
    consensus kernel's tolerance (the same bits on every rank), although the next step's first round overwrites theta
    with no step handshake in between."""
    out = []
    for N in (0, 1):
        cfg = _cfg(topology, Q, consensus_every=N)
        w = _world(cfg, R)
        table = lr_table(cfg, SPE)
        for be in w.backends:
            be.set_lr_table(table)
        sim = _sim(cfg, w, R, table, consensus_every=N)
        for s in range(1, 6):
            g = _grads(w, R, 60 + s)
            w.step(g)
            sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        rows = [be.drain_consensus() for be in w.backends]
        for be in w.backends:
            be.check_status()
        out.append([(a.theta.cpu(), a.mom.cpu(), be.bytes_sent()) for a, be in zip(w.arenas, w.backends)])
        for r in range(R):
            assert torch.equal(out[-1][r][0], sim.theta[r])
        if N:
            for r in range(R):
                assert [k for k, _, _ in rows[r]] == [k for k, _, _ in sim.consensus] == list(range(1, 6))
                for (k, D, A), (_, Ds, As) in zip(rows[r], sim.consensus):
                    assert torch.allclose(D, Ds, rtol=1e-5, atol=0) and torch.allclose(A, As, rtol=1e-5, atol=0), k
                    assert torch.equal(D, rows[0][k - 1][1]) and torch.equal(A, rows[0][k - 1][2])
            assert float(sim.consensus[-1][1].sum()) > 0
            Ds, As = consensus_stats(sim.theta, w.arenas[0].table)
            assert torch.allclose(rows[0][-1][1], Ds, rtol=1e-5, atol=0)
        w.close()
    for r in range(R):
        assert all(torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y for x, y in zip(out[0][r], out[1][r]))


@pytest.mark.parametrize("Q2,accel2", [(3, "chebyshev"), (2, "chebyshev"), (1, "chebyshev"), (3, "none"),
                                       (1, "none")])
@pytest.mark.parametrize("topology", ["ring", "exp"])
def test_cheb_checkpoint_round_trip(topology, Q2, accel2):
    """Chebyshev Q = 3, state_dict after step 3, loaded into a fresh world with Q2 rounds and accel2: it continues bit for
    bit what the simulator that switches at that step computes (the round flags and acks restart at the resuming run's
    rounds-per-step times 3; `prev` and the round inboxes are rewritten before they are read)."""
    R, at, steps = 4, 3, 7
    cfg = _cfg(topology, 3)
    a = _world(cfg, R)
    sim = _sim(cfg, a, R, None)
    for s in range(at):
        g = _grads(a, R, 400 + s)
        a.step(g)
        sim.step([x.cpu() for x in g])
    torch.cuda.synchronize()
    sds = [be.state_dict() for be in a.backends]
    arenas = [ar.state_dict() for ar in a.arenas]
    a.close()
    b = _world(_cfg(topology, Q2, accel2, double_buffer=False), R)
    for ar, be, asd, sd in zip(b.arenas, b.backends, arenas, sds):
        ar.load_state_dict(asd)
        be.load_state_dict(sd)
    sim.gossip_rounds = Q2
    sim.cheb_coef = chebyshev_coefficients(sim.offsets, R, Q2) if accel2 == "chebyshev" else None
    m = _mask(b.arenas[0].table)
    for s in range(at, steps):
        g = _grads(b, R, 400 + s)
        b.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        _check(b, sim, s + 1, m)
    for be in b.backends:
        be.check_status()
    b.close()


def test_cheb_launcher_and_backend_reject_what_they_do_not_run():
    """The Chebyshev launcher refuses a null prev or coef (and everything the power launcher refuses) before anything
    is enqueued; the p2p backend refuses the flag with anything but decent on the ring or a static graph."""
    from eventgrad_b200.ops.local_world import LocalWorld
    s = torch.cuda.current_stream().cuda_stream
    w = _world(_cfg("ring", 2), 4)
    be = w.backends[0]
    for bad in ({"prev": 0}, {"coef": 0}):
        keep = {"prev": be.cheb_prev.data_ptr(), "coef": be.d_cheb_coef.data_ptr()}
        be.cs.update(bad)
        with pytest.raises(RuntimeError, match="gossip_rounds_cheb"):
            be.C.gossip_rounds_cheb(be.rp, be.cs, be.grid, s)
        be.cs.update(keep)
    for bad in ({"rounds": 0}, {"n_slots": 3}, {"theta": 0}):
        be.rp.update(bad)
        with pytest.raises(RuntimeError, match="gossip_rounds_cheb"):
            be.C.gossip_rounds_cheb(be.rp, be.cs, be.grid, s)
    w.close()
    torch.cuda.synchronize()
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", gossip_rounds=2,
                gossip_accel="chebyshev", overlap_push=False)
    for kw in (dict(algo="event"), dict(overlap_push=True), dict(compress="int8"), dict(local_steps=2),
               dict(global_avg_period=2), dict(double_buffer=True), dict(topology="onepeer-exp")):
        cfg = TrainConfig(**{**base, **kw})                    # not validated: the backend's own check
        with pytest.raises(ValueError, match="gossip"):
            LocalWorld(cfg, 4, lambda: build_model("cnn2"), grid_cap=6, timeout_ns=5_000_000_000)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [30780]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "chebyshev_worker.py"), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "WORKER_OK" in out, out[-3000:]


def _need(world):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < world:
        pytest.skip(f"needs {world} GPUs, found {n}")


@pytest.mark.multigpu
@pytest.mark.parametrize("world,topology", [(2, "ring"), (4, "ring"), (4, "exp")])
@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_multigpu_cheb_vs_simulator(world, topology, backend):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", backend, "--topology", topology, "--gossip-rounds", "3")
