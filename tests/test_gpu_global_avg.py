"""GPU: periodic global averaging (--global-avg-period P, decent) -- the step-gated two-shot all-reduce of theta
(csrc/allreduce.cu) before the fused ring step kernel (csrc/gossip.cu) or the graph step kernel (csrc/gossip_graph.cu),
bit for bit against the simulator.  Multi-rank runs use R virtual ranks on one GPU (ops.local_world.LocalWorld); the
torchrun cases at the end need one GPU per rank and skip otherwise."""
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


def _cfg(topology="ring", P=2, **kw):
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", topology=topology,
                global_avg_period=P, double_buffer=False, **OPT)   # P = 0: the same single-slot kernel, not gossip_dbuf
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, model_fn=None, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    w = LocalWorld(cfg, R, model_fn or (lambda: build_model("cnn2")), grid_cap=grid_cap, table_mode=table_mode,
                   timeout_ns=5_000_000_000)
    assert all(be.global_avg_period == cfg.global_avg_period and not be.overlap and not be.dbuf for be in w.backends)
    assert all((be.ap_pga is not None) == (R > 1 and cfg.global_avg_period > 0) for be in w.backends)
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
                         offsets=w.cfg.topology, global_avg_period=cfg.global_avg_period)


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
        for slot, buf in _inboxes(be):
            assert torch.equal(buf[:sim.theta[r].numel()].cpu(), sim.inbox[r][slot]), f"step {s} rank {r} slot {slot}"
        assert be.bytes_sent() == sim.bytes[r], f"step {s} rank {r} bytes"
        assert bool((w.arenas[r].theta[m == 0] == 0).all()), f"step {s} rank {r}: padding of theta is not zero"


def _run(cfg, R, table_mode=False, steps=None, model_fn=None, grid_cap=6, grad_seed=40):
    P = cfg.global_avg_period
    w = _world(cfg, R, model_fn, table_mode, grid_cap)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    m = _mask(w.arenas[0].table)
    steps = steps or max(2 * P + 1, 9)      # two cycles, and past the schedule's milestone at step 7
    for s in range(1, steps + 1):
        g = _grads(w, R, grad_seed + s)
        w.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        _check(w, sim, s, m)
    for be in w.backends:
        be.check_status()
        assert int(be.d_pass.item()) == steps
        # the gate skipped every launch between averages without touching the all-reduce's launch counter
        assert int(be.ar_ctr.item()) == steps // P
    w.close()


_CASES = [(R, topo) for R in (2, 3, 4, 8) for topo in ("ring", "exp")] + [(8, "1,3")]


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("P", [2, 3, 5])
@pytest.mark.parametrize("R,topology", _CASES)
def test_global_avg_bitwise_vs_simulator(R, topology, P, mode):
    """Every step: theta, momentum, every inbox and the byte counter equal the simulator's."""
    _run(_cfg(topology, P), R, table_mode=(mode == "table"))


@pytest.mark.parametrize("R,topology,mode", [(2, "ring", "flat"), (4, "ring", "table"), (4, "exp", "flat"),
                                             (8, "ring", "flat")])
def test_global_avg_resnet18_at_the_full_persistent_grid(R, topology, mode):
    """The ResNet-18 `ref` arena (86 tensors, 8 569 tiles) at the co-resident grid of the kernels in use, P = 3."""
    from eventgrad_b200.ops import ext
    C = ext()
    cfg = _cfg(topology, 3, dataset="cifar10", model="resnet18")
    grid = min(C.gossip_max_grid(0), C.gossip_graph_max_grid(0)) // R
    _run(cfg, R, table_mode=(mode == "table"), steps=7, model_fn=lambda: build_model("resnet18"), grid_cap=grid)


@pytest.mark.parametrize("R,topology,P", [(4, "ring", 3), (8, "exp", 2), (3, "ring", 2), (2, "ring", 5)])
def test_global_avg_captured_graph_equals_eager(R, topology, P):
    """Each rank's step -- the gated all-reduce and the step kernel -- captured once in a CUDA graph and replayed over two
    cycles equals eager execution: whether a step averages comes from the device step counter."""
    steps = 2 * P
    res = []
    for captured in (False, True):
        cfg = _cfg(topology, P)
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
        res.append([(a.theta.cpu(), a.mom.cpu(), [b.cpu() for _, b in _inboxes(be)], be.bytes_sent())
                    for a, be in zip(w.arenas, w.backends)])
        del graphs
        w.close()
    for r in range(R):
        (t0, m0, i0, b0), (t1, m1, i1, b1) = res[0][r], res[1][r]
        assert torch.equal(t0, t1) and torch.equal(m0, m1) and b0 == b1, f"rank {r}"
        assert all(torch.equal(x, y) for x, y in zip(i0, i1)), f"rank {r} inboxes"


@pytest.mark.parametrize("at", [2, 3])
@pytest.mark.parametrize("topology", ["ring", "exp"])
def test_global_avg_checkpoint_round_trip(topology, at):
    """P = 3: state_dict one step before an average (step 2) and at an average (step 3) carries `global_avg_period`; a
    fresh world loaded from it continues bit for bit over two more cycles (the handshake counters restart at the
    checkpoint's step, at or above the next gossip step's WAR bound; the all-reduce counters restart at zero on every
    rank), and a world with another P refuses it."""
    R, P = 4, 3
    cfg = _cfg(topology, P)
    a = _world(cfg, R)
    for s in range(at):
        a.step(_grads(a, R, 400 + s))
    torch.cuda.synchronize()
    sds = [be.state_dict() for be in a.backends]
    arenas = [ar.state_dict() for ar in a.arenas]
    assert all(sd["global_avg_period"] == P and sd["pass_num"] == at for sd in sds)
    b = _world(cfg, R)
    for ar, be, asd, sd in zip(b.arenas, b.backends, arenas, sds):
        ar.load_state_dict(asd)
        be.load_state_dict(sd)
    for s in range(at, at + 2 * P):
        g = _grads(a, R, 400 + s)
        a.step(g)
        b.step(g)
    torch.cuda.synchronize()
    for r in range(R):
        assert torch.equal(a.arenas[r].theta, b.arenas[r].theta) and torch.equal(a.arenas[r].mom, b.arenas[r].mom)
        for (_, x), (_, y) in zip(_inboxes(a.backends[r]), _inboxes(b.backends[r])):
            assert torch.equal(x, y), f"rank {r}"
        a.backends[r].check_status()
        b.backends[r].check_status()
        assert a.backends[r].bytes_sent() == b.backends[r].bytes_sent()
    b.close()
    for other in (0, 2):
        n = _world(_cfg(topology, other), R)
        with pytest.raises(ValueError, match="global-avg-period"):
            n.backends[0].load_state_dict(sds[0])
        n.close()
    a.close()


def test_global_avg_launchers_reject_what_they_do_not_run():
    """The double-buffered, int8, tracking and exact-diffusion launchers refuse any period; the ring and graph launchers
    refuse P = 1, P < 0, and P >= 2 with a split phase, a sparse block, the trigger, a drift copy, local steps or the
    one-peer graph; the all-reduce refuses a negative gate or a gate without its pass counter.  Every case is refused
    before anything is enqueued."""
    s = torch.cuda.current_stream().cuda_stream
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter")
    from eventgrad_b200.ops.local_world import LocalWorld
    mk = lambda R=3, **kw: LocalWorld(TrainConfig(**{**base, **kw}).validate(), R, lambda: build_model("cnn2"),
                                      grid_cap=6, timeout_ns=5_000_000_000)
    w = mk(overlap_push=False)
    be = w.backends[0]
    assert be.dbuf
    for P in (1, 2):
        be.gp.update({"global_avg_period": P})
        with pytest.raises(RuntimeError, match="gossip_step_dbuf"):
            be.C.gossip_step_dbuf(be.gp, be.grid, s)
    w.close()
    for kw, fn, blk in ((dict(compress="int8"), "gossip_step_q8", "qs"), (dict(gradient_tracking=True),
                        "gossip_step_gt", "ts"), (dict(exact_diffusion=True), "gossip_step_ed", "es")):
        w = mk(**kw)
        be = w.backends[0]
        be.gp.update({"global_avg_period": 2})
        with pytest.raises(RuntimeError, match=fn):
            getattr(be.C, fn)(be.gp, getattr(be, blk), be.grid, s)
        w.close()
    for topology, fn in (("ring", "gossip_step"), ("exp", "gossip_step_graph")):
        w = mk(R=4, topology=topology, global_avg_period=2)     # exp at R = 4: offsets (1, 2), the graph kernel
        be = w.backends[0]
        assert (be.graph is None) == (topology == "ring")
        launch = ((lambda: be.C.gossip_step(be.gp, be.grid, s)) if topology == "ring"
                  else (lambda: be.C.gossip_step_graph(be.gp, be.gs, be.grid, s)))
        bads = ([{"global_avg_period": 1}, {"global_avg_period": -2}, {"fsm.enabled": 1}, {"sent": 8},
                 {"local_steps": 2}] + ([{"phase": 1}, {"sparse": 8}] if topology == "ring" else []))
        for bad in bads:
            keep = {k: (2 if k == "global_avg_period" else 1 if k == "local_steps" else 0) for k in bad}
            be.gp.update(bad)
            with pytest.raises(RuntimeError, match=fn):
                launch()
            be.gp.update(keep)
        for bad in ({"gate_period": -1}, {"gate_pass": 0}):
            keep = {"gate_period": 2, "gate_pass": be.d_pass.data_ptr()}
            be.ap_pga.update(bad)
            with pytest.raises(RuntimeError, match="allreduce"):
                be.C.allreduce(be.ap_pga, be.grid, s)
            be.ap_pga.update(keep)
        w.close()
    w = mk(R=4, topology="onepeer-exp")                        # the one-peer graph: a period in GraphSlots
    be = w.backends[0]
    assert be.graph is not None and be.graph.period > 0
    be.gp.update({"global_avg_period": 2})
    with pytest.raises(RuntimeError, match="gossip_step_graph"):
        be.C.gossip_step_graph(be.gp, be.gs, be.grid, s)
    w.close()
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [30480]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "global_avg_worker.py"), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "WORKER_OK" in out, out[-3000:]


def _need(world):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < world:
        pytest.skip(f"needs {world} GPUs, found {n}")


@pytest.mark.multigpu
@pytest.mark.parametrize("world,topology", [(2, "ring"), (4, "ring"), (8, "exp")])
@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_multigpu_global_avg_vs_simulator(world, topology, backend):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", backend, "--topology", topology, "--global-avg-period", "3")
