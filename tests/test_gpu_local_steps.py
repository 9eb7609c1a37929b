"""GPU: periodic gossip (--local-steps H, decent) in the fused ring step kernel (csrc/gossip.cu) and the graph step kernel
(csrc/gossip_graph.cu), bit for bit against the simulator.  Multi-rank runs use R virtual ranks on one GPU
(ops.local_world.LocalWorld); the torchrun cases at the end need one GPU per rank and skip otherwise."""
import math
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


def _cfg(topology="ring", H=2, **kw):
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", topology=topology,
                local_steps=H, double_buffer=False, **OPT)      # H = 1: the same single-slot kernel, not gossip_dbuf
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, model_fn=None, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    w = LocalWorld(cfg, R, model_fn or (lambda: build_model("cnn2")), grid_cap=grid_cap, table_mode=table_mode,
                   timeout_ns=5_000_000_000)
    assert all(be.local_steps == cfg.local_steps and not be.overlap and not be.dbuf for be in w.backends)
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
                         offsets=w.cfg.topology, local_steps=cfg.local_steps)


def _inboxes(be):
    """(simulator slot, device buffer) pairs: the graph's slots, or the ring's from-left / from-right inboxes (the
    2-rank ring keeps its single copy in inbox_r)."""
    if be.graph is not None:
        return [(s, be.win.view(f"inbox_{s}", torch.float32)) for s in range(be.graph.n_slots)]
    out = [(1, be.win.view("inbox_r", torch.float32))]
    if not be.wire_dedup:
        out.append((0, be.win.view("inbox_l", torch.float32)))
    return out


def _check(w, sim, R, s, m):
    for r, be in enumerate(w.backends):
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} rank {r} theta"
        assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s} rank {r} momentum"
        for slot, buf in _inboxes(be):
            assert torch.equal(buf[:sim.theta[r].numel()].cpu(), sim.inbox[r][slot]), f"step {s} rank {r} slot {slot}"
        assert be.bytes_sent() == sim.bytes[r], f"step {s} rank {r} bytes"
        assert bool((w.arenas[r].theta[m == 0] == 0).all()), f"step {s} rank {r}: padding of theta is not zero"


def _steps(R, H):
    tau = (R - 1).bit_length()
    return max(2 * tau * H + 1, 9)      # two one-peer cycles, and past the schedule's milestone at step 7


def _run(cfg, R, table_mode=False, steps=None, model_fn=None, grid_cap=6, grad_seed=40):
    w = _world(cfg, R, model_fn, table_mode, grid_cap)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    m = _mask(w.arenas[0].table)
    steps = steps or _steps(R, cfg.local_steps)
    for s in range(1, steps + 1):
        g = _grads(w, R, grad_seed + s)
        w.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        _check(w, sim, R, s, m)
    for be in w.backends:
        be.check_status()
        assert int(be.d_pass.item()) == steps
    assert all(b == (steps // cfg.local_steps) * sim.fanout * w.arenas[0].table.n_elems * 4 for b in sim.bytes)
    w.close()


_CASES = ([(R, topo) for R in (2, 3, 4, 8) for topo in ("ring", "exp", "onepeer-exp")] + [(8, "1,3")])


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("H", [1, 2, 3, 4])
@pytest.mark.parametrize("R,topology", _CASES)
def test_local_steps_bitwise_vs_simulator(R, topology, H, mode):
    """Every step: theta, momentum, every inbox and the byte counter equal the simulator's."""
    _run(_cfg(topology, H), R, table_mode=(mode == "table"))


@pytest.mark.parametrize("R,topology,mode", [(2, "ring", "flat"), (4, "ring", "table"), (4, "onepeer-exp", "flat"),
                                             (4, "exp", "flat")])
def test_local_steps_resnet18_at_the_full_persistent_grid(R, topology, mode):
    """The ResNet-18 `ref` arena (86 tensors, 8 569 tiles) at the co-resident grid of the kernel in use, H = 3."""
    from eventgrad_b200.ops import ext
    C = ext()
    cfg = _cfg(topology, 3, dataset="cifar10", model="resnet18")
    grid = min(C.gossip_max_grid(0), C.gossip_graph_max_grid(0)) // R
    _run(cfg, R, table_mode=(mode == "table"), steps=7, model_fn=lambda: build_model("resnet18"), grid_cap=grid)


@pytest.mark.parametrize("R,topology,H", [(4, "ring", 3), (4, "onepeer-exp", 3), (8, "onepeer-exp", 2),
                                          (4, "exp", 4)])
def test_local_steps_captured_graph_equals_eager(R, topology, H):
    """Each rank's step captured once in a CUDA graph and replayed over two full cycles (lcm(H, tau) * 2 steps) equals
    eager execution: which step gossips, and the one-peer slot of its round, come from the device step counter."""
    tau = (R - 1).bit_length() if topology == "onepeer-exp" else 1
    steps = 2 * (H * tau // math.gcd(H, tau))
    res = []
    for captured in (False, True):
        cfg = _cfg(topology, H)
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
            assert int(be.d_pass.item()) == steps
        res.append([(a.theta.cpu(), a.mom.cpu(), [b.cpu() for _, b in _inboxes(be)], be.bytes_sent())
                    for a, be in zip(w.arenas, w.backends)])
        del graphs
        w.close()
    for r in range(R):
        (t0, m0, i0, b0), (t1, m1, i1, b1) = res[0][r], res[1][r]
        assert torch.equal(t0, t1) and torch.equal(m0, m1) and b0 == b1, f"rank {r}"
        assert all(torch.equal(x, y) for x, y in zip(i0, i1)), f"rank {r} inboxes"


@pytest.mark.parametrize("topology", ["ring", "onepeer-exp"])
def test_local_steps_checkpoint_round_trip_mid_cycle(topology):
    """state_dict at step 4 of H = 3 carries `local_steps`; a fresh world loaded from it continues bit for bit (the
    handshake counters restart at the checkpoint's step, below the next round's WAR bound), and a world with another H
    refuses it."""
    R, H = 4, 3
    cfg = _cfg(topology, H)
    a = _world(cfg, R)
    for s in range(4):
        a.step(_grads(a, R, 400 + s))
    torch.cuda.synchronize()
    sds = [be.state_dict() for be in a.backends]
    arenas = [ar.state_dict() for ar in a.arenas]
    assert all(sd["local_steps"] == H and sd["pass_num"] == 4 for sd in sds)
    b = _world(cfg, R)
    for ar, be, asd, sd in zip(b.arenas, b.backends, arenas, sds):
        ar.load_state_dict(asd)
        be.load_state_dict(sd)
    for s in range(4, 4 + 3 * H):
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
    for other in (1, 2):
        n = _world(_cfg(topology, other), R)
        with pytest.raises(ValueError, match="local-steps"):
            n.backends[0].load_state_dict(sds[0])
        n.close()
    a.close()


def test_local_steps_launchers_reject_what_they_do_not_run():
    """The double-buffered, int8 and tracking launchers gossip at every step and refuse local_steps > 1; the ring and
    graph launchers refuse it with a split phase, a sparse block, the trigger or a drift copy.  Every case is refused
    before anything is enqueued."""
    s = torch.cuda.current_stream().cuda_stream
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter")
    from eventgrad_b200.ops.local_world import LocalWorld
    mk = lambda R=3, **kw: LocalWorld(TrainConfig(**{**base, **kw}).validate(), R, lambda: build_model("cnn2"),
                                      grid_cap=6, timeout_ns=5_000_000_000)
    w = mk(overlap_push=False)
    be = w.backends[0]
    assert be.dbuf
    be.gp.update({"local_steps": 2})
    with pytest.raises(RuntimeError, match="gossip_step_dbuf"):
        be.C.gossip_step_dbuf(be.gp, be.grid, s)
    w.close()
    w = mk(compress="int8")
    be = w.backends[0]
    be.gp.update({"local_steps": 2})
    with pytest.raises(RuntimeError, match="gossip_step_q8"):
        be.C.gossip_step_q8(be.gp, be.qs, be.grid, s)
    w.close()
    w = mk(gradient_tracking=True)
    be = w.backends[0]
    be.gp.update({"local_steps": 2})
    with pytest.raises(RuntimeError, match="gossip_step_gt"):
        be.C.gossip_step_gt(be.gp, be.ts, be.grid, s)
    w.close()
    for topology, fn in (("ring", "gossip_step"), ("exp", "gossip_step_graph")):
        w = mk(R=4, topology=topology, local_steps=2)          # exp at R = 4: offsets (1, 2), the graph kernel
        be = w.backends[0]
        assert (be.graph is None) == (topology == "ring")
        bads = [{"fsm.enabled": 1}, {"sent": 8}] + ([{"phase": 1}, {"sparse": 8}] if topology == "ring" else [])
        for bad in bads:
            keep = {k: 0 for k in bad}
            be.gp.update(bad)
            with pytest.raises(RuntimeError, match=fn):
                if topology == "ring":
                    be.C.gossip_step(be.gp, be.grid, s)
                else:
                    be.C.gossip_step_graph(be.gp, be.gs, be.grid, s)
            be.gp.update(keep)
        w.close()
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [29980]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "local_steps_worker.py"), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "WORKER_OK" in out, out[-3000:]


def _need(world):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < world:
        pytest.skip(f"needs {world} GPUs, found {n}")


@pytest.mark.multigpu
@pytest.mark.parametrize("world,topology", [(2, "ring"), (4, "ring"), (4, "onepeer-exp"), (8, "exp")])
@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_multigpu_local_steps_vs_simulator(world, topology, backend):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", backend, "--topology", topology, "--local-steps", "3")
