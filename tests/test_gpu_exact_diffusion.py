"""GPU: exact diffusion (--exact-diffusion, decent on the ring) in the fused step kernel (csrc/gossip_ed.cu).  Multi-rank
runs use R virtual ranks on one GPU (ops.local_world.LocalWorld) and compare with the simulator bit for bit at every
step (theta, momentum, psi, bytes); the quadratic case checks what exact diffusion is for, in fp32 through the kernel;
the torchrun cases at the end need one GPU per rank and skip otherwise."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

from eventgrad_b200.config import TrainConfig
from eventgrad_b200.engine.lr_schedule import lr_table
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPE = 3          # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=4)
PLAIN = dict(momentum=0.9)
NOMOM = dict(momentum=0.0)


def _cfg(opt=OPT, **kw):
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", exact_diffusion=True,
                **opt)
    base.update(kw)
    return TrainConfig(**base).validate()


def _cap(R):
    from eventgrad_b200.ops import ext
    return ext().gossip_ed_max_grid(0) // R


def _world(cfg, R, model_fn=None, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    w = LocalWorld(cfg, R, model_fn or (lambda: build_model("cnn2")), grid_cap=grid_cap, table_mode=table_mode,
                   timeout_ns=5_000_000_000)
    if cfg.exact_diffusion:
        assert all(be.ed and be.es is not None and not be.gt and not be.overlap and not be.dbuf for be in w.backends)
        assert all(be.wire_dedup == (R == 2) for be in w.backends)
    return w


def _mask(t):
    m = torch.zeros(t.n_padded, device="cuda")
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


def _grads(w, R, seed):
    """Per-rank gradients with a rank-dependent mean, as on label-sorted shards."""
    t = w.arenas[0].table
    m = _mask(t)
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [(torch.randn(t.n_padded, generator=g, device="cuda") * 0.05 + 0.01 * (r - 1)) * m for r in range(R)]


def _sim(cfg, w, R, table):
    return RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, "decent", lr=cfg.lr, momentum=cfg.momentum,
                         serial_skip=False, weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table,
                         exact_diffusion=True)


def _check(w, sim, R, s, m):
    for r, be in enumerate(w.backends):
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} rank {r} theta"
        if sim.mu != 0.0:
            assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s} rank {r} momentum"
        assert torch.equal(be.psi.cpu(), sim.psi[r]), f"step {s} rank {r} psi"
        assert be.bytes_sent() == sim.bytes[r], f"step {s} rank {r} bytes"
        for name, buf in (("theta", w.arenas[r].theta), ("psi", be.psi)):
            assert bool((buf[m == 0] == 0).all()), f"step {s} rank {r}: padding of {name} is not zero"


def _run(cfg, R, table_mode=False, steps=10, model_fn=None, grid_cap=6, grad_seed=40):
    w = _world(cfg, R, model_fn, table_mode, grid_cap)
    table = lr_table(cfg, SPE) if cfg.lr_schedule != "constant" else None
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    m = _mask(w.arenas[0].table)
    for s in range(1, steps + 1):
        g = _grads(w, R, grad_seed + s)
        w.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        _check(w, sim, R, s, m)
    for be in w.backends:
        be.check_status()
        assert int(be.d_pass.item()) == steps
    w.close()


@pytest.mark.parametrize("opt", ["opt", "plain", "nomom"])
@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("R", [2, 3, 4, 8])
def test_exact_diffusion_bitwise_vs_simulator(R, mode, opt):
    _run(_cfg({"opt": OPT, "plain": PLAIN, "nomom": NOMOM}[opt]), R, table_mode=(mode == "table"))


@pytest.mark.parametrize("R,mode", [(2, "flat"), (4, "flat"), (3, "table")])
def test_exact_diffusion_resnet18_at_the_full_persistent_grid(R, mode):
    """The ResNet-18 `ref` arena (86 tensors, 8 569 tiles) at the co-resident grid of the exact-diffusion kernel."""
    cfg = _cfg(dataset="cifar10", model="resnet18")
    _run(cfg, R, table_mode=(mode == "table"), steps=4, model_fn=lambda: build_model("resnet18"), grid_cap=_cap(R))


def test_exact_diffusion_captured_graph_equals_eager():
    """Each rank's step captured once in a CUDA graph and replayed 10 times equals eager execution."""
    R, steps = 4, 10
    res = []
    for captured in (False, True):
        cfg = _cfg()
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
        res.append([(a.theta.cpu(), a.mom.cpu(), be.psi.cpu(), be.bytes_sent())
                    for a, be in zip(w.arenas, w.backends)])
        del graphs
        w.close()
    for r in range(R):
        for x, y in zip(res[0][r], res[1][r]):
            assert (torch.equal(x, y) if torch.is_tensor(x) else x == y), f"rank {r}"


# ---------------------------------------------------------------------------------------- what exact diffusion is for
class _Quad(nn.Module):
    SIZES = (37, 300)

    def __init__(self):
        super().__init__()
        self.p = nn.ParameterList(nn.Parameter(torch.zeros(n)) for n in self.SIZES)


def _quadratics(t, R, seed=4, device="cpu", dtype=torch.float64):
    """f_r = 1/2 (theta - c_r)^T A_r (theta - c_r), diagonal A_r > 0 on the real lanes; returns A, c, theta*."""
    m = torch.zeros(t.n_padded, dtype=dtype)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    g = torch.Generator().manual_seed(seed)
    A = [(0.5 + 1.5 * torch.rand(t.n_padded, generator=g, dtype=dtype)) * m for _ in range(R)]
    c = [(torch.randn(t.n_padded, generator=g, dtype=dtype) * 2.0 + r) * m for r in range(R)]
    sa = torch.stack(A).sum(0)
    opt = torch.stack([a * x for a, x in zip(A, c)]).sum(0) / torch.where(m > 0, sa, torch.ones_like(sa))
    cast = lambda xs: [x.to(device=device, dtype=torch.float32) for x in xs]
    return A, c, opt, cast(A), cast(c)


def test_exact_diffusion_reaches_the_minimiser_through_the_kernel():
    """Heterogeneous quadratics at a constant lr, fp32 through the kernel.  The kernel computes the fp32 simulator's bits,
    exact diffusion ends within 1e-3 of the global minimiser (the float64 simulator reaches it to 1e-10), and plain decent
    stays where the float64 simulator's decent stays, about 0.9 away.  The fp32 error is not a few ulps: at the fixed
    point every step rounds the same values the same way, so sum(theta) - sum(psi) drifts by the same amount each step
    and the error grows linearly with the steps (about 5e-4 after 600 here; DESIGN.md section 6)."""
    R, steps, lr = 4, 600, 0.1
    from eventgrad_b200.parallel.arena import TILE, TensorTable
    t = TensorTable.from_named(list(_Quad().named_parameters()), TILE)
    A, c, opt, Ag, cg = _quadratics(t, R, device="cuda")
    err = {}
    for ed in (True, False):
        sim = RingSimulator(R, torch.zeros(t.n_padded, dtype=torch.float64), t, "decent", lr=lr, serial_skip=False,
                            exact_diffusion=ed)
        s32 = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", lr=lr, serial_skip=False, exact_diffusion=ed)
        A32, c32 = [x.cpu() for x in Ag], [x.cpu() for x in cg]
        for _ in range(steps):
            sim.step([a * (th - x) for a, x, th in zip(A, c, sim.theta)])
            s32.step([a * (th - x) for a, x, th in zip(A32, c32, s32.theta)])
        e64 = max(float((th - opt).abs().max()) for th in sim.theta)
        cfg = _cfg(NOMOM, lr=lr, exact_diffusion=ed)
        w = _world(cfg, R, _Quad)
        for _ in range(steps):
            w.step([a * (ar.theta - x) for a, x, ar in zip(Ag, cg, w.arenas)])
        torch.cuda.synchronize()
        for be in w.backends:
            be.check_status()
        for r, ar in enumerate(w.arenas):
            assert torch.equal(ar.theta.cpu(), s32.theta[r]), f"exact_diffusion={ed} rank {r}: kernel != fp32 simulator"
        e32 = max(float((ar.theta.double().cpu() - opt).abs().max()) for ar in w.arenas)
        err[ed] = (e64, e32)
        w.close()
    (ed64, ed32), (dp64, dp32) = err[True], err[False]
    assert ed64 < 1e-10 and dp64 > 1e-2, err
    assert ed32 < 1e-3 and ed32 < 1e-3 * dp32, err
    assert abs(dp32 - dp64) < 0.05 * dp64, err


# ---------------------------------------------------------------------------------------- state and launcher
def test_exact_diffusion_checkpoint_round_trip_and_plain_guard():
    """state_dict carries psi, the inboxes and `exact_diffusion`; loading it into a fresh world continues bit for bit,
    and a plain decent backend refuses it."""
    R = 3
    cfg = _cfg()
    a = _world(cfg, R)
    for s in range(5):
        a.step(_grads(a, R, 400 + s))
    torch.cuda.synchronize()
    sds = [be.state_dict() for be in a.backends]
    arenas = [ar.state_dict() for ar in a.arenas]
    assert all(sd["exact_diffusion"] is True and all(k in sd for k in ("psi", "inbox_l", "inbox_r")) for sd in sds)
    b = _world(cfg, R)
    for ar, be, asd, sd in zip(b.arenas, b.backends, arenas, sds):
        ar.load_state_dict(asd)
        be.load_state_dict(sd)
    for s in range(5, 9):
        g = _grads(a, R, 400 + s)
        a.step(g)
        b.step(g)
    torch.cuda.synchronize()
    for r in range(R):
        for x, y in ((a.arenas[r].theta, b.arenas[r].theta), (a.arenas[r].mom, b.arenas[r].mom),
                     (a.backends[r].psi, b.backends[r].psi)):
            assert torch.equal(x, y), f"rank {r}"
        a.backends[r].check_status()
        b.backends[r].check_status()
    assert a.backends[0].bytes_sent() == b.backends[0].bytes_sent()
    b.close()
    n = _world(_cfg(exact_diffusion=False), R)
    with pytest.raises(ValueError, match="exact-diffusion"):
        n.backends[0].load_state_dict(sds[0])
    n.close()
    a.close()


def test_exact_diffusion_launcher_rejects_what_it_does_not_run():
    R = 3
    cfg = _cfg(PLAIN)
    w = _world(cfg, R)
    be = w.backends[0]
    s = torch.cuda.current_stream().cuda_stream
    win, L, Rn = be.win, be.ring.left, be.ring.right
    good = {"sync": 1, "phase": 0, "do_push": 1, "do_mix": 1, "send_ack": 1, "sparse": 0, "sent": 0, "fsm.enabled": 0,
            "local_steps": 1, "ack_from_l": win.addr("ack_from_l"), "ack_to_r": win.addr("ack_from_l", Rn),
            "push_l": win.addr("inbox_r", L)}
    # every case is refused before anything is enqueued
    for bad in ({"sync": 0}, {"phase": 1}, {"phase": 2}, {"do_push": 0}, {"do_mix": 0}, {"send_ack": 0}, {"sparse": 8},
                {"sent": 8}, {"fsm.enabled": 1}, {"local_steps": 2}, {"ack_from_l": 0}, {"ack_to_r": 0}, {"push_l": 0}):
        be.gp.update(bad)
        with pytest.raises(RuntimeError, match="gossip_step_ed"):
            be.C.gossip_step_ed(be.gp, be.es, be.grid, s)
        be.gp.update({k: good[k] for k in bad})
    with pytest.raises(RuntimeError, match="gossip_step_ed"):
        be.C.gossip_step_ed(be.gp, be.C.EdSlots(), be.grid, s)       # psi null
    torch.cuda.synchronize()
    # nothing ran and the parameters are restored: the next steps equal the simulator's first steps
    sim = _sim(cfg, w, R, None)
    m = _mask(w.arenas[0].table)
    for k in range(1, 3):
        g = _grads(w, R, 70 + k)
        w.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        _check(w, sim, R, k, m)
    for b in w.backends:
        b.check_status()
    w.close()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [30050]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "exact_diffusion_worker.py"), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "WORKER_OK" in out, out[-3000:]


def _need(world):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < world:
        pytest.skip(f"needs {world} GPUs, found {n}")


@pytest.mark.multigpu
@pytest.mark.parametrize("backend", ["p2p", "nccl"])
@pytest.mark.parametrize("world", [2, 4])
def test_multigpu_exact_diffusion_vs_simulator(world, backend):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", backend, "--steps", "8")
