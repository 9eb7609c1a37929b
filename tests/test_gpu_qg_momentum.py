"""GPU: quasi-global momentum (--quasi-global-momentum) in the ring, double-buffered and graph step kernels
(csrc/gossip.cu, the kQG instance), bit for bit against the simulator: theta and m_hat at every step.  Multi-rank runs use
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
from eventgrad_b200.parallel.trigger import TriggerConfig

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SPE = 3          # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=12)


def _cfg(algo="decent", topology="ring", **kw):
    base = dict(algo=algo, dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", topology=topology,
                horizon=1.0, thres_type=1, initial_comm_passes=3, topk_percent=10.0, quasi_global_momentum=True,
                **OPT)
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, model_fn=None, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    w = LocalWorld(cfg, R, model_fn or (lambda: build_model("cnn2")), grid_cap=grid_cap, table_mode=table_mode,
                   timeout_ns=5_000_000_000)
    assert all(be.qg == cfg.quasi_global_momentum for be in w.backends)
    return w


def _grads(w, R, seed):
    t = w.arenas[0].table
    m = torch.zeros(t.n_padded, device="cuda")
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(t.n_padded, generator=g, device="cuda") * 0.05 * m for _ in range(R)]


def _run(cfg, R, table_mode=False, steps=9, model_fn=None, grid_cap=6):
    w = _world(cfg, R, model_fn, table_mode, grid_cap)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, cfg.algo, TriggerConfig.from_train(cfg),
                        lr=cfg.lr, momentum=cfg.momentum, topk_percent=cfg.topk_percent, serial_skip=False,
                        weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table,
                        offsets=w.cfg.topology, local_steps=cfg.local_steps, quasi_global=True)
    for s in range(1, steps + 1):
        fires = [be.fire.clone().bool().cpu() for be in w.backends] if cfg.algo != "decent" else None
        norms = [be.cur_norm.clone().cpu() for be in w.backends] if cfg.algo != "decent" else None
        g = _grads(w, R, 40 + s)
        w.step(g)
        if cfg.algo == "decent":
            sim.step([x.cpu() for x in g])
        elif cfg.trigger == "drift":
            sim.step([x.cpu() for x in g], norms=norms)
        else:
            sim.step([x.cpu() for x in g], fires=fires)
        torch.cuda.synchronize()
        for r, be in enumerate(w.backends):
            assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} rank {r} theta"
            assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s} rank {r} m_hat"
    for be in w.backends:
        be.check_status()
        assert int(be.d_pass.item()) == steps
    w.close()


_CASES = ([(R, "decent", "ring", dict(double_buffer=False)) for R in (2, 3, 4, 8)]
          + [(R, "decent", "ring", dict(overlap_push=False)) for R in (2, 4)]             # double-buffered inbox
          + [(R, "decent", "ring", dict(overlap_push=True)) for R in (2, 3)]              # split step
          + [(4, "decent", "exp", {}), (8, "decent", "exp", {}), (8, "decent", "1,3", {}),
             (4, "decent", "onepeer-exp", {}), (8, "decent", "onepeer-exp", {})]
          + [(3, "decent", "ring", dict(local_steps=2)), (4, "decent", "exp", dict(local_steps=2)),
             (4, "decent", "onepeer-exp", dict(local_steps=2))]
          + [(R, "event", "ring", dict(overlap_push=False)) for R in (2, 3)]
          + [(3, "event", "ring", dict(overlap_push=True)), (4, "event", "exp", {}), (8, "event", "1,3", {}),
             (4, "event", "onepeer-exp", {}), (3, "event", "ring", dict(trigger="drift", overlap_push=False)),
             (4, "event", "exp", dict(trigger="drift"))]
          + [(2, "spevent", "ring", {}), (3, "spevent", "ring", {}), (4, "spevent", "ring", dict(trigger="drift"))])


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("R,algo,topology,kw", _CASES)
def test_qg_bitwise_vs_simulator(R, algo, topology, kw, mode):
    _run(_cfg(algo, topology, **kw), R, table_mode=(mode == "table"))


@pytest.mark.parametrize("R,topology,algo", [(2, "ring", "decent"), (4, "ring", "event"), (4, "exp", "decent"),
                                             (8, "ring", "decent")])
def test_qg_resnet18_at_the_full_persistent_grid(R, topology, algo):
    from eventgrad_b200.ops import ext
    C = ext()
    cfg = _cfg(algo, topology, dataset="cifar10", model="resnet18", overlap_push=False)
    grid = min(C.gossip_max_grid(0), C.gossip_graph_max_grid(0), C.gossip_dbuf_max_grid(0)) // R
    _run(cfg, R, steps=5, model_fn=lambda: build_model("resnet18"), grid_cap=grid)


@pytest.mark.parametrize("R,topology", [(3, "ring"), (4, "exp")])
def test_qg_captured_graph_equals_eager_over_a_local_steps_cycle(R, topology):
    steps, res = 6, []
    for captured in (False, True):
        cfg = _cfg("decent", topology, local_steps=3)
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
        res.append([(a.theta.cpu(), a.mom.cpu(), be.bytes_sent()) for a, be in zip(w.arenas, w.backends)])
        del graphs
        w.close()
    for (t0, m0, b0), (t1, m1, b1) in zip(res[0], res[1]):
        assert torch.equal(t0, t1) and torch.equal(m0, m1) and b0 == b1


@pytest.mark.parametrize("nesterov", [False, True])
def test_qg_quadratic_through_the_kernel_equals_the_fp32_simulator(nesterov):
    """Heterogeneous least squares (5 dims, R = 4 ring, full gradients) in fp32: the kernel's theta and m_hat equal the
    fp32 simulator's bit for bit at every step."""
    from eventgrad_b200.ops.local_world import LocalWorld
    R, dim, steps = 4, 5, 40
    gen = torch.Generator().manual_seed(0)
    A = [torch.eye(dim) + 0.3 * torch.randn(dim, dim, generator=gen) for _ in range(R)]
    b = [torch.randn(dim, generator=gen) * 2 + 3 * r for r in range(R)]
    model_fn = lambda: torch.nn.Linear(dim, 1, bias=False)
    cfg = _cfg("decent", "ring", lr=0.02, momentum=0.9, nesterov=nesterov, weight_decay=0.0, lr_schedule="constant",
               lr_warmup_epochs=0.0, double_buffer=False)
    w = LocalWorld(cfg, R, model_fn, grid_cap=2, timeout_ns=5_000_000_000)
    for a in w.arenas:
        a.theta.zero_()
    t = w.arenas[0].table
    sim = RingSimulator(R, torch.zeros(t.n_padded), t, "decent", lr=0.02, momentum=0.9, nesterov=nesterov,
                        serial_skip=False, quasi_global=True)
    for s in range(steps):
        grads = []
        for r in range(R):
            gr = torch.zeros(t.n_padded)
            x = sim.theta[r][:dim]
            gr[:dim] = A[r].T @ (A[r] @ x - b[r])
            grads.append(gr)
        w.step([x.cuda() for x in grads])
        sim.step(grads)
        torch.cuda.synchronize()
        for r in range(R):
            assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s + 1} rank {r}"
            assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s + 1} rank {r} m_hat"
    w.close()


def test_qg_launchers_reject_what_they_do_not_run():
    """The ring, double-buffered and graph launchers refuse quasi_global with mu = 0, without a momentum buffer, in async
    mode and with a global-averaging period; the int8, tracking and exact-diffusion launchers refuse it outright.  Every
    case is refused before anything is enqueued."""
    s = torch.cuda.current_stream().cuda_stream
    from eventgrad_b200.ops.local_world import LocalWorld
    mk = lambda R=3, **kw: LocalWorld(_cfg(**kw), R, lambda: build_model("cnn2"), grid_cap=6,
                                      timeout_ns=5_000_000_000)
    bads = [{"mu": 0.0}, {"mom": 0}, {"sync": 0}, {"global_avg_period": 2}]
    for kw, fn, blk in ((dict(double_buffer=False), "gossip_step", None), (dict(overlap_push=False), "gossip_step_dbuf",
                                                                           None),
                        (dict(R=4, topology="exp"), "gossip_step_graph", "gs")):
        w = mk(**kw)
        be = w.backends[0]
        keep = {"mu": 0.9, "mom": w.arenas[0].mom.data_ptr(), "sync": 1, "global_avg_period": 0}
        for bad in bads:
            be.gp.update(bad)
            args = (be.gp, getattr(be, blk), be.grid, s) if blk else (be.gp, be.grid, s)
            with pytest.raises(RuntimeError, match=fn):
                getattr(be.C, fn)(*args)
            be.gp.update({k: keep[k] for k in bad})
        w.close()
    for kw, fn, blk in ((dict(compress="int8", quasi_global_momentum=False), "gossip_step_q8", "qs"),
                        (dict(gradient_tracking=True, quasi_global_momentum=False), "gossip_step_gt", "ts"),
                        (dict(exact_diffusion=True, quasi_global_momentum=False), "gossip_step_ed", "es")):
        w = mk(**kw)
        be = w.backends[0]
        be.gp.update({"quasi_global": 1})
        with pytest.raises(RuntimeError, match=fn):
            getattr(be.C, fn)(be.gp, getattr(be, blk), be.grid, s)
        w.close()
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [30780]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "qg_momentum_worker.py"), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "WORKER_OK" in out, out[-3000:]


def _need(world):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < world:
        pytest.skip(f"needs {world} GPUs, found {n}")


@pytest.mark.multigpu
@pytest.mark.parametrize("world,algo,topology", [(2, "decent", "ring"), (4, "event", "ring"), (8, "decent", "exp")])
@pytest.mark.parametrize("backend", ["p2p", "nccl"])
def test_multigpu_qg_vs_simulator(world, algo, topology, backend):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", backend, "--algo", algo, "--topology", topology)
