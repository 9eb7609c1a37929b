"""GPU: random pairwise matchings (--topology random-match) in the fused single-inbox step kernel (csrc/gossip_match.cu),
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
from eventgrad_b200.parallel.topology import match_pairs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "random-match"
SEED = 5

SPE = 3          # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=4)
PLAIN = dict(momentum=0.0, weight_decay=0.0, nesterov=False, lr_schedule="constant")


def _cfg(opt=True, **kw):
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", topology=NAME,
                topology_seed=SEED, **(OPT if opt else PLAIN))
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, table_mode=False, grid_cap=6, model_fn=None):
    from eventgrad_b200.ops.local_world import LocalWorld
    return LocalWorld(cfg, R, model_fn or (lambda: build_model("cnn2")), grid_cap=grid_cap, table_mode=table_mode,
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


def _sim(cfg, w, R, table, **kw):
    return RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, "decent", lr=cfg.lr, momentum=cfg.momentum,
                         serial_skip=False, weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table,
                         offsets=NAME, topology_seed=cfg.topology_seed, **kw)


def _check(w, sim, s):
    for r, be in enumerate(w.backends):
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} rank {r} theta differs"
        assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s} rank {r} momentum differs"
        assert be.num_events() == 0 and be.bytes_sent() == sim.bytes[r], f"step {s} rank {r} counters"


def _run(cfg, R, steps=9, table_mode=False, grid_cap=6, model_fn=None):
    w = _world(cfg, R, table_mode=table_mode, grid_cap=grid_cap, model_fn=model_fn)
    assert all(be.match is not None and be.ms is not None for be in w.backends)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    for s in range(1, steps + 1):
        g = _grads(w, R, 40 + s)
        w.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        _check(w, sim, s)
    for be in w.backends:
        be.check_status()
        assert int(be.d_pass.item()) == steps
    w.close()
    return sim


@pytest.mark.parametrize("opt", [True, False])
@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("R", [2, 3, 4, 5, 8])
def test_match_step_bitwise_vs_simulator(R, mode, opt):
    """theta, momentum and bytes at every step, with and without momentum / Nesterov / weight decay / an lr schedule;
    odd R has an idle rank at every step."""
    sim = _run(_cfg(opt), R, table_mode=(mode == "table"))
    if R % 2:                                     # some rank is idle at every step, and sends nothing then
        assert min(sim.bytes) < 9 * sim.table.n_elems * 4


def test_partners_hold_bitwise_equal_theta_after_the_mix():
    """lr = 0 and no momentum: after step k both ranks of every pair of match_pairs(seed, R, k) hold the same bits."""
    R = 6
    cfg = _cfg(False, lr=0.0)
    w = _world(cfg, R)
    t = w.arenas[0].table
    m = _mask(t)
    g = torch.Generator(device="cuda").manual_seed(1)
    for r in range(R):
        w.arenas[r].theta.copy_(torch.randn(t.n_padded, generator=g, device="cuda") * m)
    torch.cuda.synchronize()
    zeros = [torch.zeros(t.n_padded, device="cuda") for _ in range(R)]
    for k in range(1, 6):
        w.step(zeros)
        torch.cuda.synchronize()
        for a, b in match_pairs(SEED, R, k):
            assert torch.equal(w.arenas[a].theta, w.arenas[b].theta), (k, a, b)
    for be in w.backends:
        be.check_status()
    w.close()


@pytest.mark.parametrize("R", [4, 5])
def test_match_resnet18_at_the_full_persistent_grid(R):
    """The ResNet-18 `ref` arena at the co-resident grid of the match kernel, shared by R virtual ranks."""
    from eventgrad_b200.ops import ext
    C = ext()
    cfg = _cfg(dataset="cifar10", model="resnet18")
    grid = min(C.gossip_max_grid(0), C.gossip_match_max_grid(0)) // R
    _run(cfg, R, steps=4, model_fn=lambda: build_model("resnet18"), grid_cap=grid)


@pytest.mark.parametrize("R", [3, 4])
def test_match_captured_graph_equals_eager(R):
    """Each rank's step captured once in a CUDA graph and replayed equals eager execution and the simulator: the
    partner comes from the device step counter, so one graph walks through every matching."""
    cfg = _cfg()
    steps, res = 6, []
    for captured in (False, True):
        w = _world(cfg, R)
        table = lr_table(cfg, SPE)
        for be in w.backends:
            be.set_lr_table(table)
        sim = _sim(cfg, w, R, table)
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
            if captured:
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
            else:
                w.step(gr)
            torch.cuda.synchronize()
            sim.step([x.cpu() for x in gr])
            _check(w, sim, s)
        for be in w.backends:
            be.check_status()
        res.append([(a.theta.cpu(), a.mom.cpu(), be.bytes_sent()) for a, be in zip(w.arenas, w.backends)])
        del graphs
        w.close()
    for r in range(R):
        assert torch.equal(res[0][r][0], res[1][r][0]) and torch.equal(res[0][r][1], res[1][r][1])
        assert res[0][r][2] == res[1][r][2]


@pytest.mark.parametrize("R", [4, 5])
def test_match_with_consensus_every_step(R):
    """--consensus-every 1 leaves training bit for bit unchanged, and every measurement is the simulator's within the
    consensus kernel's tolerance (the same bits on every rank)."""
    out = []
    for N in (0, 1):
        cfg = _cfg(consensus_every=N)
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
        out.append([a.theta.cpu() for a in w.arenas])
        for r in range(R):
            assert torch.equal(out[-1][r], sim.theta[r])
        if N:
            for r in range(R):
                assert [k for k, _, _ in rows[r]] == [k for k, _, _ in sim.consensus] == list(range(1, 6))
                for (k, D, A), (_, Ds, As) in zip(rows[r], sim.consensus):
                    assert torch.allclose(D, Ds, rtol=1e-5, atol=0) and torch.allclose(A, As, rtol=1e-5, atol=0), k
                    assert torch.equal(D, rows[0][k - 1][1]) and torch.equal(A, rows[0][k - 1][2])
        w.close()
    for r in range(R):
        assert torch.equal(out[0][r], out[1][r])


@pytest.mark.parametrize("R", [4, 5])
def test_match_checkpoint_round_trip(R):
    """state_dict after step 3 loaded into a fresh world continues the same matchings bit for bit (flags and `done`
    restart at the step), and a world with another seed refuses it."""
    at, steps = 3, 8
    cfg = _cfg()
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
    assert sds[0]["topology"] == NAME and sds[0]["topology_seed"] == SEED
    other = _world(_cfg(topology_seed=SEED + 1), R)
    with pytest.raises(ValueError, match="topology"):
        other.backends[0].load_state_dict(sds[0])
    other.close()
    b = _world(cfg, R)
    for ar, be, asd, sd in zip(b.arenas, b.backends, arenas, sds):
        ar.load_state_dict(asd)
        be.load_state_dict(sd)
    for s in range(at, steps):
        g = _grads(b, R, 400 + s)
        b.step(g)
        sim.step([x.cpu() for x in g])
        torch.cuda.synchronize()
        _check(b, sim, s + 1)
    for be in b.backends:
        be.check_status()
    b.close()


def test_match_launcher_and_backend_reject_what_they_do_not_run():
    """The match launcher refuses a bad world, rank or seed and a missing pointer before anything is enqueued, and
    every GossipParams setting the step does not run; the backend refuses everything but plain iter-sync decent."""
    from eventgrad_b200.ops.local_world import LocalWorld
    s = torch.cuda.current_stream().cuda_stream
    R = 4
    w = _world(_cfg(), R)
    be = w.backends[0]
    C = be.C
    good = {"world": R, "rank": 0, "seed": SEED, "peers": be.d_match_peers.data_ptr(),
            "inbox": be.win.addr("match_inbox"), "flag_from": be.win.addr("match_flag"),
            "done": be.win.addr("match_done")}
    for bad in ({"world": 1}, {"world": 1025}, {"rank": 4}, {"rank": -1}, {"seed": -1}, {"peers": 0}, {"inbox": 0},
                {"flag_from": 0}, {"done": 0}):
        ms = C.MatchSlots()
        ms.update({**good, **bad})
        with pytest.raises(RuntimeError, match="gossip_step_match"):
            C.gossip_step_match(be.gp, ms, be.grid, s)
    ms = C.MatchSlots()
    ms.update(good)
    for bad, keep in (({"phase": 1}, {"phase": 0}), ({"sync": 0}, {"sync": 1}), ({"do_mix": 0}, {"do_mix": 1}),
                      ({"send_ack": 0}, {"send_ack": 1}), ({"local_steps": 2}, {"local_steps": 1}),
                      ({"global_avg_period": 2}, {"global_avg_period": 0}), ({"quasi_global": 1}, {"quasi_global": 0}),
                      ({"fsm.enabled": 1}, {"fsm.enabled": 0})):
        be.gp.update(bad)
        with pytest.raises(RuntimeError, match="gossip_step_match"):
            C.gossip_step_match(be.gp, ms, be.grid, s)
        be.gp.update(keep)
    torch.cuda.synchronize()
    for be_ in w.backends:
        be_.check_status()
    w.close()
    torch.cuda.synchronize()
    base = dict(algo="decent", dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter")
    ok = TrainConfig(**base).validate()
    for kw in (dict(overlap_push=True), dict(gossip_rounds=2), dict(local_steps=2)):
        bad = ok.replace(**kw)                                    # bypasses validate(): the backend must refuse it
        with pytest.raises(ValueError):
            LocalWorld(bad, 4, lambda: build_model("cnn2"), grid_cap=4, topology=NAME, timeout_ns=1_000_000_000)
    with pytest.raises(ValueError):
        LocalWorld(TrainConfig(**base, topology=NAME).validate().replace(algo="event"), 4, lambda: build_model("cnn2"),
                   grid_cap=4, timeout_ns=1_000_000_000)


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [29700]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "random_match_worker.py"), *args]
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
def test_multigpu_random_match_vs_simulator(world, backend):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", backend, "--steps", "9")
