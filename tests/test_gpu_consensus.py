"""GPU: the consensus distance (--consensus-every N) -- the step-gated consensus kernel of csrc/allreduce.cu after every
step kernel, against the oracle parallel/trigger.py:consensus_stats, and training bit-identical to N = 0.  Multi-rank
runs use R virtual ranks on one GPU (ops.local_world.LocalWorld); the torchrun cases at the end need one GPU per rank
and skip otherwise."""
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import TrainConfig
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.trigger import consensus_stats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the step paths the kernel follows: (algo, TrainConfig overrides); LocalWorld resolves the topology per world
PATHS = {
    "ring": ("decent", dict(double_buffer=False)),
    "dbuf": ("decent", {}),
    "split": ("decent", dict(overlap_push=True)),
    "split_event": ("event", dict(overlap_push=True)),
    "event": ("event", {}),
    "graph": ("decent", dict(topology="exp")),
    "onepeer": ("decent", dict(topology="onepeer-exp")),
    "int8": ("event", dict(compress="int8")),
    "gt": ("decent", dict(gradient_tracking=True)),
    "ed": ("decent", dict(exact_diffusion=True)),
    "local": ("decent", dict(local_steps=2)),
    "pga": ("decent", dict(global_avg_period=3)),
    "qg": ("event", dict(quasi_global_momentum=True)),
    "slowmo": ("decent", dict(slowmo_period=3)),
    "spevent": ("spevent", {}),
}


def _cfg(path, N, **kw):
    algo, over = PATHS[path]
    base = dict(algo=algo, dataset="mnist", model="cnn2", lr=0.05, momentum=0.9, sync_mode="iter",
                consensus_every=N, initial_comm_passes=2)
    base.update(over)
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, model_fn=None, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    return LocalWorld(cfg, R, model_fn or (lambda: build_model("cnn2")), grid_cap=grid_cap, table_mode=table_mode,
                      timeout_ns=5_000_000_000)


def _grads(t, R, seed):
    m = torch.zeros(t.n_padded, device="cuda")
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(t.n_padded, generator=g, device="cuda") * 0.05 * m for _ in range(R)]


def _state(w):
    return [(a.theta.cpu(), None if a.mom is None else a.mom.cpu(), be.bytes_sent(), be.num_events(),
             int(be.d_pass.item())) for a, be in zip(w.arenas, w.backends)]


def _run(path, R, N, steps=7, table_mode=False, model_fn=None, grid_cap=6, **kw):
    """`steps` steps of the world with consensus_every N.  Returns the final training state, every rank's drained
    rows and, per measured step, the oracle's (D, A) of the theta the ranks held after it."""
    w = _world(_cfg(path, N, **kw), R, model_fn, table_mode, grid_cap)
    t = w.arenas[0].table
    rows, oracle = [[] for _ in range(R)], {}
    for s in range(1, steps + 1):
        w.step(_grads(t, R, 100 + s))
        if N and s % N == 0:
            torch.cuda.synchronize()
            oracle[s] = consensus_stats([a.theta.cpu() for a in w.arenas], t)
        if s % 3 == 0 or s == steps:
            for r, be in enumerate(w.backends):
                rows[r] += be.drain_consensus()
    torch.cuda.synchronize()
    for be in w.backends:
        be.check_status()
    st = _state(w)
    w.close()
    return st, rows, oracle


def _check_rows(rows, oracle, R):
    for r in range(R):
        assert [k for k, _, _ in rows[r]] == sorted(oracle), f"rank {r} steps"
        for k, D, A in rows[r]:
            Do, Ao = oracle[k]
            assert torch.allclose(D, Do, rtol=1e-5, atol=0), f"rank {r} step {k} D {D} vs {Do}"
            assert torch.allclose(A, Ao, rtol=1e-5, atol=0), f"rank {r} step {k} A"
        # every rank holds the same bits
        assert all(torch.equal(D, D0) and torch.equal(A, A0) for (_, D, A), (_, D0, A0) in zip(rows[r], rows[0]))
    assert any(float(D.sum()) > 0 for _, D, _ in rows[0])


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("path,R", [("ring", 3), ("dbuf", 4), ("split", 2), ("split", 4), ("split_event", 3),
                                    ("event", 5), ("graph", 8), ("onepeer", 4), ("int8", 3), ("gt", 4), ("ed", 3),
                                    ("local", 4), ("pga", 4), ("qg", 3), ("slowmo", 4), ("spevent", 3)])
def test_consensus_kernel_vs_oracle_and_training_unchanged(path, R, mode):
    """Per tensor within rtol 1e-5 of the oracle at every N-th step, the same bits on every rank, and theta, momentum,
    bytes, events and the step counter bit for bit what N = 0 gives."""
    table_mode = mode == "table"
    if path == "spevent" and table_mode:
        pytest.skip("spevent reads the gradient arena")
    N = 2
    st, rows, oracle = _run(path, R, N, table_mode=table_mode)
    st0, rows0, _ = _run(path, R, 0, table_mode=table_mode)
    assert all(r == [] for r in rows0)
    for r in range(R):
        for x, y in zip(st[r], st0[r]):
            assert (torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y), f"rank {r}"
    _check_rows(rows, oracle, R)


def test_consensus_two_runs_give_the_same_bits():
    _, a, _ = _run("ring", 4, 1, steps=4)
    _, b, _ = _run("ring", 4, 1, steps=4)
    assert all(torch.equal(x[1], y[1]) and torch.equal(x[2], y[2]) for x, y in zip(a[0], b[0]))


@pytest.mark.parametrize("R,path,mode", [(2, "split", "table"), (4, "ring", "flat"), (8, "graph", "table")])
def test_consensus_resnet18_at_the_full_persistent_grid(R, path, mode):
    from eventgrad_b200.ops import ext
    C = ext()
    grid = min(C.gossip_max_grid(0), C.gossip_graph_max_grid(0)) // R
    st, rows, oracle = _run(path, R, 2, steps=4, table_mode=(mode == "table"),
                            model_fn=lambda: build_model("resnet18"), grid_cap=grid, dataset="cifar10",
                            model="resnet18")
    _check_rows(rows, oracle, R)


@pytest.mark.parametrize("R,path,N", [(4, "ring", 2), (3, "split", 3), (4, "pga", 2)])
def test_consensus_captured_graph_equals_eager(R, path, N):
    """Each rank's step kernels plus the gated consensus kernel captured once and replayed over two cycles give the
    eager rows and state: whether a step measures comes from the device pass counter."""
    steps = 2 * N + 1
    res = []
    for captured in (False, True):
        w = _world(_cfg(path, N), R)
        t = w.arenas[0].table
        graphs = []
        if captured:
            torch.cuda.synchronize()
            for r in range(R):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    w.backends[r].launch_pre()
                    w.backends[r].launch()
                graphs.append(g)
            torch.cuda.synchronize()
        cur = torch.cuda.current_stream()
        for s in range(1, steps + 1):
            gr = _grads(t, R, 20 + s)
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
        rows = [be.drain_consensus() for be in w.backends]
        assert [k for k, _, _ in rows[0]] == list(range(N, steps + 1, N))
        res.append((_state(w), rows))
        del graphs
        w.close()
    (s0, r0), (s1, r1) = res
    for r in range(R):
        assert all((torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y) for x, y in zip(s0[r], s1[r]))
        assert all(k0 == k1 and torch.equal(D0, D1) and torch.equal(A0, A1)
                   for (k0, D0, A0), (k1, D1, A1) in zip(r0[r], r1[r]))


def test_consensus_one_rank_launches_nothing():
    from eventgrad_b200.ops import ext
    C = ext()
    w = _world(_cfg("ring", 1), 1)
    t = w.arenas[0].table
    be = w.backends[0]
    assert not be.cons and be.cp is None
    before = dict(C.launch_counts())
    for s in range(3):
        w.step(_grads(t, 1, s))
    after = dict(C.launch_counts())
    assert after.get("allreduce", 0) == before.get("allreduce", 0)
    rows = be.drain_consensus()
    assert [k for k, _, _ in rows] == [1, 2, 3]
    assert all(float(D.abs().sum()) == 0 and float(A.abs().sum()) == 0 for _, D, A in rows)
    D, A = w.measure_consensus()[0]
    assert float(D.abs().sum()) == 0
    w.close()


def test_consensus_ungated_measurement_and_ring_overflow():
    """measure_consensus() measures at any step and leaves earlier rows for the next drain; a ring that wrapped over
    undrained rows raises."""
    R = 3
    w = _world(_cfg("ring", 2), R)
    t = w.arenas[0].table
    for be in w.backends:
        be.set_consensus_capacity(2)
    for s in range(1, 4):
        w.step(_grads(t, R, s))
    got = w.measure_consensus()
    Do, Ao = consensus_stats([a.theta.cpu() for a in w.arenas], t)
    for D, A in got:
        assert torch.allclose(D, Do, rtol=1e-5) and torch.allclose(A, Ao, rtol=1e-5)
    assert [k for k, _, _ in w.backends[0].drain_consensus()] == [2]
    for s in range(4, 11):
        w.step(_grads(t, R, s))
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="overwrote"):
        w.backends[0].drain_consensus()
    w.close()


def test_consensus_launcher_rejects_what_it_does_not_run():
    """The launcher refuses N < 1, a missing gate counter, one-shot mode, null ring or partial buffers and a zero
    capacity before anything is enqueued."""
    s = torch.cuda.current_stream().cuda_stream
    w = _world(_cfg("ring", 2), 3)
    be = w.backends[0]
    good = {"gate_period": 2, "gate_pass": be.d_pass.data_ptr(), "two_shot": 1, "ring": be.cons_ring.data_ptr(),
            "ring_step": be.cons_step.data_ptr(), "ring_ctr": be.cons_ctr.data_ptr(), "cap": be.cons_cap,
            "peer_part": be.d_peer_part.data_ptr(), "part": be.win.addr("cons_part"),
            "tile_tensor": be.d_tile_tensor.data_ptr()}
    bads = [{"gate_period": 0}, {"gate_period": -1}, {"gate_pass": 0}, {"two_shot": 0}, {"ring": 0},
            {"ring_step": 0}, {"ring_ctr": 0}, {"peer_part": 0}, {"part": 0}, {"cap": 0}, {"tile_tensor": 0}]
    for bad in bads:
        be.cp.update(bad)
        with pytest.raises(RuntimeError, match="consensus"):
            be.C.consensus(be.cp, be.grid, s)
        be.cp.update(good)
    torch.cuda.synchronize()
    for b in w.backends:
        b.check_status()
        assert int(b.ar_ctr.item()) == 0 and int(b.cons_ctr.item()) == 0
    w.close()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [30780]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "consensus_worker.py"), *args]
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
def test_multigpu_consensus_vs_simulator(world, algo, topology, backend):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", backend, "--algo", algo, "--topology", topology)
