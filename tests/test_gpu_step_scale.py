"""GPU: the fused step kernels at the product's scale, bit for bit against the simulator (engine.simulator.RingSimulator).

The other multi-rank GPU tests run cnn2 (8 tensors, 20 tiles) on 6-8 CTAs.  These run the ResNet-18 arena (86 tensors,
8 569 tiles, one tensor of 1 152 tiles) and _EdgeNet (tensors of 1, 7, 8, 9, TILE - 1, TILE, TILE + 1 elements, one of
more than 64 tiles and a run of 220 one-tile tensors) at two kinds of persistent grid:
  full      R * grid = the variant's co-resident maximum (_cap), the grid a real run uses;
  uncached  a small grid whose CTAs run more than EG_TI_CACHE tiles, so the step kernel resolves tiles past its cache
            and one CTA completes many tensors (the norm / trigger tail takes several warp rounds).
That reaches what cnn2 never does: the uncached tile look-up, more than 8 tensors finished by one CTA, the steady state
of the iter-sync pipeline, the sparse select's candidate loops and its tie look-back beyond 32 tiles, the two-shot
all-reduce at R = 3, and the scalar gradient tail of table mode with fp32 and bf16 gradients.  Every case also checks
that the padding lanes of every arena-sized buffer stay exactly zero.  R virtual ranks share one GPU
(ops.local_world.LocalWorld) and their grids spin on each other, so no case runs more than _cap(R, variant) CTAs per
rank."""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from eventgrad_b200.config import TrainConfig
from eventgrad_b200.engine.lr_schedule import lr_table
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.arena import TILE
from eventgrad_b200.parallel.trigger import TriggerConfig

pytestmark = pytest.mark.gpu

TI_CACHE = 64      # EG_TI_CACHE (csrc/gossip.cu): tile-info entries the step kernel caches per CTA
WARPS = 8          # EG_WARPS: the norm / trigger tail handles one tensor per warp
SPE = 3            # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=4)
PLAIN = dict(momentum=0.9)


class _EdgeNet(nn.Module):
    """Parameters only (the tests hand in flat gradients).  Default sizes: the tile and 8-lane edges, one tensor of 71
    tiles, 220 one-tile tensors of assorted sizes (most not a multiple of 8) and a short tail."""
    EDGES = (1, 7, 8, 9, TILE - 1, TILE, TILE + 1, 70 * TILE + 3)

    def __init__(self, sizes=None):
        super().__init__()
        if sizes is None:
            sizes = list(self.EDGES) + [1 + (97 * i) % TILE for i in range(220)] + [3 * TILE + 5, 13]
        self.p = nn.ParameterList(nn.Parameter(torch.randn(n) * 0.1) for n in sizes)


def _net(name):
    return (lambda: build_model("resnet18")) if name == "resnet18" else _EdgeNet


def _cap(R, variant):
    """Largest per-rank grid that keeps R grids of `variant` co-resident on the GPU."""
    from eventgrad_b200.ops import ext
    C = ext()
    fn = {"ring": C.gossip_max_grid, "dbuf": C.gossip_dbuf_max_grid, "graph": C.gossip_graph_max_grid,
          "q8": C.gossip_q8_max_grid}[variant]
    return fn(0) // R


def _cfg(algo, opt=OPT, **kw):
    base = dict(algo=algo, dataset="cifar10", model="resnet18", lr=0.05, sync_mode="iter", horizon=1.0, thres_type=1,
                topk_percent=10.0, initial_comm_passes=4, **opt)
    base.update(kw)
    return TrainConfig(**base).validate()


def _one_tile_tensors_per_cta(t, grid):
    """Most one-tile tensors in one CTA's tile set (tiles are strided over the grid: CTA b runs b, b + grid, ...)."""
    n = [0] * grid
    for s, c in zip(t.tile_start, t.tile_count):
        if c == 1:
            n[s % grid] += 1
    return max(n)


def _world(cfg, R, net, grid, variant, table_mode=False):
    from eventgrad_b200.ops.local_world import LocalWorld
    full = _cap(R, variant)
    cap = full if grid == "full" else grid
    assert cap <= full
    w = LocalWorld(cfg, R, _net(net), grid_cap=cap, table_mode=table_mode, timeout_ns=5_000_000_000)
    be, t = w.backends[0], w.arenas[0].table
    assert be.grid <= cap and all(b.grid == be.grid for b in w.backends)
    assert be.dbuf == (variant == "dbuf") and be.q8 == (variant == "q8") and (be.graph is not None) == (variant == "graph")
    if grid != "full":      # the step kernel runs past its tile-info cache
        assert math.ceil(t.n_tiles / be.grid) > TI_CACHE, (t.n_tiles, be.grid)
        if net == "edge":   # ... and one CTA finishes more tensors than it has warps
            assert _one_tile_tensors_per_cta(t, be.grid) > WARPS
    return w


def _mask(t):
    m = torch.zeros(t.n_padded, device="cuda")
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


def _grads(gen, t, R, m, kind):
    out = []
    for _ in range(R):
        if kind == "ties":       # three values: thousands of equal |theta - prev| keys per tensor
            u = torch.rand(t.n_padded, generator=gen, device="cuda")
            g = torch.where(u < 0.3, -0.0625, torch.where(u < 0.6, 0.0, 0.0625)).to(torch.float32)
        else:
            g = torch.randn(t.n_padded, generator=gen, device="cuda") * 0.05
        out.append(g * m)
    return out


def _step_table(w, grads, dtype):
    """One step in table mode: each rank's gradient is a list of per-tensor leaves of `dtype`, read in place by the
    step kernel (P2PBackend.update_grad_table)."""
    t = w.arenas[0].table
    for r in range(w.world):
        leaves = []
        for i in range(t.n_tensors):
            leaf = torch.zeros(t.shapes[i], dtype=dtype, device="cuda", requires_grad=True)
            leaf.grad = w.arenas[r].flat(grads[r], i).reshape(t.shapes[i]).to(dtype).clone()
            leaves.append(leaf)
        w.backends[r].update_grad_table(leaves)
    cur = torch.cuda.current_stream()
    for st in w.streams:
        st.wait_stream(cur)
    for r in range(w.world):
        with torch.cuda.stream(w.streams[r]):
            w.backends[r].step()
    for st in w.streams:
        cur.wait_stream(st)


def _ref_norms(be, t, x):
    """float64 per-tensor L2 norm of an arena-sized buffer whose padding lanes are zero."""
    ss = x.double().square().view(t.n_tiles, TILE).sum(1)
    return torch.zeros(t.n_tensors, dtype=torch.float64, device=x.device).index_add_(
        0, be.d_tile_tensor.long(), ss).sqrt()


def _check_norms(w, when):
    """Norm-on-write (per-warp fp32 partials, fixed-order double reduction per tensor) against float64: ||theta||, or
    ||theta - sent|| under the drift trigger."""
    t = w.arenas[0].table
    for r, (a, be) in enumerate(zip(w.arenas, w.backends)):
        x = a.theta.double() - be.sent.double() if be.drift else a.theta
        torch.testing.assert_close(be.cur_norm.double(), _ref_norms(be, t, x), rtol=3e-6, atol=0,
                                   msg=lambda m: f"{when}, rank {r}: norm-on-write differs from float64\n{m}")


def _lookback_past_32_tiles(diff, k):
    """True when the tie look-back of sparse_compact_kernel walks further than 32 tiles for this tensor: some tile
    holding keys equal to tau (the k-th largest |theta - prev|) sits 33 or more tiles into the tensor and the 32 tiles
    before it hold fewer ties than the record takes."""
    n = diff.numel()
    tau = diff.kthvalue(n - k + 1).values
    need = k - int((diff > tau).sum())
    q = F.pad((diff == tau).int(), (0, (-n) % TILE)).view(-1, TILE).sum(1)
    c = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(q, 0)])      # c[j]: ties in tiles [0, j)
    tt = torch.nonzero(q).flatten()
    tt = tt[tt >= 33]
    return bool(((c[tt] - c[tt - 32]) < need).any())


def _run(w, cfg, steps, seed, grads="gauss", table_dtype=None, ties_probe=False):
    """`steps` steps on the world and the simulator; returns the simulator after the end-of-run checks."""
    R, t = w.world, w.arenas[0].table
    m = _mask(t)
    pad = m == 0
    sched = lr_table(cfg, SPE) if cfg.lr_schedule != "constant" else None
    for be in w.backends:
        if sched is not None:
            be.set_lr_table(sched)
    sim = RingSimulator(R, w.arenas[0].theta.cpu(), t, cfg.algo, TriggerConfig.from_train(cfg), lr=cfg.lr,
                        momentum=cfg.momentum, topk_percent=cfg.topk_percent, serial_skip=False,
                        weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=sched, offsets=w.cfg.topology,
                        compress=cfg.compress)
    trig = cfg.algo in ("event", "spevent")
    gen = torch.Generator(device="cuda").manual_seed(seed)
    deep_ties = False
    for s in range(1, steps + 1):
        fires = norms = None
        if trig:      # the kernel's decisions for this step and the norms it took them from
            fires = [be.fire.clone().bool().cpu() for be in w.backends]
            norms = [be.cur_norm.clone().cpu() for be in w.backends]
            _check_norms(w, f"before step {s}")
        g = _grads(gen, t, R, m, grads)
        if table_dtype is not None:
            g = [x.to(table_dtype).float() for x in g]      # what the kernel reads from the bf16 leaves
            _step_table(w, g, table_dtype)
        else:
            w.step(g)
        if ties_probe and not deep_ties:
            for r in range(R):
                for i in range(t.n_tensors):
                    if fires[r][i] and t.tile_count[i] > 33:
                        o, n = t.offsets[i], t.numels[i]
                        diff = (sim.theta[r][o:o + n] - sim.prev[r][o:o + n]).abs()
                        deep_ties = deep_ties or _lookback_past_32_tiles(diff, sim.k[i])
        # the oracle FSM runs on the kernel's norms; its decisions must be the kernel's
        sim.step([x.cpu() for x in g], norms=norms)
        if trig:
            for r in range(R):
                assert torch.equal(fires[r], sim.fire_history[-1][r]), f"step {s} rank {r}: fire mask differs"
    torch.cuda.synchronize()
    if ties_probe:
        assert deep_ties, "no tie look-back walked past 32 tiles: the heavy-tie case missed its target"
    if trig:
        _check_norms(w, f"after step {steps}")
    for r, (a, be) in enumerate(zip(w.arenas, w.backends)):
        be.check_status()
        assert torch.equal(a.theta.cpu(), sim.theta[r]), f"rank {r}: theta differs"
        assert torch.equal(a.mom.cpu(), sim.mom[r]), f"rank {r}: momentum differs"
        if be.sparse or be.q8:
            assert torch.equal(be.prev.cpu(), sim.prev[r]), f"rank {r}: prev differs"
            assert torch.equal(be.rep_l.cpu(), sim.rep_l[r]), f"rank {r}: rep_l differs"
            assert torch.equal(be.rep_r.cpu(), sim.rep_r[r]), f"rank {r}: rep_r differs"
        if be.drift:
            assert torch.equal(be.sent.cpu(), sim.sent[r]), f"rank {r}: sent differs"
        assert be.num_events() == sim.events[r], f"rank {r}: events"
        assert be.bytes_sent() == sim.bytes[r], f"rank {r}: bytes"
        assert int(be.d_pass.item()) == steps
        assert int(a.grad.count_nonzero()) == 0, f"rank {r}: gradient arena not zero after the step"
        bufs = {"theta": a.theta, "mom": a.mom}
        for k in ("prev", "rep_l", "rep_r", "sent"):
            if getattr(be, k, None) is not None:
                bufs[k] = getattr(be, k)
        for k, x in bufs.items():
            assert int(x[pad].count_nonzero()) == 0, f"rank {r}: padding lanes of {k} are not zero"
    return sim


# ---------------------------------------------------------------------------------------------------------- decent
DECENT_KW = {"dbuf": dict(), "single": dict(double_buffer=False), "split": dict(overlap_push=True)}


@pytest.mark.parametrize("variant,R,grid", [(v, R, "full") for v in DECENT_KW for R in (2, 3, 4)]
                         + [(v, 2, 8) for v in DECENT_KW])
def test_decent_resnet_bitwise_vs_simulator(variant, R, grid):
    cfg = _cfg("decent", opt=OPT if grid == "full" else PLAIN, **DECENT_KW[variant])
    w = _world(cfg, R, "resnet18", grid, "dbuf" if variant == "dbuf" else "ring")
    assert all(be.overlap == (variant == "split") for be in w.backends)
    _run(w, cfg, 7, 100 + R)
    w.close()


# ----------------------------------------------------------------------------------------------------------- event
@pytest.mark.parametrize("trigger,R,grid", [(tr, R, "full") for tr in ("norm", "drift") for R in (2, 3)]
                         + [(tr, 2, 8) for tr in ("norm", "drift")])
def test_event_resnet_bitwise_vs_simulator(trigger, R, grid):
    cfg = _cfg("event", opt=OPT if grid == "full" else PLAIN, trigger=trigger)
    w = _world(cfg, R, "resnet18", grid, "ring")
    sim = _run(w, cfg, 8, 200 + R)
    fired = sum(int(f.sum()) for h in sim.fire_history for f in h)
    assert 0 < fired < 8 * R * w.arenas[0].table.n_tensors      # the trigger both fired and held
    w.close()


# --------------------------------------------------------------------------------------------------------- spevent
@pytest.mark.parametrize("pct,grads,R,net,grid",
                         [(p, g, R, "resnet18", "full") for p in (1.0, 10.0) for g in ("gauss", "ties") for R in (2, 3)]
                         + [(10.0, "ties", 2, "resnet18", 8)]
                         + [(10.0, g, 2, "edge", grid) for g in ("gauss", "ties") for grid in (1, 3, "full")])
def test_spevent_bitwise_vs_simulator(pct, grads, R, net, grid):
    ties = grads == "ties"
    cfg = _cfg("spevent", opt=dict(momentum=0.0) if ties else PLAIN, topk_percent=pct, initial_comm_passes=3)
    w = _world(cfg, R, net, grid, "ring")
    _run(w, cfg, 5, 300 + R, grads=grads, ties_probe=ties and net == "resnet18")
    w.close()


# ------------------------------------------------------------------------------------------------------------ int8
@pytest.mark.parametrize("algo,R,net,grid", [(a, R, "resnet18", "full") for a in ("decent", "event") for R in (2, 4)]
                         + [(a, 2, "edge", 3) for a in ("decent", "event")])
def test_q8_bitwise_vs_simulator(algo, R, net, grid):
    trigger = "drift" if (algo == "event" and R == 4) else "norm"
    cfg = _cfg(algo, opt=OPT if grid == "full" else PLAIN, compress="int8", trigger=trigger)
    w = _world(cfg, R, net, grid, "q8")
    _run(w, cfg, 7, 400 + R)
    w.close()


# ----------------------------------------------------------------------------------------------------------- graphs
@pytest.mark.parametrize("R,topology", [(8, "exp"), (4, "onepeer-exp")])
def test_graph_resnet_bitwise_vs_simulator(R, topology):
    cfg = _cfg("event", topology=topology)
    w = _world(cfg, R, "resnet18", "full", "graph")
    _run(w, cfg, 6, 500 + R)
    w.close()


# ------------------------------------------------------------------------------------------------------------- cent
@pytest.mark.parametrize("two_shot", [0, 1])
@pytest.mark.parametrize("R", [2, 3, 4])
def test_cent_resnet_bitwise_vs_simulator(R, two_shot):
    cfg = _cfg("cent")
    w = _world(cfg, R, "resnet18", "full", "ring")
    for be in w.backends:
        be.ap.update({"two_shot": two_shot})
    _run(w, cfg, 6, 600 + R)
    w.close()


@pytest.mark.parametrize("net", ["resnet18", "edge"])
def test_final_average_two_shot_r3(net):
    R = 3
    cfg = _cfg("event")
    w = _world(cfg, R, net, "full", "ring")
    t = w.arenas[0].table
    m = _mask(t)
    gen = torch.Generator(device="cuda").manual_seed(7)
    vals = [torch.randn(t.n_padded, generator=gen, device="cuda") * m for _ in range(R)]
    for r in range(R):
        w.arenas[r].theta.copy_(vals[r])
    torch.cuda.synchronize()
    w.final_average()
    # on the CPU: CUDA torch divides by a Python scalar as a multiply by its reciprocal, the kernel truly divides
    a, b, c = (v.cpu() for v in vals)
    ref = ((a + b) + c) / 3.0
    for r in range(R):
        assert torch.equal(w.arenas[r].theta.cpu(), ref), f"rank {r}"
        assert int(w.arenas[r].theta[m == 0].count_nonzero()) == 0
    w.close()


# -------------------------------------------------------------------------------------------------- table mode, edges
@pytest.mark.parametrize("grid", [1, 3, "full"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("algo", ["decent", "event"])
def test_table_mode_edge_sizes_bitwise_vs_simulator(algo, dtype, grid):
    cfg = _cfg(algo)
    w = _world(cfg, 2, "edge", grid, "dbuf" if algo == "decent" else "ring", table_mode=True)
    t = w.arenas[0].table
    assert all(be.table_mode for be in w.backends)
    assert set(_EdgeNet.EDGES) <= set(t.numels) and sum(n % 8 != 0 for n in t.numels) > 100
    _run(w, cfg, 8, 700, table_dtype=dtype)
    w.close()


def test_more_than_1024_tensors_is_refused():
    from eventgrad_b200.parallel.p2p import P2PBackend, preallocate_arena_buffers
    from eventgrad_b200.parallel import ParamArena, Ring
    from eventgrad_b200.utils.dist import DistEnv
    cfg = _cfg("event")
    env = DistEnv(0, 1, 0, torch.device("cuda", 0), "none")
    model = _EdgeNet([1] * 1025)
    theta, grad, symm = preallocate_arena_buffers(model, cfg, env)
    arena = ParamArena(model, env.device, theta=theta, grad=grad)
    with pytest.raises(ValueError, match="EG_MAX_OWN"):
        P2PBackend(cfg, arena, Ring(0, 1), env, symm=symm, timeout_ns=5_000_000_000)
    symm["window"].close()
