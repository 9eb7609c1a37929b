"""GPU: the drift trigger (--trigger drift) in the fused step kernels -- every pushed tile also stores theta_k into
`sent`, and norm-on-write accumulates ||theta_{k+1} - sent|| for the device FSM.  Multi-rank runs use R virtual ranks on
one GPU (ops.local_world.LocalWorld) and compare with the simulator bit for bit at every step."""
import pytest
import torch

from eventgrad_b200.config import TrainConfig
from eventgrad_b200.engine.lr_schedule import lr_table
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.trigger import TriggerConfig, TriggerState, trigger_step

pytestmark = pytest.mark.gpu

SPE = 3          # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=4)


def _cfg(algo="event", **kw):
    base = dict(algo=algo, dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", horizon=1.0, thres_type=1,
                initial_comm_passes=4, trigger="drift", **OPT)
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, topology=None, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    return LocalWorld(cfg, R, lambda: build_model("cnn2"), grid_cap=grid_cap, topology=topology,
                      table_mode=table_mode, timeout_ns=5_000_000_000)


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


def _sim(cfg, w, R, table, topology="ring", **kw):
    return RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, cfg.algo, TriggerConfig.from_train(cfg),
                         lr=cfg.lr, momentum=cfg.momentum, serial_skip=False, weight_decay=cfg.weight_decay,
                         nesterov=cfg.nesterov, lr_table=table, offsets=topology, **kw)


def _kernel_view(w, R, sim):
    """The kernel's decisions for the coming step and the drift values it took them from (checked against the
    simulator's own drift to float tolerance)."""
    fires = [be.fire.clone().bool().cpu() for be in w.backends]
    norms = [be.cur_norm.clone().cpu() for be in w.backends]
    for r in range(R):
        torch.testing.assert_close(norms[r], sim.trigger_norms(r), rtol=3e-6, atol=1e-7)
    return fires, norms


def _check(w, sim, R, s, fires):
    for r, be in enumerate(w.backends):
        assert torch.equal(fires[r], sim.fire_history[-1][r]), f"step {s} rank {r} fire mask differs from the oracle"
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} rank {r} theta differs"
        assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s} rank {r} momentum differs"
        assert torch.equal(be.sent.cpu(), sim.sent[r]), f"step {s} rank {r} sent differs"
        assert be.num_events() == sim.events[r], f"step {s} rank {r} events"
        assert be.bytes_sent() == sim.bytes[r], f"step {s} rank {r} bytes"


def _run(cfg, R, topology, mode, steps=10, grad_seed=40):
    w = _world(cfg, R, topology=topology, table_mode=(mode == "table"))
    assert all(be.drift and be.sent is not None for be in w.backends)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table, topology)
    fired = held = 0
    for s in range(1, steps + 1):
        fires, norms = _kernel_view(w, R, sim)
        fired += sum(int(f.sum()) for f in fires)
        held += sum(int((~f).sum()) for f in fires)
        g = _grads(w, R, grad_seed + s)
        w.step(g)
        sim.step([x.cpu() for x in g], norms=norms)
        torch.cuda.synchronize()
        _check(w, sim, R, s, fires)
    for r, be in enumerate(w.backends):
        be.check_status()
        assert int(be.d_pass.item()) == steps
        nxt = trigger_step(sim.state[r].clone(), be.cur_norm.cpu(), sim.pass_num + 1, sim.tcfg)
        assert torch.equal(nxt, be.fire.bool().cpu())
    assert held > 0 and fired > 0, (fired, held)
    w.close()


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("R,topology", [(2, "ring"), (3, "ring"), (4, "exp"), (5, "exp"), (8, "exp"), (5, "2"),
                                        (4, "onepeer-exp"), (5, "onepeer-exp")])
def test_drift_event_bitwise_vs_simulator(R, topology, mode):
    _run(_cfg(), R, topology, mode)


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("pct", [1.0, 10.0, 100.0])
def test_drift_spevent_vs_simulator(R, pct):
    cfg = _cfg("spevent", topk_percent=pct)
    w = _world(cfg, R)
    assert all(be.sent is be.prev for be in w.backends)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table, topk_percent=pct)
    for s in range(1, 11):
        fires, norms = _kernel_view(w, R, sim)
        g = _grads(w, R, 900 + s)
        w.step(g)
        sim.step([x.cpu() for x in g], norms=norms)
        torch.cuda.synchronize()
        for r, be in enumerate(w.backends):
            assert torch.equal(fires[r], sim.fire_history[-1][r]), f"step {s} rank {r} fire mask"
            assert torch.equal(be.prev.cpu(), sim.prev[r]), f"step {s} prev rank {r}"
            assert torch.equal(be.rep_l.cpu(), sim.rep_l[r]), f"step {s} rep_l rank {r}"
            assert torch.equal(be.rep_r.cpu(), sim.rep_r[r]), f"step {s} rep_r rank {r}"
            assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} theta rank {r}"
            assert be.num_events() == sim.events[r] and be.bytes_sent() == sim.bytes[r]
    for be in w.backends:
        be.check_status()
    w.close()


def test_drift_spevent_fresh_replicas_redecides_from_the_new_prev():
    """--fresh-replicas: prev starts at a random network, and the first decision is taken from theta_0 - prev."""
    R = 2
    cfg = _cfg("spevent", initial_comm_passes=1, spevent_fresh_replicas=True)
    w = _world(cfg, R)
    t = w.arenas[0].table
    m = _mask(t)
    gen = torch.Generator(device="cuda").manual_seed(11)
    extra = [torch.randn(t.n_padded, generator=gen, device="cuda") * m for _ in range(3)]
    for be in w.backends:
        be.set_sparse_init(*extra)
    torch.cuda.synchronize()
    sim = _sim(cfg, w, R, None, sparse_init=tuple(x.cpu() for x in extra))
    for s in range(1, 6):
        fires, norms = _kernel_view(w, R, sim)
        g = _grads(w, R, 300 + s)
        w.step(g)
        sim.step([x.cpu() for x in g], norms=norms)
        torch.cuda.synchronize()
        for r, be in enumerate(w.backends):
            assert torch.equal(fires[r], sim.fire_history[-1][r]), f"step {s} rank {r} fire mask"
            assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} theta rank {r}"
            assert torch.equal(be.prev.cpu(), sim.prev[r])
    w.close()


def test_drift_split_step_equals_fused_step():
    """Ring, R = 3, event: the split step (push phase on a side stream, then wait + mix) equals the fused step."""
    R, steps = 3, 9
    out = []
    for overlap in (False, True):
        w = _world(_cfg(overlap_push=overlap), R)
        assert all(be.overlap == overlap for be in w.backends)
        hist = []
        for s in range(1, steps + 1):
            w.step(_grads(w, R, 70 + s))
            torch.cuda.synchronize()
            hist.append([(a.theta.clone(), be.sent.clone(), be.fire.clone(), be.cur_norm.clone(), be.counters.clone())
                         for a, be in zip(w.arenas, w.backends)])
        for be in w.backends:
            be.check_status()
        out.append(hist)
        w.close()
    for s, (a, b) in enumerate(zip(*out)):
        for r in range(R):
            for x, y in zip(a[r], b[r]):
                assert torch.equal(x, y), f"step {s + 1} rank {r}"


@pytest.mark.parametrize("topology", ["ring", "exp"])
def test_drift_captured_graph_equals_eager(topology):
    """Each rank's step captured once in a CUDA graph and replayed 10 times equals eager execution."""
    R, steps = 4, 10
    res = []
    for captured in (False, True):
        cfg = _cfg()
        w = _world(cfg, R, topology=topology)
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
        res.append([(a.theta.cpu(), be.sent.cpu(), be.fire.cpu(), be.counters.cpu())
                    for a, be in zip(w.arenas, w.backends)])
        del graphs
        w.close()
    for r in range(R):
        for x, y in zip(res[0][r], res[1][r]):
            assert torch.equal(x, y), f"rank {r}"


def test_fsm_decide_drift_metric_vs_oracle():
    cfg = _cfg(horizon=0.9, initial_comm_passes=3)
    w = _world(cfg, 1)
    be = w.backends[0]
    sz = w.arenas[0].table.n_tensors
    tc = TriggerConfig.from_train(cfg)
    assert tc.metric == "drift"
    be.gp.update({"fsm.metric": 1})
    st = TriggerState(sz, cfg.sent_history)
    for x in (be.thres, be.last_norm, be.last_iter, be.slopes):
        x.zero_()
    be.d_pass.zero_()
    g = torch.Generator().manual_seed(0)
    for k in range(1, 40):
        drift = torch.rand(sz, generator=g) * 0.02 * (1 + (k % 7 == 0) * 5)
        dn = drift.float().cuda()
        be.C.fsm_decide(be.gp, dn.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        fire = trigger_step(st, drift.float(), k, tc)
        assert torch.equal(be.fire.cpu().bool(), fire), f"step {k}"
        assert torch.equal(be.thres.cpu(), st.thres)
        assert torch.equal(be.last_norm.cpu(), st.last_norm)
        assert torch.equal(be.cur_norm.cpu(), drift.float())
        assert torch.equal(be.slopes.cpu().view(sz, -1), st.slopes)
    w.close()


@pytest.mark.parametrize("R,topology", [(3, "ring"), (4, "exp"), (4, "onepeer-exp")])
def test_drift_async_runs_clean(R, topology):
    cfg = _cfg(sync_mode="async")
    w = _world(cfg, R, topology=topology)
    steps = 12
    for s in range(steps):
        w.step(_grads(w, R, 90 + s))
        torch.cuda.synchronize()
    for r, be in enumerate(w.backends):
        be.check_status()
        assert int(be.status.item()) == 0
        assert bool(torch.isfinite(w.arenas[r].theta).all())
        assert int(be.d_pass.item()) == steps
    w.close()


def test_drift_p2p_checkpoint_round_trip_and_trigger_guard():
    """state_dict carries `sent` and the trigger; loading it into a fresh world continues bit for bit, and a norm
    backend refuses it."""
    R = 3
    cfg = _cfg()
    a = _world(cfg, R)
    for s in range(5):
        a.step(_grads(a, R, 400 + s))
    torch.cuda.synchronize()
    sds = [be.state_dict() for be in a.backends]
    arenas = [ar.state_dict() for ar in a.arenas]
    assert all(sd["trigger"] == "drift" and "sent" in sd for sd in sds)
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
        assert torch.equal(a.arenas[r].theta, b.arenas[r].theta)
        assert torch.equal(a.backends[r].sent, b.backends[r].sent)
        assert torch.equal(a.backends[r].counters, b.backends[r].counters)
    b.close()
    n = _world(_cfg(trigger="norm"), R)
    with pytest.raises(ValueError, match="trigger"):
        n.backends[0].load_state_dict(sds[0])
    n.close()
    a.close()
