"""GPU: the 1-bit scaled-sign codec (--compress sign) and the CHOCO mix (--choco-gamma) in the fused compressed ring step
kernel (csrc/gossip_q8.cu).  Multi-rank runs use R virtual ranks on one GPU (ops.local_world.LocalWorld) and compare
with the fp32 simulator bit for bit at every step; the torchrun cases at the end need one GPU per rank and skip
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
from eventgrad_b200.parallel.arena import TILE
from eventgrad_b200.parallel.trigger import Q8_BLOCK, TriggerConfig, sign_decode, sign_encode, trigger_step

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPE = 3          # steps per epoch of the test schedule: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=4)


def _cfg(algo="event", compress="sign", gamma=0.5, **kw):
    base = dict(algo=algo, dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", horizon=1.0, thres_type=1,
                initial_comm_passes=4, compress=compress, choco_gamma=gamma, **OPT)
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, table_mode=False, grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    return LocalWorld(cfg, R, lambda: build_model("cnn2"), grid_cap=grid_cap, table_mode=table_mode,
                      timeout_ns=5_000_000_000)


def _mask(t, device="cuda"):
    m = torch.zeros(t.n_padded, device=device)
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    return m


def _grads(w, R, seed):
    t = w.arenas[0].table
    m = _mask(t)
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(t.n_padded, generator=g, device="cuda") * 0.05 * m for _ in range(R)]


def _sim(cfg, w, R, table):
    return RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, cfg.algo, TriggerConfig.from_train(cfg),
                         lr=cfg.lr, momentum=cfg.momentum, serial_skip=False, weight_decay=cfg.weight_decay,
                         nesterov=cfg.nesterov, lr_table=table, compress=cfg.compress, choco_gamma=cfg.choco_gamma)


def _replica_invariant(w, R, s):
    for r in range(R):
        L, Rn = (r - 1) % R, (r + 1) % R
        prev = w.backends[r].prev
        assert torch.equal(w.backends[L].rep_r, prev), f"step {s}: rank {L}'s rep_r is not rank {r}'s prev"
        assert torch.equal(w.backends[Rn].rep_l, prev), f"step {s}: rank {Rn}'s rep_l is not rank {r}'s prev"


def _run(cfg, R, mode, steps=10, grad_seed=40):
    w = _world(cfg, R, table_mode=(mode == "table"))
    assert all(be.q8 and be.qs is not None and not be.overlap and not be.dbuf for be in w.backends)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
    sim = _sim(cfg, w, R, table)
    event = cfg.algo == "event"
    fired = held = 0
    for s in range(1, steps + 1):
        fires = [be.fire.clone().bool().cpu() for be in w.backends]
        norms = [be.cur_norm.clone().cpu() for be in w.backends]
        fired += sum(int(f.sum()) for f in fires)
        held += sum(int((~f).sum()) for f in fires)
        g = _grads(w, R, grad_seed + s)
        w.step(g)
        # the oracle FSM runs on the kernel's norms; its decisions must be the kernel's
        sim.step([x.cpu() for x in g], norms=norms if event else None)
        torch.cuda.synchronize()
        for r, be in enumerate(w.backends):
            if event:
                assert torch.equal(fires[r], sim.fire_history[-1][r]), f"step {s} rank {r} fire mask"
            assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"step {s} rank {r} theta"
            assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"step {s} rank {r} momentum"
            assert torch.equal(be.prev.cpu(), sim.prev[r]), f"step {s} rank {r} prev"
            assert torch.equal(be.rep_l.cpu(), sim.rep_l[r]), f"step {s} rank {r} rep_l"
            assert torch.equal(be.rep_r.cpu(), sim.rep_r[r]), f"step {s} rank {r} rep_r"
            assert be.num_events() == sim.events[r], f"step {s} rank {r} events"
            assert be.bytes_sent() == sim.bytes[r], f"step {s} rank {r} bytes"
        _replica_invariant(w, R, s)
    for r, be in enumerate(w.backends):
        be.check_status()
        assert int(be.d_pass.item()) == steps
        if event:
            nxt = trigger_step(sim.state[r].clone(), be.cur_norm.cpu(), sim.pass_num + 1, sim.tcfg)
            assert torch.equal(nxt, be.fire.bool().cpu())
    if event:
        assert held > 0 and fired > 0, (fired, held)
    w.close()


# int8 with the error-feedback mix (gamma 0) is test_gpu_compress.py's matrix
CODEC_MIX = [("int8", 0.2), ("int8", 0.5), ("sign", 0.0), ("sign", 0.2), ("sign", 0.5)]


@pytest.mark.parametrize("mode", ["flat", "table"])
@pytest.mark.parametrize("algo,trigger", [("decent", "norm"), ("event", "norm"), ("event", "drift")])
@pytest.mark.parametrize("compress,gamma", CODEC_MIX)
@pytest.mark.parametrize("R", [2, 3, 4, 8])
def test_choco_bitwise_vs_simulator(R, compress, gamma, algo, trigger, mode):
    _run(_cfg(algo, compress, gamma, trigger=trigger), R, mode)


def test_sign_codec_edge_cases_through_the_kernel():
    """One step at lr = 0, mu = 0 from crafted theta / prev: the kernel's new prev is sign_encode's, bit for bit --
    zero blocks, +-0, a subnormal scale, a scale that underflows to 0, and the partial last tiles of small tensors."""
    R = 2
    cfg = _cfg("decent", "sign", 0.0, momentum=0.0, nesterov=False, weight_decay=0.0, lr=0.0,
               lr_schedule="constant", lr_warmup_epochs=0.0)
    w = _world(cfg, R)
    t = w.arenas[0].table
    m = _mask(t, "cpu")
    g = torch.Generator().manual_seed(17)
    thetas, prevs = [], []
    for r in range(R):
        th = torch.randn(t.n_padded, generator=g) * m
        pv = (th + torch.randn(t.n_padded, generator=g) * 1e-3) * m
        i = max(range(t.n_tensors), key=lambda k: t.numels[k])       # a tensor with several blocks
        o = t.offsets[i]
        pv[o:o + Q8_BLOCK] = th[o:o + Q8_BLOCK]                         # a zero block
        b = o + Q8_BLOCK                                                 # signed zeros
        th[b:b + Q8_BLOCK] = pv[b:b + Q8_BLOCK]
        th[b:b + 4] = torch.tensor([0.0, -0.0, 0.0, -0.0])
        pv[b:b + 4] = torch.tensor([-0.0, 0.0, 0.0, -0.0])
        th[b + 9] = pv[b + 9] + 1.0
        b += Q8_BLOCK                                                    # subnormal scale
        th[b:b + Q8_BLOCK] = pv[b:b + Q8_BLOCK]
        pv[b + 3], th[b + 3] = 0.0, -3e-38
        b += Q8_BLOCK                                                    # a scale that underflows to zero
        th[b:b + Q8_BLOCK] = pv[b:b + Q8_BLOCK]
        pv[b + 5], th[b + 5] = 0.0, 1e-45
        thetas.append(th)
        prevs.append(pv)
    assert any(n % TILE for n in t.numels)
    for r in range(R):
        w.arenas[r].theta.copy_(thetas[r].cuda())
        w.backends[r].prev.copy_(prevs[r].cuda())
        other = w.backends[1 - r]
        other.rep_l.copy_(prevs[r].cuda())
        other.rep_r.copy_(prevs[r].cuda())
    torch.cuda.synchronize()
    w.step([torch.zeros(t.n_padded, device="cuda") for _ in range(R)])
    torch.cuda.synchronize()
    for r, be in enumerate(w.backends):
        be.check_status()
        bits, s = sign_encode(thetas[r] - prevs[r])
        assert float(s[(t.offsets[i] + 2 * Q8_BLOCK) // Q8_BLOCK]) != 0.0     # the subnormal scale survives
        want = prevs[r].clone()
        for o, n, c in zip(t.offsets, t.numels, t.tile_count):             # tensor by tensor: padding decodes to 0
            span = slice(o, o + c * t.tile)
            want[span] += sign_decode(bits[o // 8:(o + c * t.tile) // 8], s[o // Q8_BLOCK:(o + c * t.tile) // Q8_BLOCK],
                                      n)
        assert torch.equal(be.prev.cpu(), want), f"rank {r}: prev differs from sign_encode's"
        assert bool((be.prev.cpu()[m == 0] == 0).all())
    _replica_invariant(w, R, 1)
    w.close()


@pytest.mark.parametrize("compress", ["int8", "sign"])
def test_choco_captured_graph_equals_eager(compress):
    """Each rank's step captured once in a CUDA graph and replayed 10 times equals eager execution."""
    R, steps = 4, 10
    res = []
    for captured in (False, True):
        cfg = _cfg(compress=compress, gamma=0.5, trigger="drift")
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
        res.append([(a.theta.cpu(), be.prev.cpu(), be.rep_l.cpu(), be.rep_r.cpu(), be.fire.cpu(), be.counters.cpu())
                    for a, be in zip(w.arenas, w.backends)])
        del graphs
        w.close()
    for r in range(R):
        for x, y in zip(res[0][r], res[1][r]):
            assert torch.equal(x, y), f"rank {r}"


@pytest.mark.parametrize("algo", ["decent", "event"])
def test_choco_checkpoint_round_trip_and_guards(algo):
    """state_dict carries `compress` = "sign" and `choco_gamma`; a fresh world continues bit for bit from it, and
    worlds under another gamma, gamma 0 or the int8 codec refuse it."""
    R = 3
    cfg = _cfg(algo, "sign", 0.5)
    a = _world(cfg, R)
    for s in range(5):
        a.step(_grads(a, R, 400 + s))
    torch.cuda.synchronize()
    sds = [be.state_dict() for be in a.backends]
    arenas = [ar.state_dict() for ar in a.arenas]
    assert all(sd["compress"] == "sign" and sd["choco_gamma"] == 0.5 and "prev" in sd for sd in sds)
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
                     (a.backends[r].prev, b.backends[r].prev), (a.backends[r].rep_l, b.backends[r].rep_l),
                     (a.backends[r].rep_r, b.backends[r].rep_r), (a.backends[r].counters, b.backends[r].counters)):
            assert torch.equal(x, y), f"rank {r}"
        a.backends[r].check_status()
        b.backends[r].check_status()
    b.close()
    for kw, match in ((dict(gamma=0.2), "choco-gamma"), (dict(gamma=0.0), "choco-gamma"),
                      (dict(compress="int8"), "compress")):
        n = _world(_cfg(algo, **{"compress": "sign", "gamma": 0.5, **kw}), R)
        with pytest.raises(ValueError, match=match):
            n.backends[0].load_state_dict(sds[0])
        n.close()
    a.close()


def test_choco_launcher_rejects_what_it_does_not_run():
    cfg = _cfg()
    w = _world(cfg, 2)
    be = w.backends[0]
    s = torch.cuda.current_stream().cuda_stream
    # every case is refused before anything is enqueued
    for bad in ({"codec": 2}, {"codec": -1}, {"gamma": -0.5}, {"gamma": 1.5}, {"gamma": float("nan")},
                {"gamma": float("inf")}):
        be.qs.update(bad)
        with pytest.raises(RuntimeError, match="gossip_step_q8"):
            be.C.gossip_step_q8(be.gp, be.qs, be.grid, s)
        be.qs.update({"codec": 1, "gamma": 0.5})
    torch.cuda.synchronize()
    w.close()


def test_choco_lr0_keeps_the_mean_within_rounding():
    """lr = 0, mu = 0, sign + CHOCO gamma 0.2 at R = 4 from a spread start, 300 steps: the kernel equals the fp32
    simulator bit for bit, so the drift of the ranks' mean is the fp32 simulator's.  It is bounded by the rounding of
    the per-step ops: a few ulps of |theta| per step and rank, accumulated as a random walk -- checked against
    sqrt(steps) * 8 ulps of max|theta| -- while the consensus distance shrinks."""
    R, steps = 4, 300
    cfg = _cfg("decent", "sign", 0.2, momentum=0.0, nesterov=False, weight_decay=0.0, lr=0.0,
               lr_schedule="constant", lr_warmup_epochs=0.0)
    w = _world(cfg, R)
    t = w.arenas[0].table
    m = _mask(t, "cpu")
    g = torch.Generator().manual_seed(5)
    start = [torch.randn(t.n_padded, generator=g) * m for _ in range(R)]
    # prev and the replicas keep the common theta_0 the backends were built with
    sim = RingSimulator(R, w.arenas[0].theta.cpu(), t, "decent", lr=0.0, serial_skip=False, compress="sign",
                        choco_gamma=0.2)
    for r in range(R):
        w.arenas[r].theta.copy_(start[r].cuda())
    for r in range(R):
        sim.theta[r] = start[r].clone()
    zero_d = [torch.zeros(t.n_padded, device="cuda") for _ in range(R)]
    zero_h = [torch.zeros(t.n_padded) for _ in range(R)]
    mean0 = torch.stack([x.double() for x in start]).mean(0)

    def spread(th):
        bar = torch.stack([x.double() for x in th]).mean(0)
        return max(float((x.double() - bar).abs().max()) for x in th)

    s0 = spread(start)
    for s in range(steps):
        w.step(zero_d)
        sim.step(zero_h)
    torch.cuda.synchronize()
    got = [a.theta.cpu() for a in w.arenas]
    for r in range(R):
        w.backends[r].check_status()
        assert torch.equal(got[r], sim.theta[r]), f"rank {r}"
    drift = float((torch.stack([x.double() for x in got]).mean(0) - mean0).abs().max())
    ulp = float(torch.finfo(torch.float32).eps) * float(max(x.abs().max() for x in start))
    assert drift <= 8 * ulp * steps ** 0.5, (drift, ulp)
    assert spread(got) < 0.5 * s0, (spread(got), s0)
    w.close()


# ---------------------------------------------------------------------------------------- one process per GPU
_PORT = [29950]


def _torchrun(world, *args):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "choco_worker.py"), *args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "WORKER_OK" in out, out[-3000:]


def _need(world):
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < world:
        pytest.skip(f"needs {world} GPUs, found {n}")


@pytest.mark.multigpu
@pytest.mark.parametrize("backend", ["p2p", "nccl"])
@pytest.mark.parametrize("algo", ["decent", "event"])
@pytest.mark.parametrize("world", [2, 4])
def test_multigpu_choco_vs_simulator(world, algo, backend):
    _need(world)
    _torchrun(world, "--mode", "sim", "--backend", backend, "--algo", algo, "--compress", "sign", "--gamma", "0.5",
              "--steps", "8")
