"""GPU: weight decay, Nesterov momentum and a learning-rate schedule inside the fused step kernels
(csrc/gossip.cu, csrc/allreduce.cu), bit for bit against the simulator, through CUDA-graph replays and across a
checkpoint resume.  Multi-rank runs use R virtual ranks on one GPU (ops.local_world.LocalWorld)."""
import pytest
import torch

from eventgrad_b200.config import TrainConfig, preset
from eventgrad_b200.data import synthetic_source
from eventgrad_b200.engine.lr_schedule import lr_table
from eventgrad_b200.engine.simulator import RingSimulator
from eventgrad_b200.engine.trainer import Trainer
from eventgrad_b200.models import build_model
from eventgrad_b200.parallel.trigger import TriggerConfig
from eventgrad_b200.utils.dist import DistEnv

pytestmark = pytest.mark.gpu

SPE = 3          # steps per epoch of the test schedules: milestone at epoch 2 = step 7
OPT = dict(momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep", lr_milestones=(2,),
           lr_gamma=0.1, lr_warmup_epochs=1.0, epochs=4)


def _cfg(algo, **kw):
    base = dict(algo=algo, dataset="mnist", model="cnn2", lr=0.05, sync_mode="iter", horizon=1.0, thres_type=1,
                topk_percent=10.0, initial_comm_passes=4, **OPT)
    base.update(kw)
    return TrainConfig(**base).validate()


def _world(cfg, R, model="cnn2", grid_cap=6):
    from eventgrad_b200.ops.local_world import LocalWorld
    return LocalWorld(cfg, R, lambda: build_model(model), grid_cap=grid_cap, timeout_ns=5_000_000_000)


def _grads(w, R, seed):
    t = w.arenas[0].table
    m = torch.zeros(t.n_padded, device="cuda")
    for o, n in zip(t.offsets, t.numels):
        m[o:o + n] = 1
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(t.n_padded, generator=g, device="cuda") * 0.05 * m for _ in range(R)]


def _sim(cfg, w, R, table, **kw):
    return RingSimulator(R, w.arenas[0].theta.cpu(), w.arenas[0].table, cfg.algo, TriggerConfig.from_train(cfg),
                         lr=cfg.lr, momentum=cfg.momentum, topk_percent=cfg.topk_percent,
                         weight_decay=cfg.weight_decay, nesterov=cfg.nesterov, lr_table=table, **kw)


def _run_vs_sim(cfg, R, steps=10, two_shot=None, model="cnn2", grid_cap=6):
    w = _world(cfg, R, model=model, grid_cap=grid_cap)
    table = lr_table(cfg, SPE)
    for be in w.backends:
        be.set_lr_table(table)
        if two_shot is not None:
            be.ap.update({"two_shot": int(two_shot)})
    sim = _sim(cfg, w, R, table, serial_skip=False)
    for s in range(steps):
        fires = [be.fire.clone().bool() for be in w.backends] if cfg.algo in ("event", "spevent") else None
        g = _grads(w, R, 40 + s)
        w.step(g)
        sim.step([x.cpu() for x in g], fires=fires)
    torch.cuda.synchronize()
    for r, be in enumerate(w.backends):
        be.check_status()
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r]), f"rank {r} theta differs"
        assert torch.equal(w.arenas[r].mom.cpu(), sim.mom[r]), f"rank {r} momentum differs"
        assert int(be.d_pass.item()) == steps        # the device step index that selects the lr
    w.close()


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("variant", ["dbuf", "single", "split"])
def test_decent_variants_bitwise_vs_simulator(variant, R):
    kw = {"dbuf": dict(), "single": dict(double_buffer=False), "split": dict(overlap_push=True)}[variant]
    _run_vs_sim(_cfg("decent", **kw), R)


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("algo", ["event", "spevent"])
def test_event_and_spevent_bitwise_vs_simulator(algo, R):
    _run_vs_sim(_cfg(algo), R)


def test_cent_serial_plain_sgd_bitwise_vs_simulator():
    _run_vs_sim(_cfg("cent", model="mlp"), 1, model="mlp")


@pytest.mark.parametrize("R", [2, 4])
@pytest.mark.parametrize("two_shot", [0, 1])
def test_cent_allreduce_sgd_bitwise_vs_simulator(R, two_shot):
    _run_vs_sim(_cfg("cent", model="mlp"), R, two_shot=two_shot, model="mlp", grid_cap=16)


def test_default_options_pass_no_table_and_keep_the_scalar_lr():
    w = _world(_cfg("decent", momentum=0.9, weight_decay=0.0, nesterov=False, lr_schedule="constant",
                    lr_warmup_epochs=0.0), 2)
    sim = RingSimulator(2, w.arenas[0].theta.cpu(), w.arenas[0].table, "decent", lr=0.05, momentum=0.9,
                        serial_skip=False)
    for s in range(5):
        g = _grads(w, 2, 70 + s)
        w.step(g)
        sim.step([x.cpu() for x in g])
    torch.cuda.synchronize()
    for r in range(2):
        assert w.backends[r].d_lr is None
        assert torch.equal(w.arenas[r].theta.cpu(), sim.theta[r])
    w.close()


def test_grad_pointer_table_mode_bitwise_vs_simulator():
    """Table mode: the step kernel reads autograd's own (fp32) gradient tensors in place."""
    from eventgrad_b200.parallel import ParamArena, Ring
    from eventgrad_b200.parallel.p2p import P2PBackend, preallocate_arena_buffers
    cfg = _cfg("event")
    env = _env()
    torch.manual_seed(0)
    model = build_model("cnn2")
    theta, grad, symm = preallocate_arena_buffers(model, cfg, env)
    arena = ParamArena(model, env.device, theta=theta, grad=grad)
    arena.enable_table_mode(shadow=False)
    be = P2PBackend(cfg, arena, Ring(0, 1), env, symm=symm, grid_cap=6, timeout_ns=5_000_000_000)
    assert be.table_mode
    table = lr_table(cfg, SPE)
    be.set_lr_table(table)
    t = arena.table
    sim = RingSimulator(1, arena.theta.cpu(), t, "event", TriggerConfig.from_train(cfg), lr=cfg.lr,
                        momentum=cfg.momentum, serial_skip=False, weight_decay=cfg.weight_decay,
                        nesterov=cfg.nesterov, lr_table=table)
    gen = torch.Generator(device="cuda").manual_seed(9)
    for s in range(9):
        fires = [be.fire.clone().bool()]
        flat = torch.zeros(t.n_padded, device="cuda")
        for i, c in enumerate(arena.compute):
            c.grad = torch.randn(c.shape, generator=gen, device="cuda") * 0.05
            arena.flat(flat, i).copy_(c.grad.reshape(-1))
        be.update_grad_table(arena.compute)
        be.launch()
        be.account_step()
        sim.step([flat.cpu()], fires=fires)
    torch.cuda.synchronize()
    be.check_status()
    assert torch.equal(arena.theta.cpu(), sim.theta[0])
    be.close()


# ---------------------------------------------------------------------------------------- Trainer
def _env():
    return DistEnv(0, 1, 0, torch.device("cuda", 0), "none")


def _trainer(name, **kw):
    base = dict(backend="p2p", device="cuda", train_samples=256, test_samples=64, batch_size=64,
                batch_mode="per_rank", quiet=True, momentum=0.9, weight_decay=5e-4, nesterov=True)
    base.update(kw)
    torch.manual_seed(0)
    return Trainer(preset(name, **base), _env(), train_source=synthetic_source("mnist", 256).pin(),
                   test_source=synthetic_source("mnist", 64, train=False).pin())


def _steps(tr):
    """Run the whole schedule step by step; theta after every step."""
    snaps = []
    for ep in range(tr.cfg.epochs):
        tr.sampler.set_epoch(ep)
        for x, y in tr.loader:
            tr.train_step(x, y)
            snaps.append(tr.arena.theta.clone())
    torch.cuda.synchronize()
    tr.backend.check_status()
    return snaps


def test_cuda_graph_replays_follow_the_schedule():
    """Serial cent (MLP, cuBLAS fp32): gamma = 0 at the milestone of epoch 2 (step 9), long after the graph was
    captured (step 4).  theta must stop changing exactly there -- the replays read the device table -- and equal the
    eager run bit for bit at every step."""
    sched = dict(epochs=3, lr_schedule="multistep", lr_milestones=(2,), lr_gamma=0.0)
    g = _trainer("cent", cuda_graph=True, **sched)
    e = _trainer("cent", cuda_graph=False, **sched)
    sg, se = _steps(g), _steps(e)
    assert len(g._graphs) == 1 and not e._graphs
    assert len(sg) == 12 and int(g.backend.d_pass.item()) == 12
    assert not torch.equal(sg[7], sg[6])                        # step 8 (lr > 0) still moves theta
    for k in range(8, 12):
        assert torch.equal(sg[k], sg[7]), f"theta changed at step {k + 1} although lr = 0"
    for k in range(12):
        assert torch.equal(sg[k], se[k]), f"graph and eager differ after step {k + 1}"
    g.close(); e.close()


def test_p2p_trainer_resumes_mid_schedule(tmp_path):
    """decent self-loop (MNIST semantics, 1 GPU): checkpoint after epoch 1, resume, cross the milestone of epoch 2;
    the device pass counter restored from the checkpoint puts the kernels back at the right table entry."""
    from eventgrad_b200.utils.ckpt import ckpt_path
    sched = dict(epochs=3, lr_schedule="multistep", lr_milestones=(2,), lr_gamma=0.1, lr_warmup_epochs=0.5)
    full = _trainer("decent", **sched)
    full.fit()
    th_full = full.arena.theta.clone()
    full.close()
    part = _trainer("decent", ckpt_dir=str(tmp_path), ckpt_every=1, max_steps=4, **sched)
    part.fit()
    assert part.epoch == 1 and int(part.backend.d_pass.item()) == 4
    part.close()
    res = _trainer("decent", resume=ckpt_path(str(tmp_path), 0), **sched)
    assert res.epoch == 1 and int(res.backend.d_pass.item()) == 4
    res.fit()
    res.backend.check_status()
    assert int(res.backend.d_pass.item()) == 12
    assert torch.equal(res.arena.theta, th_full)
    res.close()
