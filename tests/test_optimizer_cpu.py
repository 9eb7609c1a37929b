"""Optimizer options (weight decay, Nesterov) and learning-rate schedules: the oracle against torch.optim, the
schedule table against torch.optim.lr_scheduler, configuration / CLI, every CPU backend against the simulator and
an exact checkpoint resume in the middle of a schedule."""
import math
import os
import subprocess
import sys

import pytest
import torch

from eventgrad_b200.config import PRESETS, TrainConfig, parse_cli, preset
from eventgrad_b200.data import synthetic_source
from eventgrad_b200.engine import lr_schedule
from eventgrad_b200.engine.lr_schedule import lr_at, lr_table
from eventgrad_b200.engine.trainer import Trainer
from eventgrad_b200.parallel.trigger import sgd_
from eventgrad_b200.utils.ckpt import ckpt_path
from eventgrad_b200.utils.dist import DistEnv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------- sgd_ oracle
@pytest.mark.parametrize("wd,nesterov,mu", [(wd, n, mu) for wd in (0.0, 5e-4) for mu in (0.0, 0.9)
                                            for n in (False, True) if not (n and mu == 0.0)])
def test_sgd_oracle_equals_torch_optim_sgd(wd, nesterov, mu):
    g = torch.Generator().manual_seed(3)
    n = 10007                                    # not a multiple of any vector width: tails are covered too
    p = torch.nn.Parameter(torch.randn(n, generator=g))
    theta, mom = p.detach().clone(), torch.zeros(n)
    opt = torch.optim.SGD([p], lr=0.1, momentum=mu, weight_decay=wd, nesterov=nesterov, foreach=False)
    if mu != 0.0:
        opt.state[p]["momentum_buffer"] = torch.zeros(n)          # the arena's zero-initialised momentum
    for k, lr in enumerate((0.1, 0.05, 0.05, 0.0125, 3e-3)):
        grad = torch.randn(n, generator=g) * 0.3
        for grp in opt.param_groups:
            grp["lr"] = lr
        p.grad = grad.clone()
        opt.step()
        before = grad.clone()
        sgd_(theta, grad, mom, lr, mu, wd, nesterov)
        assert torch.equal(grad, before), "sgd_ modified its grad argument"
        assert torch.equal(theta, p.detach()), f"step {k}"
        if mu != 0.0:
            assert torch.equal(mom, opt.state[p]["momentum_buffer"])


def test_sgd_oracle_defaults_are_plain_heavy_ball():
    g = torch.Generator().manual_seed(1)
    th, gr = torch.randn(4096, generator=g), torch.randn(4096, generator=g)
    a, ma = th.clone(), torch.zeros(4096)
    sgd_(a, gr, ma, 0.01, 0.9)
    m = torch.zeros(4096).mul_(0.9).add_(gr)
    assert torch.equal(a, th.clone().add_(m, alpha=-0.01))


# ---------------------------------------------------------------------------------------- schedule table
def _torch_epoch_lrs(cfg, make):
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=cfg.lr)
    sch = make(opt)
    out = []
    for _ in range(cfg.epochs):
        out.append(sch.get_last_lr()[0])
        opt.step()
        sch.step()
    return out


@pytest.mark.parametrize("kind", ["constant", "step", "multistep", "cosine"])
def test_lr_table_matches_torch_schedulers(kind):
    from torch.optim import lr_scheduler as S
    cfg = TrainConfig(lr=0.1, epochs=17, lr_schedule=kind, lr_step_epochs=4, lr_milestones=(3, 8, 11),
                      lr_gamma=0.2, lr_min=1e-3)
    make = {"constant": lambda o: S.LambdaLR(o, lambda e: 1.0),
            "step": lambda o: S.StepLR(o, step_size=4, gamma=0.2),
            "multistep": lambda o: S.MultiStepLR(o, milestones=[3, 8, 11], gamma=0.2),
            "cosine": lambda o: S.CosineAnnealingLR(o, T_max=17, eta_min=1e-3)}[kind]
    ref = _torch_epoch_lrs(cfg, make)
    spe = 5
    tab = lr_table(cfg, spe)
    assert tab.dtype == torch.float32 and tab.numel() == cfg.epochs * spe
    for e in range(cfg.epochs):
        exact = lr_schedule.epoch_lr(cfg, e)
        assert math.isclose(exact, ref[e], rel_tol=1e-12), (e, exact, ref[e])
        for j in range(spe):
            assert float(tab[e * spe + j]) == float(torch.tensor(exact, dtype=torch.float64).float())
    # clamping: steps past the end keep the last value
    n = tab.numel()
    assert lr_at(tab, n, 0.0) == lr_at(tab, n + 1, 0.0) == lr_at(tab, 10 * n, 0.0) == float(tab[-1])
    assert lr_at(tab, 1, 0.0) == float(tab[0]) and lr_at(None, 7, 0.25) == 0.25


def test_lr_table_warmup_matches_linear_lr_per_step():
    from torch.optim import lr_scheduler as S
    spe = 6
    cfg = TrainConfig(lr=0.4, epochs=5, lr_schedule="multistep", lr_milestones=(1, 3), lr_gamma=0.5,
                      lr_warmup_epochs=1.5)
    W = lr_schedule.warmup_steps(cfg, spe)
    assert W == 9
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=1.0)
    warm = S.LinearLR(opt, start_factor=1.0 / W, end_factor=1.0, total_iters=W - 1)
    tab = lr_table(cfg, spe)
    for i in range(cfg.epochs * spe):
        factor = warm.get_last_lr()[0]
        exact = lr_schedule.epoch_lr(cfg, i // spe) * factor
        assert math.isclose(float(tab[i]), exact, rel_tol=1e-7), (i, float(tab[i]), exact)
        opt.step()
        warm.step()
    assert float(tab[W]) == float(torch.tensor(0.2, dtype=torch.float64).float())      # epoch 1: after milestone 1
    assert lr_schedule.is_constant(TrainConfig()) and not lr_schedule.is_constant(TrainConfig(lr_warmup_epochs=1))


# ---------------------------------------------------------------------------------------- config / CLI
def test_config_validation_rejects_bad_optimizer_settings():
    with pytest.raises(ValueError):
        TrainConfig(weight_decay=-1e-4).validate()
    with pytest.raises(ValueError):
        TrainConfig(momentum=0.0, nesterov=True).validate()
    with pytest.raises(ValueError):
        TrainConfig(lr_schedule="multistep", lr_milestones=(5, 5)).validate()
    with pytest.raises(ValueError):
        TrainConfig(lr_schedule="multistep", lr_milestones=(8, 3)).validate()
    with pytest.raises(ValueError):
        TrainConfig(lr_schedule="plateau").validate()
    with pytest.raises(ValueError):
        TrainConfig(lr_schedule="step", lr_step_epochs=0).validate()
    with pytest.raises(ValueError):
        TrainConfig(lr_warmup_epochs=-1).validate()
    TrainConfig(weight_decay=5e-4, momentum=0.9, nesterov=True, lr_schedule="multistep",
                lr_milestones=(10, 15)).validate()


def test_cli_flags_parse_and_preset_defaults_are_unchanged():
    c = parse_cli("cifar_event", ["0", "1", "1.0", "--weight-decay", "5e-4", "--nesterov", "--lr-schedule",
                                  "multistep", "--lr-milestones", "10,15", "--lr-gamma", "0.2",
                                  "--lr-warmup-epochs", "0.5"])
    assert (c.weight_decay, c.nesterov, c.lr_schedule, c.lr_milestones, c.lr_gamma, c.lr_warmup_epochs) == \
        (5e-4, True, "multistep", (10, 15), 0.2, 0.5)
    assert (c.file_write, c.thres_type, c.horizon) == (0, 1, 1.0)          # positional arguments untouched
    c = parse_cli("cifar_spevent", ["0", "1", "1.0", "5", "--lr-schedule", "cosine", "--lr-min", "1e-4",
                                    "--lr-step-epochs", "7"])
    assert c.lr_schedule == "cosine" and c.lr_min == 1e-4 and c.lr_step_epochs == 7 and c.topk_percent == 5.0
    with pytest.raises(ValueError):
        parse_cli("mnist_event", ["0", "1", "1.0", "--nesterov"])           # the preset has momentum 0
    with pytest.raises(SystemExit):
        parse_cli("decent", ["0", "--lr-schedule", "plateau"])
    d = TrainConfig()
    for name in PRESETS:
        c = preset(name)
        assert (c.weight_decay, c.nesterov, c.lr_schedule, c.lr_warmup_epochs) == (0.0, False, "constant", 0.0)
        assert lr_schedule.is_constant(c)
        prog = {"cent": [], "decent": ["0"]}.get(name, ["0", "1", "1.0"])
        cli = parse_cli(name, prog)
        assert (cli.weight_decay, cli.nesterov, cli.lr_schedule, cli.lr_milestones) == \
            (d.weight_decay, d.nesterov, d.lr_schedule, d.lr_milestones)


# ---------------------------------------------------------------------------------------- gloo / refport
_PORT = [31900 + (os.getpid() % 50) * 10]


def _torchrun(world, *args, backend="gloo"):
    _PORT[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(_PORT[0]),
           os.path.join(ROOT, "tests", "optimizer_worker.py"), "--backend", backend, *args]
    env = dict(os.environ, OMP_NUM_THREADS="1", EGB_WORKER_CPU="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("algo,world", [("cent", 2), ("decent", 3), ("event", 2), ("event", 3), ("spevent", 3)])
def test_gloo_backend_with_wd_nesterov_multistep_matches_simulator(algo, world):
    rc, out = _torchrun(world, "--algo", algo, "--steps", "10")
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


@pytest.mark.parametrize("algo", ["cent", "event"])
def test_refport_backend_with_wd_nesterov_multistep_matches_simulator(algo):
    rc, out = _torchrun(3 if algo == "event" else 2, "--algo", algo, "--steps", "8", backend="refport")
    assert rc == 0 and "WORKER_OK" in out, out[-2000:]


# ---------------------------------------------------------------------------------------- Trainer resume
def _trainer(tmp_path, **kw):
    base = dict(device="cpu", backend="gloo", model="cnn2", train_samples=256, test_samples=64, batch_size=64,
                epochs=3, quiet=True, momentum=0.9, weight_decay=5e-4, nesterov=True, lr_schedule="multistep",
                lr_milestones=(2,), lr_gamma=0.1, lr_warmup_epochs=0.5)
    base.update(kw)
    torch.manual_seed(0)
    cfg = preset("mnist_event", **base)
    return Trainer(cfg, DistEnv(0, 1, 0, torch.device("cpu"), "none"),
                   train_source=synthetic_source("mnist", 256), test_source=synthetic_source("mnist", 64, train=False))


def test_cpu_trainer_resume_mid_schedule_is_exact(tmp_path):
    full = _trainer(tmp_path)
    assert full.backend.lr_table is not None and full.backend.lr_table.numel() == 3 * 4
    full.fit()
    part = _trainer(tmp_path, ckpt_dir=str(tmp_path), ckpt_every=1, max_steps=4)      # stops after epoch 1
    part.fit()
    assert part.epoch == 1 and part.backend.pass_num == 4
    res = _trainer(tmp_path, resume=ckpt_path(str(tmp_path), 0))
    assert res.epoch == 1 and res.backend.pass_num == 4
    res.fit()
    assert res.backend.pass_num == full.backend.pass_num == 12
    assert torch.equal(res.arena.theta, full.arena.theta)
    assert not torch.equal(part.arena.theta, full.arena.theta)
