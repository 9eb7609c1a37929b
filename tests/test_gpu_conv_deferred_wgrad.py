"""The weight gradients of the tensor-core convolutions run on a side stream that the backward joins once, at its end,
when AccumulateGrad only steals dw (table mode); with a preset .grad it joins per layer.  Either way the step must
compute bit for bit what the serial reference path (EGB_CONV_PAR_BWD=0: every wgrad on the main stream) computes: a
missing record_stream or an early read of dw shows up here as a mismatch."""
import pytest
import torch

from eventgrad_b200.config import preset
from eventgrad_b200.data import synthetic_source
from eventgrad_b200.engine.trainer import Trainer
from eventgrad_b200.ops import conv_tc, ext
from eventgrad_b200.utils.dist import DistEnv

pytestmark = pytest.mark.gpu


def _run(monkeypatch, par, batch, table, graph):
    monkeypatch.setattr(conv_tc, "PAR_BWD", par)
    steps = Trainer.GRAPH_WARMUP_STEPS + 3 if graph else 3
    cfg = preset("cifar_event", backend="p2p", device="cuda", dtype="fp32", train_samples=2 * batch,
                 test_samples=128, batch_size=batch, epochs=100, quiet=True, max_steps=steps, augment=False,
                 grad_table=table, cuda_graph=graph)
    torch.manual_seed(0)
    tr = Trainer(cfg, DistEnv(0, 1, 0, torch.device("cuda", 0), "none"),
                 train_source=synthetic_source("cifar10", 2 * batch).pin(),
                 test_source=synthetic_source("cifar10", 128, train=False).pin())
    tr.fit()
    tr.backend.check_status()
    torch.cuda.synchronize()
    assert tr.arena.table_mode == table
    out = {"loss": tr.last_loss.clone(), "theta": tr.arena.theta.clone()}
    for n, p in tr.model.named_parameters():
        out["grad." + n] = p.grad.clone()
    tr.close()
    return out


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("table", [True, False], ids=["table", "preset_grad"])
@pytest.mark.parametrize("batch", [256, 32])
def test_side_stream_wgrad_is_bitwise_the_serial_path(monkeypatch, batch, table, graph):
    joins = []
    real = conv_tc._join_at_end
    monkeypatch.setattr(conv_tc, "_join_at_end", lambda cur, side: (joins.append(1), real(cur, side)))
    par = _run(monkeypatch, True, batch, table, graph)
    assert (len(joins) > 0) == table                   # deferred exactly when no .grad is preset
    ref = _run(monkeypatch, False, batch, table, graph)
    assert par.keys() == ref.keys()
    for k in ref:
        assert torch.equal(par[k], ref[k]), k


def test_accumulate_grad_steals_the_deferred_dw(monkeypatch):
    """Table mode: every conv weight's .grad is the very tensor its wgrad wrote (AccumulateGrad stole it, no copy
    kernel read it on the main stream before the end-of-backward join)."""
    written = set()
    real = conv_tc.wgrad

    def spy_wgrad(*a, **kw):
        dw = real(*a, **kw)
        written.add(dw.data_ptr())
        return dw
    monkeypatch.setattr(conv_tc, "wgrad", spy_wgrad)
    monkeypatch.setattr(conv_tc, "PAR_BWD", True)
    cfg = preset("cifar_event", backend="p2p", device="cuda", dtype="fp32", train_samples=64, test_samples=128,
                 batch_size=32, epochs=100, quiet=True, max_steps=1, augment=False, grad_table=True,
                 cuda_graph=False)
    torch.manual_seed(0)
    tr = Trainer(cfg, DistEnv(0, 1, 0, torch.device("cuda", 0), "none"),
                 train_source=synthetic_source("cifar10", 64).pin(),
                 test_source=synthetic_source("cifar10", 128, train=False).pin())
    tr.fit()
    torch.cuda.synchronize()
    convs = [p for p in tr.model.parameters() if p.dim() == 4 and p.shape[1] > 3]      # the stem's dw is a slice
    assert len(convs) > 10 and len(written) == len(convs) + 1
    assert {p.grad.data_ptr() for p in convs} < written
    tr.close()


def test_captured_graph_carries_the_wgrad_priority(monkeypatch):
    """The weight-gradient kernel nodes of the Trainer's captured step carry the lowest priority and the data-gradient /
    forward nodes a higher one: in the graph itself, not only in eager launches."""
    monkeypatch.setattr(conv_tc, "PAR_BWD", True)
    real_graph = torch.cuda.CUDAGraph
    monkeypatch.setattr(torch.cuda, "CUDAGraph", lambda: real_graph(keep_graph=True))
    cfg = preset("cifar_event", backend="p2p", device="cuda", dtype="fp32", train_samples=64, test_samples=128,
                 batch_size=32, epochs=100, quiet=True, max_steps=Trainer.GRAPH_WARMUP_STEPS + 1, augment=False,
                 grad_table=True, cuda_graph=True)
    torch.manual_seed(0)
    tr = Trainer(cfg, DistEnv(0, 1, 0, torch.device("cuda", 0), "none"),
                 train_source=synthetic_source("cifar10", 64).pin(),
                 test_source=synthetic_source("cifar10", 128, train=False).pin())
    tr.fit()
    torch.cuda.synchronize()
    (g, *_), = tr._graphs.values()
    nodes = ext().conv_graph_kernel_priorities(g.raw_cuda_graph())
    least, _ = torch.cuda.Stream.priority_range()
    wgrad = [p for k, p in nodes if k == 1]
    fprop = [p for k, p in nodes if k == 2]
    assert len(wgrad) > 10 and len(fprop) > 10
    assert all(p == least for p in wgrad), nodes
    assert all(p < least for p in fprop), nodes         # numerically lower = higher priority
    tr.close()
