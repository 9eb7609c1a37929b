"""Training driver shared by the five reference-equivalent programs.

Reference structure being reproduced (one flat main() per program, SURVEY.md section 3):
  epoch loop -> batch loop -> zero_grad / forward / loss / backward
             -> [communication + consensus average]  -> optimizer.step -> accuracy count
  then: training time, per-rank event count, final model all-reduce average, total events,
  rank-0 evaluation of the averaged model
  (/root/reference/dcifar10/event/event.cpp:245-573, /root/reference/dmnist/cent/cent.cpp:100-214).

What is different by design:
  * everything after backward() is ONE backend call (fused kernel on the p2p backend);
  * no host synchronisation inside the step: accuracy / loss / event counters live on the
    device and are read at epoch boundaries (the reference does 1+3*sz `.item()` per step);
  * forward+backward (and the fused comm kernel) can be replayed from a CUDA graph.
"""
from __future__ import annotations

import os
import time
from typing import Optional

import torch
import torch.nn.functional as F

from ..config import TrainConfig
from ..data import BatchLoader, ShardSampler, eval_batches, load_source, per_rank_batch
from ..models import build_model
from ..parallel import Graph, ParamArena, Ring, make_backend
from ..parallel.trigger import consensus_values
from ..utils.ckpt import ckpt_path, load_checkpoint, save_checkpoint
from ..utils.dist import DistEnv, barrier
from ..utils.logfiles import RefLogWriter
from ..utils.timers import PhaseTimer
from . import lr_schedule


def _compute_dtype(cfg: TrainConfig):
    return torch.bfloat16 if cfg.dtype == "bf16" else torch.float32


class Trainer:
    def __init__(self, cfg: TrainConfig, env: DistEnv, group=None, train_source=None,
                 test_source=None):
        cfg = cfg.validate().resolved(env.device.type, env.world)
        self.cfg, self.env = cfg, env
        graph = Graph.build(env.rank, env.world, cfg.topology, seed=cfg.topology_seed)    # ValueError: offsets out of range for this world
        self.ring = Ring(env.rank, env.world) if graph.is_ring else graph
        dev = env.device
        self.device = dev
        if dev.type == "cuda":
            # fp32 means fp32: the reference computes in IEEE fp32 on the CPU (event.cpp:279), so TF32 is only used
            # when asked for (cuDNN's allow_tf32 defaults to True in PyTorch)
            tf32 = cfg.dtype == "tf32"
            torch.backends.cuda.matmul.allow_tf32 = tf32
            torch.backends.cudnn.allow_tf32 = tf32
            from ..ops import conv_tc as _conv_tc
            _conv_tc.set_enabled(bool(cfg.conv_tc))       # fp32: eligible 3x3 convs on wgmma at fp32 accuracy
        if dev.type == "cuda":
            torch.backends.cudnn.benchmark = bool(cfg.cudnn_benchmark)
            if cfg.host_threads > 0:
                # The host side of a GPU step is a 0.8 MB gather + a few launches.  A 64-thread OpenMP
                # pool for that costs milliseconds per step (wake-ups contending with the thread that
                # polls CUDA events; benchmarks/e2e_probe.py isolates it).
                torch.set_num_threads(cfg.host_threads)
        # identical initial weights on every rank: torch::manual_seed(0) (event.cpp:115)
        torch.manual_seed(cfg.seed)
        self.model = build_model(cfg.model, resnet_variant=cfg.resnet_variant)
        extra = None
        if cfg.algo == "spevent" and cfg.spevent_fresh_replicas:
            # quirk Q8: prev_model, left_model, right_model are constructed right after the model, in this
            # order, from the same RNG stream (spevent.cpp:123-136)
            extra = [build_model(cfg.model, resnet_variant=cfg.resnet_variant) for _ in range(3)]
        want_p2p = cfg.backend == "p2p" or (cfg.backend == "auto" and dev.type == "cuda")
        theta_buf = grad_buf = None
        self._symm = None
        if want_p2p:
            from ..parallel.p2p import preallocate_arena_buffers
            theta_buf, grad_buf, self._symm = preallocate_arena_buffers(self.model, cfg, env, group)
        self.arena = ParamArena(self.model, dev, theta=theta_buf, grad=grad_buf,
                                with_momentum=True, channels_last=cfg.channels_last and dev.type == "cuda")
        if want_p2p and cfg.grad_table and cfg.algo != "cent":
            self.arena.enable_table_mode(shadow=(cfg.dtype == "bf16"))
        if cfg.channels_last and dev.type == "cuda":
            pass  # activations are produced NHWC by the loader; conv weights already NHWC views
        self.backend = make_backend(cfg, self.arena, self.ring, env, group) if not want_p2p else \
            self._make_p2p(group)
        if extra is not None:
            self.backend.set_sparse_init(*[self.arena.pack(m) for m in extra])
            del extra
        # ---- data ------------------------------------------------------------------
        self.train_src = train_source or load_source(cfg.dataset, cfg.data, cfg.train_samples, True)
        self.test_src = test_source
        mode = cfg.sampler
        self.sampler = ShardSampler(len(self.train_src), env.world, env.rank, mode, seed=cfg.seed,
                                    partition=cfg.partition, labels=self.train_src.labels)
        self.batch = per_rank_batch(cfg, env.world, self.sampler.local_size)
        self.loader = BatchLoader(self.train_src, self.sampler, self.batch, dev,
                                  augment=cfg.augment and cfg.dataset == "cifar10",
                                  out_dtype=torch.float32, channels_last=cfg.channels_last,
                                  seed=cfg.seed, native=cfg.native_loader)
        if not lr_schedule.is_constant(cfg):
            # one lr per step of the run, indexed by the backend's (device) pass counter -- also after a resume
            self.backend.set_lr_table(lr_schedule.lr_table(cfg, len(self.loader)))
        if cfg.consensus_every:
            # the measurements are drained at every epoch boundary: room for one epoch's worth
            self.backend.set_consensus_capacity(len(self.loader) // cfg.consensus_every + 1)
        self.consensus_last = None                # (step, distance, relative) of the latest measurement
        self.logw = RefLogWriter(cfg.log_dir, env.rank, cfg.algo, cfg.dataset, bool(cfg.file_write))
        self.timer = PhaseTimer(dev, enabled=bool(cfg.phase_timers))
        self.correct = torch.zeros((), dtype=torch.int64, device=dev)
        self.loss_sum = torch.zeros((), dtype=torch.float32, device=dev)
        self.last_loss: Optional[torch.Tensor] = None
        self.epoch = 0
        self.steps_done = 0
        self._graphs = {}
        self._graph_launches = {}                 # graph key -> kernels of OUR extension captured in that graph
        self.own_launches_per_step = {}           # family -> kernels of our extension in the most recent step
        self.own_launches_total = 0               # ... summed over every step executed so far (replays included)
        self._graph_warm = {}
        self._side = None
        self._capture_stream = None
        self._graph_keepalive = []
        self.train_time_s = 0.0
        if cfg.resume:
            sd = load_checkpoint(cfg.resume, arena=self.arena, backend=self.backend, model=self.model,
                                 loader=self.loader)
            self.epoch = int(sd["epoch"])
            self.steps_done = int(sd.get("steps_done", 0))
        if env.rank == 0 and not cfg.quiet:
            t = self.arena.table
            print(f"Number of parameters - {t.n_tensors}", flush=True)       # event.cpp:127-130
            print(f"Number of elements - {t.n_elems}", flush=True)
            if cfg.algo == "spevent":
                print(f"Number of topk elements - {sum(t.topk_counts(cfg.topk_percent))}", flush=True)

    def _make_p2p(self, group):
        from ..parallel.p2p import P2PBackend
        return P2PBackend(self.cfg, self.arena, self.ring, self.env, group, symm=self._symm)

    # ------------------------------------------------------------------ one step
    def _autocast(self):
        if self.cfg.dtype == "bf16":
            return torch.autocast(self.device.type, dtype=torch.bfloat16)
        return torch.autocast(self.device.type, enabled=False)

    def _fwd_bwd(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        with self._autocast():
            out = self.model(x)
        loss = F.cross_entropy(out.float(), y)     # == nll_loss(log_softmax(.)) (event.cpp:268,:291)
        if self.arena.table_mode:
            self.arena.clear_compute_grads()       # fresh gradient tensors, consumed in place by the step kernel
        loss.backward()
        with torch.no_grad():
            self.correct += (out.argmax(1) == y).sum()
        return loss.detach()

    GRAPH_WARMUP_STEPS = 3

    def _own_counts(self):
        """Per-family count of kernels enqueued so far by OUR extension (csrc/api.h eg_count_launch)."""
        if self.device.type != "cuda":
            return None
        from ..ops import ext
        return dict(ext().launch_counts())

    def _fwd_bwd_launch(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """forward/backward + the backend's kernels, with the theta_k-only half of a split step
        (neighbour pushes / top-k records) forked onto a side stream so that its NVLink traffic is
        hidden behind the compute.  Pure enqueue: usable eagerly and under graph capture."""
        be = self.backend
        if getattr(be, "overlap", False):
            cur = torch.cuda.current_stream(self.device)
            if self._side is None:
                self._side = torch.cuda.Stream(self.device)
            self._side.wait_stream(cur)
            with torch.cuda.stream(self._side):
                be.launch_pre()
            loss = self._fwd_bwd(x, y)
            cur.wait_stream(self._side)
        else:
            loss = self._fwd_bwd(x, y)
        if self.arena.table_mode:
            keep = be.update_grad_table(self.arena.compute, persistent=torch.cuda.is_current_stream_capturing())
            if torch.cuda.is_current_stream_capturing():
                self._graph_keepalive.append(keep)
        be.launch()
        return loss

    def _eager_step(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        if getattr(self.backend, "graph_safe", False):
            with self.timer.phase("step(fwd+bwd+fused_update)"):
                loss = self._fwd_bwd_launch(x, y)
            self.backend.account_step()
        else:
            with self.timer.phase("fwd_bwd"):
                loss = self._fwd_bwd(x, y)
            with self.timer.phase("comm_update"):
                self.backend.step()
        return loss

    def _graphed_step(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """Replay the step from a CUDA graph (per input shape).  The first GRAPH_WARMUP_STEPS steps
        of a shape run eagerly (cuDNN autotune, lazy kernel loading, allocator warm-up); then the
        step is captured once.  With a graph-safe backend (p2p) the capture holds the WHOLE step --
        forward, backward and the fused exchange/average/SGD kernel, which spins on its neighbours'
        flags from inside the graph; otherwise only forward+backward are captured."""
        key = tuple(x.shape)
        ent = self._graphs.get(key)
        whole = bool(getattr(self.backend, "graph_safe", False))
        if ent is None:
            n = self._graph_warm.get(key, 0)
            if n < self.GRAPH_WARMUP_STEPS:
                self._graph_warm[key] = n + 1
                return self._eager_step(x, y)
            sx, sy = x.clone(), y.clone()
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            before = self._own_counts()
            # captured at a higher priority than the default streams': every kernel node of the step outranks the
            # weight gradients, which conv_tc launches at the lowest priority on a side stream
            if self._capture_stream is None:
                self._capture_stream = torch.cuda.Stream(self.device, priority=-1)
            with torch.cuda.graph(g, stream=self._capture_stream):
                if whole:
                    sloss = self._fwd_bwd_launch(sx, sy)
                else:
                    sloss = self._fwd_bwd(sx, sy)
            after = self._own_counts()
            self._graph_launches[key] = {k: after[k] - before.get(k, 0) for k in after}
            ent = (g, sx, sy, sloss)
            self._graphs[key] = ent
        g, sx, sy, sloss = ent
        sx.copy_(x)
        sy.copy_(y)
        g.replay()
        self._replayed = self._graph_launches[key]
        if whole:
            self.backend.account_step()
        else:
            self.backend.step()
        return sloss

    def train_step(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """zero_grad -> forward -> loss -> backward -> [comm + average + SGD]."""
        if not getattr(self.backend, "zeroes_grad", False):
            self.arena.zero_grad()
        before = self._own_counts()
        self._replayed = None
        if self.cfg.cuda_graph and self.device.type == "cuda":
            loss = self._graphed_step(x, y)
        else:
            loss = self._eager_step(x, y)
        if before is not None:
            after = self._own_counts()
            step = {k: after[k] - before.get(k, 0) for k in after}      # launched eagerly by this call ...
            for k, v in (self._replayed or {}).items():                 # ... plus what the replayed graph holds
                step[k] = step.get(k, 0) + v
            self.own_launches_per_step = step
            self.own_launches_total += sum(step.values())
        self.steps_done += 1
        self.last_loss = loss
        return loss

    # ------------------------------------------------------------------ epochs
    def fit(self) -> None:
        cfg, env = self.cfg, self.env
        barrier(env)
        t0 = time.perf_counter()
        stop = False
        while self.epoch < cfg.epochs and not stop:
            self.epoch += 1
            self.model.train()
            self.correct.zero_()
            self.sampler.set_epoch(self.epoch - 1)
            ep_losses = []
            for x, y in self.loader:
                loss = self.train_step(x, y)
                if cfg.file_write:
                    ep_losses.append((self.backend.pass_num, loss.clone()))
                if cfg.max_steps and self.steps_done >= cfg.max_steps:
                    stop = True
                    break
            # ---- epoch boundary: the only host syncs of the training loop ----------------
            acc = 100.0 * float(self.correct.item()) / max(1, self.sampler.local_size)
            self._check_device_status()
            if not cfg.quiet:
                if cfg.dataset == "mnist":
                    print(f"{self.epoch}, {acc:g}", flush=True)                       # event.cpp:498
                else:
                    print(f"Accuracy in epoch {self.epoch} - {acc:g}", flush=True)     # event.cpp:489
            self.last_train_acc = acc
            if cfg.consensus_every:
                self._drain_consensus()
            if cfg.file_write:
                self.logw.write_steps(self.backend.drain_logs())
                for pn, l in ep_losses:
                    self.logw.write_train(pn, float(l))
                if ep_losses:
                    self.logw.write_value(self.epoch, float(ep_losses[-1][1]))
            if cfg.ckpt_dir and cfg.ckpt_every and self.epoch % cfg.ckpt_every == 0:
                save_checkpoint(ckpt_path(cfg.ckpt_dir, env.rank), epoch=self.epoch, arena=self.arena,
                                backend=self.backend, model=self.model, loader=self.loader,
                                steps_done=self.steps_done)
                barrier(env)       # a slow writer must not leave its neighbours spinning against the device timeout
        self.backend.synchronize()
        self.train_time_s = time.perf_counter() - t0
        if env.rank == 0 and not cfg.quiet:
            print(f"Training time - {self.train_time_s:g}", flush=True)               # event.cpp:495-497
        if cfg.phase_timers:
            ms = self.timer.summary_ms()
            if env.rank == 0 and not cfg.quiet:
                print("phase timers (ms/call): " + ", ".join(f"{k}={v:.3f}" for k, v in ms.items()), flush=True)
            self.phase_ms = ms

    def _drain_consensus(self) -> None:
        """Epoch boundary under --consensus-every: take the epoch's measurements from the backend, print the latest
        relative distance (rank 0) and append them to consensus.csv / consensus_tensors.csv in --log-dir (rank 0;
        every rank holds the same values)."""
        rows = self.backend.drain_consensus()
        if not rows:
            return
        R, names = self.env.world, self.arena.table.names
        vals = [(k, *consensus_values(D, A, R)) for k, D, A in rows]
        self.consensus_last = vals[-1]
        if self.env.rank != 0:
            return
        if not self.cfg.quiet:
            print(f"Consensus distance in epoch {self.epoch} - {vals[-1][2]:g}", flush=True)
        os.makedirs(self.cfg.log_dir, exist_ok=True)
        for fname, header, lines in (
                ("consensus.csv", "step,distance,relative", [f"{k},{d!r},{r!r}" for k, d, r in vals]),
                ("consensus_tensors.csv", "step,tensor,sq_dist,sq_norm_mean",
                 [f"{k},{names[i]},{float(D[i])!r},{float(A[i])!r}" for k, D, A in rows for i in range(len(names))])):
            path = os.path.join(self.cfg.log_dir, fname)
            if not self._consensus_files_open:
                # a fresh run starts the files; a resumed one appends to what the run before it wrote
                if not self.cfg.resume or not os.path.exists(path):
                    with open(path, "w") as f:
                        f.write(header + "\n")
            with open(path, "a") as f:
                f.write("".join(line + "\n" for line in lines))
        self._consensus_files_open = True

    _consensus_files_open = False

    def _check_device_status(self) -> None:
        """Raise if a device-side wait timed out (sticky status words of the fused kernels): a wedged
        or dead peer shows up here as an exception instead of a hang (the reference would block
        forever in MPI_Recv / silently average a frozen copy -- SURVEY.md section 5)."""
        if hasattr(self.backend, "check_status"):
            self.backend.check_status()
        if self.device.type == "cuda":
            from ..ops.bn_act import bn_status
            st = bn_status(self.device)
            if st != 0:
                raise RuntimeError(f"fused BN kernels: device status {st} (flag wait timed out)")

    def finalize(self, evaluate: bool = True) -> dict:
        """Event statistics, final model averaging, rank-0 test (event.cpp:499-573)."""
        cfg, env = self.cfg, self.env
        res = {"rank": env.rank, "train_time_s": self.train_time_s, "steps": self.steps_done}
        gossip = cfg.algo in ("event", "spevent")
        if gossip and not cfg.quiet:
            print(f"No of events in rank {env.rank} - {self.backend.num_events()}", flush=True)
        res["events_rank"] = self.backend.num_events()
        res["bytes_sent_rank"] = self.backend.bytes_sent()
        if cfg.consensus_every:
            res["consensus_last"] = None if self.consensus_last is None else self.consensus_last[2]
        if cfg.algo != "cent":
            if cfg.consensus_every:
                # one more, ungated measurement of the models the final average is about to merge
                barrier(env)
                D, A = self.backend.measure_consensus()
                res["consensus_before_final_average"] = consensus_values(D, A, env.world)[1]
            # ranks may be skewed here (async mode has no per-step handshake; a slow checkpoint write or autotune on
            # one rank): meet on the host first so nobody spins in the all-reduce kernel against its device timeout
            barrier(env)
            self.backend.final_average()
        res["events_total"] = self.backend.total_events() if gossip else 0
        if gossip and env.rank == 0 and not cfg.quiet:
            print(f"Total number of events - {res['events_total']}", flush=True)
        dense = self.ring.fanout * self.arena.table.n_tensors * self.backend.pass_num * env.world
        dense *= cfg.gossip_rounds if env.world > 1 else 1      # --gossip-rounds: every round sends every tensor
        res["dense_messages"] = dense
        res["messages_saved"] = (1.0 - res["events_total"] / dense) if (gossip and dense) else 0.0
        if evaluate and env.rank == 0:
            res.update(self.evaluate())
        self.logw.close()
        return res

    @torch.no_grad()
    def evaluate(self) -> dict:
        cfg = self.cfg
        src = self.test_src or load_source(cfg.dataset, cfg.data, cfg.test_samples, False)
        self.model.eval()
        # MNIST: the whole test set as one batch (dmnist/event/event.cpp:542-546); CIFAR: 100
        bs = len(src) if cfg.dataset == "mnist" else cfg.test_batch_size
        correct, loss_sum, n = 0, 0.0, 0
        for x, y in eval_batches(src, bs, self.device, channels_last=cfg.channels_last):
            with self._autocast():
                out = self.model(x)
            loss_sum += float(F.cross_entropy(out.float(), y, reduction="sum"))
            correct += int((out.argmax(1) == y).sum())
            n += y.numel()
        acc = 100.0 * correct / max(1, n)
        if not cfg.quiet:
            if cfg.dataset == "mnist":
                print(f"Test loss - {loss_sum / max(1, n):g} ", flush=True)
            print(f"Num correct - {correct}", flush=True)
            print(f"Test Accuracy - {acc:g}", flush=True)
        self.model.train()
        return {"test_correct": correct, "test_acc": acc, "test_loss": loss_sum / max(1, n)}

    def close(self) -> None:
        self.backend.close()
