#!/usr/bin/env python
"""Micro-benchmark of the fused exchange kernels on N GPUs (torchrun), device-timed, max over ranks.

For the ResNet arena (69.8 MB of parameters, 86 tensors) it reports per launch:
  * fused dense gossip step (push both neighbours + handshake + mix + SGD + norm-on-write):
    time, NVLink egress GB/s per GPU (2 x model bytes / time) against the 450 GB/s per direction of
    H100 NVLink 4 (data sheet), and HBM bytes/s of the mix+SGD stream;
  * fused event step at a chosen fire fraction (bytes scale with events);
  * fused all-reduce(+1/R+SGD) vs NCCL all_reduce + eager scale + eager SGD;
  * the NCCL-only gossip baseline (batch_isend_irecv + eager mix + eager SGD).
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from eventgrad_b200.config import TrainConfig  # noqa: E402
from eventgrad_b200.models import build_model  # noqa: E402
from eventgrad_b200.parallel import ParamArena, Ring  # noqa: E402
from eventgrad_b200.parallel.collective import CollectiveBackend  # noqa: E402
from eventgrad_b200.parallel.p2p import P2PBackend, preallocate_arena_buffers  # noqa: E402
from eventgrad_b200.utils.dist import barrier, init_distributed, max_over_ranks, shutdown  # noqa: E402


NVL = None          # NvlinkCounters of this rank's GPU (set in main)
NVLINK_GBPS = 450.0  # H100 SXM, NVLink 4, one direction (data sheet)
LAST_NVLINK = {}    # measured NVLink bytes per launch of the most recent timed() call (this rank)


def timed(fn, env, iters, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    # the NVML counter read takes tens of ms and differs per rank: do it BEFORE the barrier, or the ranks enter the
    # timed region skewed and the first launch of the fast ranks spins on the slow one
    c0 = NVL.read() if (NVL is not None and NVL.ok) else None
    barrier(env)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    barrier(env)                       # every rank's traffic has landed before anybody reads its counters
    c1 = NVL.read() if c0 is not None else None
    LAST_NVLINK.clear()
    if c0 is not None and c1 is not None:
        LAST_NVLINK.update({"nvlink_" + k + "_bytes_per_launch_measured": (c1[k] - c0[k]) / iters for k in c0})
    barrier(env)
    return max_over_ranks(e0.elapsed_time(e1), env) / iters


def make(cfg, env, model_name, **kw):
    torch.manual_seed(0)
    model = build_model(model_name)
    theta, grad, symm = preallocate_arena_buffers(model, cfg, env)
    arena = ParamArena(model, env.device, theta=theta, grad=grad)
    be = P2PBackend(cfg, arena, Ring(env.rank, env.world), env, symm=symm, **kw)
    return arena, be


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="resnet18")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    ap.add_argument("--skip-nccl", action="store_true")
    ap.add_argument("--only", default="", help="comma list of row-name prefixes to run (default: everything)")
    a = ap.parse_args()
    env = init_distributed("cuda")
    W = env.world
    global NVL
    from eventgrad_b200.utils.clocks import NvlinkCounters
    NVL = NvlinkCounters(env.device.index or 0)
    res = {"world": W, "model": a.model, "nvlink_counters": "NVML NVLINK_THROUGHPUT_{DATA,RAW}_{TX,RX}, rank 0's GPU" if NVL.ok else "unavailable"}
    base = dict(dataset="mnist", model=a.model, lr=1e-2, momentum=0.9)   # mnist => comm even at W=1 (self loop)
    only = [x for x in a.only.split(",") if x]
    want = lambda name: (not only) or any(name.startswith(o) for o in only)

    # ---- dense fused gossip (decent) -----------------------------------------------------------
    # "ack_*": single inbox slot + WAR ack (round-1 protocol); "dbuf": two slots, no ack (the default since round 2)
    for name, dbuf, kw in (("ack", False, dict()), ("ack_d1", False, dict(group_iters=1)), ("ack_d4", False, dict(group_iters=4)),
                           ("dbuf", None, dict()), ("dbuf_d4", None, dict(group_iters=4))):
        if not want(f"gossip_dense_{name}"):
            continue
        cfg = TrainConfig(algo="decent", sync_mode="iter", double_buffer=dbuf, **base).validate()
        arena, be = make(cfg, env, a.model, **kw)
        assert be.dbuf == (dbuf is None)
        n_bytes = arena.table.n_elems * 4
        ms = timed(be.step, env, a.iters)
        be.check_status()
        wire = (1 if be.wire_dedup else 2) * n_bytes          # 2-rank ring: theta crosses the link once
        res[f"gossip_dense_{name}"] = {"ms": ms, "egress_GBps_per_gpu": wire / ms / 1e6,
                                      "frac_of_nvlink": wire / ms / 1e6 / NVLINK_GBPS,
                                      "wire_bytes_per_gpu": wire,
                                      "hbm_GBps": 9 * arena.table.n_padded * 4 / ms / 1e6, "grid": be.grid, **LAST_NVLINK}
        be.close()
        del arena, be
        torch.cuda.empty_cache()

    # ---- push-only kernel (phase 1): the ceiling of SM-issued NVLink stores, vs grid size ----------
    if only and not want("push"):
        return finish(res, env, a)
    cfg = TrainConfig(algo="decent", sync_mode="iter", overlap_push=True, **base).validate()
    arena, be = make(cfg, env, a.model)
    n_bytes = arena.table.n_elems * 4
    for g in (32, 64, 128, 296, 592):
        def both():
            be.C.gossip_step_phase(be.gp, 1, g, be._stream())
            be.C.gossip_step_phase(be.gp, 2, be.grid, be._stream())
        ms_both = timed(both, env, a.iters)
        res[f"push_only_grid{g}"] = {"ms_push_plus_mix": ms_both}
    if True:
        def both_ce():                                   # copy engines instead of the SM push kernel
            be.C.ce_push(be.gp, be._stream())
            be.C.gossip_step_phase(be.gp, 2, be.grid, be._stream())
        res["push_copy_engine"] = {"ms_push_plus_mix": timed(both_ce, env, a.iters)}
    ms_mix = None
    be.check_status()
    be.close(); del arena, be; torch.cuda.empty_cache()

    # ---- async dense (no handshake) and event at ~0 fire fraction -------------------------------
    cfg = TrainConfig(algo="event", sync_mode="async", thres_type=0, constant=0.0, **base).validate()
    arena, be = make(cfg, env, a.model)
    n_bytes = arena.table.n_elems * 4
    ms = timed(be.step, env, a.iters)
    wire = (1 if be.wire_dedup else 2) * n_bytes
    res["event_async_allfire"] = {"ms": ms, "egress_GBps_per_gpu": wire / ms / 1e6, "frac_of_nvlink": wire / ms / 1e6 / NVLINK_GBPS,
                                  "wire_bytes_per_gpu": wire, **LAST_NVLINK}
    be.close(); del arena, be; torch.cuda.empty_cache()
    cfg = TrainConfig(algo="event", sync_mode="iter", thres_type=0, constant=1e30, initial_comm_passes=0,
                      **base).validate()
    arena, be = make(cfg, env, a.model)
    ms = timed(be.step, env, a.iters)
    res["event_sync_nofire"] = {"ms": ms, "hbm_GBps": 7 * arena.table.n_padded * 4 / ms / 1e6,
                                "events": be.num_events()}
    be.close(); del arena, be; torch.cuda.empty_cache()

    # ---- sparse 1% / 10% -----------------------------------------------------------------------
    for pct in (1.0, 10.0):
        cfg = TrainConfig(algo="spevent", sync_mode="iter", thres_type=0, constant=0.0, topk_percent=pct,
                          **base).validate()
        arena, be = make(cfg, env, a.model)
        def stp():
            arena.grad.normal_(0, 0.01)
            be.step()
        ms = timed(stp, env, max(10, a.iters // 3))
        nvl = dict(LAST_NVLINK)
        ms_g = timed(lambda: arena.grad.normal_(0, 0.01), env, 20)
        res[f"spevent_{pct:g}pct"] = {"ms": ms - ms_g, "K": be.K, "launches_per_step": 4, **nvl,
                                      "wire_bytes_per_gpu": (1 if be.wire_dedup else 2) * 2 * be.K * 4}
        be.check_status()
        be.close(); del arena, be; torch.cuda.empty_cache()

    # ---- fused all-reduce + SGD (cent) vs NCCL ------------------------------------------------
    for model in ("mlp", a.model):
        cfg = TrainConfig(algo="cent", **dict(base, model=model)).validate()
        arena, be = make(cfg, env, model)
        n_bytes = arena.table.n_elems * 4
        ms = timed(be.step, env, a.iters)
        be.check_status()
        entry = {"ms_fused": ms, "bytes": n_bytes, **LAST_NVLINK,
                 "busbw_GBps": (2 * (W - 1) / W) * n_bytes / ms / 1e6 if W > 1 else 0.0}
        if W > 1 and not a.skip_nccl:
            g = torch.zeros(arena.table.n_padded, device=env.device)
            th, mom = torch.zeros_like(g), torch.zeros_like(g)
            def nccl_step():
                dist.all_reduce(g)
                g.div_(W)
                mom.mul_(0.9).add_(g)
                th.add_(mom, alpha=-1e-2)
                g.zero_()
            entry["ms_nccl_eager"] = timed(nccl_step, env, a.iters)
        be.close(); del arena, be; torch.cuda.empty_cache()
        if W > 1 and model != "mlp":
            # NVLS: window in torch symmetric memory, in-switch reduction (multimem.ld_reduce) + multicast store
            os.environ["EGB_NVLS"] = "1"
            try:
                arena, be = make(cfg, env, model)
                if be.nvls_step:
                    entry["ms_fused_nvls"] = timed(be.step, env, a.iters)
                    be.check_status()
                    entry["busbw_GBps_nvls"] = (2 * (W - 1) / W) * n_bytes / entry["ms_fused_nvls"] / 1e6
                else:
                    entry["ms_fused_nvls"] = None
                be.close(); del arena, be; torch.cuda.empty_cache()
            except Exception as e:  # noqa: BLE001
                entry["nvls_error"] = repr(e)[:200]
            finally:
                os.environ["EGB_NVLS"] = "0"
        res[f"allreduce_sgd_{model}"] = entry

    # ---- NCCL-only gossip baseline -------------------------------------------------------------
    if W > 1 and not a.skip_nccl:
        cfg = TrainConfig(algo="decent", backend="nccl", **base).validate()
        torch.manual_seed(0)
        model = build_model(a.model)
        arena = ParamArena(model, env.device)
        be = CollectiveBackend(cfg, arena, Ring(env.rank, W))
        def st():
            arena.grad.zero_()
            be.step()
        res["gossip_dense_nccl_baseline"] = {"ms": timed(st, env, max(10, a.iters // 2))}

    finish(res, env, a)


def finish(res, env, a):
    if env.rank == 0:
        print(json.dumps(res, indent=1))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            json.dump(res, open(a.out, "w"), indent=1)
    shutdown()


if __name__ == "__main__":
    main()
