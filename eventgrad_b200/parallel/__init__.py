from .topology import Graph, Ring, parse_topology  # noqa
from .arena import ParamArena, TensorTable, TILE  # noqa
from .trigger import TriggerConfig, TriggerState, trigger_step, mix2_, mix3_, mixk_, sgd_, topk_select  # noqa
from .base import CommBackend, StepLog  # noqa


def make_backend(cfg, arena, ring, env, group=None):
    """backend=auto: fused P2P kernels on CUDA, gloo collectives on CPU."""
    name = cfg.backend
    if name == "auto":
        name = "p2p" if arena.theta.is_cuda else "gloo"
    if name == "p2p":
        from .p2p import P2PBackend
        return P2PBackend(cfg, arena, ring, env, group)
    if name == "refport":
        from .refstyle import ReferenceStyleBackend
        return ReferenceStyleBackend(cfg, arena, ring, group)
    from .collective import CollectiveBackend
    return CollectiveBackend(cfg, arena, ring, group)
