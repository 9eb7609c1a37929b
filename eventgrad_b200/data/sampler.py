"""Data sharding = the data-parallel split.

Mirrors LibTorch's distributed samplers as used by the reference (SURVEY.md C13):
  DistributedRandomSampler(size, R, rank, allow_duplicates=false)   cent / CIFAR programs
  DistributedSequentialSampler(size, R, rank, false)                decent / dmnist/event
Each rank owns floor(size/R) samples: the contiguous block [rank*local, (rank+1)*local) of
either the identity order (sequential) or a permutation seeded by the sampler epoch
(random).  The reference never calls set_epoch(), so the same order is replayed every epoch;
`reshuffle=True` opts into per-epoch reshuffling.  The partial last batch is kept
(DataLoader drop_last=false, SURVEY.md A.4).

partition="label" cuts heterogeneous shards instead (the setting of decentralized training on non-IID data): every rank
computes the same order p = randperm(size, seed), order = p[argsort(labels[p], stable)], and owns the block
order[rank*local, (rank+1)*local), so each rank sees one or a few classes and every shard still has floor(size/R)
samples (iter-sync ranks stay in lock-step).  `random` then permutes inside the shard, seeded as above; `sequential`
keeps the shard in class order.
"""
from __future__ import annotations

import torch


class ShardSampler:
    def __init__(self, size: int, world: int, rank: int, mode: str = "random",
                 seed: int = 0, reshuffle: bool = False, partition: str = "iid", labels=None):
        if mode not in ("random", "sequential"):
            raise ValueError("mode must be random|sequential")
        if partition not in ("iid", "label"):
            raise ValueError("partition must be iid|label")
        self.size, self.world, self.rank, self.mode = size, world, rank, mode
        self.seed, self.reshuffle = seed, reshuffle
        self.partition = partition
        self.local_size = size // world
        self.epoch = 0
        self._shard = None
        if partition == "label":
            if labels is None or len(labels) != size:
                raise ValueError("partition=label needs one label per sample")
            p = torch.randperm(size, generator=torch.Generator().manual_seed(seed))
            order = p[torch.argsort(torch.as_tensor(labels).cpu()[p], stable=True)]
            self._shard = order[rank * self.local_size:(rank + 1) * self.local_size].clone()

    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch

    def indices(self) -> torch.Tensor:
        if self._shard is not None:
            if self.mode == "sequential":
                return self._shard.clone()
            ep = self.epoch if self.reshuffle else 0
            g = torch.Generator().manual_seed(self.seed + ep)
            return self._shard[torch.randperm(self.local_size, generator=g)]
        b, e = self.rank * self.local_size, (self.rank + 1) * self.local_size
        if self.mode == "sequential":
            return torch.arange(b, e)
        ep = self.epoch if self.reshuffle else 0
        g = torch.Generator().manual_seed(self.seed + ep)
        return torch.randperm(self.size, generator=g)[b:e]

    def num_batches(self, batch: int) -> int:
        return -(-self.local_size // batch)


def per_rank_batch(cfg, world: int, local_size: int) -> int:
    """Batch size on one rank for the three batch modes of the reference programs:
    global/R (dcifar10/event/event.cpp:91), fixed per rank (dmnist/event/event.cpp:145),
    or the whole shard (dmnist/cent/cent.cpp:62-65)."""
    if cfg.batch_mode == "full":
        return local_size
    if cfg.batch_mode == "global":
        return max(1, cfg.batch_size // world)
    return cfg.batch_size
