"""Logical gossip topologies (rank order), including the degenerate sizes.

Reference: left=(rank-1) mod N, right=(rank+1) mod N
(/root/reference/dmnist/event/event.cpp:114-122); the CIFAR programs only set it
when numranks>1 (/root/reference/dcifar10/event/event.cpp:70-81).

On NVSwitch every peer is one hop away, so the graph is purely logical: no
topology-aware placement is needed and ring order == rank order.

Beyond the reference's ring, `Graph` is a circulant graph given by a set of offsets
O = {o_1 < o_2 < ...} within [1, R//2].  Rank r has 2|O| inbox *slots* in a fixed order: for
each o ascending, "from r-o" (slot 2k), then "from r+o" (slot 2k+1).  The mix is
    theta' = (((theta + s_0) + s_1) + ... + s_{2|O|-1}) / (2|O| + 1)
so the mixing matrix W = (I + sum_o (S^o + S^-o)) / (2|O|+1) is symmetric and doubly stochastic.
When o == R/2 both slots of o come from the same peer and that peer counts twice (the rule the
ring follows at R == 2, quirk Q15).  O == (1,) is the ring, bit for bit.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Tuple

MAX_OFFSETS = 4          # degree <= 8 (csrc/api.h EG_MAX_SLOTS)
RING = (1,)


@dataclass(frozen=True)
class Ring:
    rank: int
    world: int

    def __post_init__(self):
        if not (0 <= self.rank < self.world):
            raise ValueError(f"rank {self.rank} outside world {self.world}")

    offsets = RING

    @property
    def is_ring(self) -> bool:
        return True

    @property
    def left(self) -> int:
        return (self.rank - 1) % self.world

    @property
    def right(self) -> int:
        return (self.rank + 1) % self.world

    @property
    def degenerate_pair(self) -> bool:
        """R == 2: left == right, the same peer is counted twice -> (theta + 2 theta')/3
        (SURVEY.md A.4 / Q15)."""
        return self.world == 2

    @property
    def serial(self) -> bool:
        return self.world == 1

    @property
    def n_slots(self) -> int:
        return 2

    def neighbours(self):
        return self.left, self.right

    def slots(self) -> List[int]:
        return [self.left, self.right]

    def out_slots(self) -> List[Tuple[int, int]]:
        """(peer, peer's slot) I push into: my right neighbour's "from left" (0), my left neighbour's "from right" (1)."""
        return [(self.right, 0), (self.left, 1)]

    def mixing_row(self):
        """Row of the doubly-stochastic mixing matrix W for this rank (weights 1/3)."""
        row = [0.0] * self.world
        row[self.rank] += 1.0 / 3.0
        row[self.left] += 1.0 / 3.0
        row[self.right] += 1.0 / 3.0
        return row


def parse_topology(spec, world: int) -> Tuple[int, ...]:
    """Offsets of a topology name for a world of `world` ranks.

    ring          (1,)
    exp           (1, 2, 4, ...) up to world // 2 (at most MAX_OFFSETS of them)
    "o1,o2,..."   explicit offsets: ascending, distinct, each in [1, world // 2], at most MAX_OFFSETS
    At world == 1 every name resolves to the ring (serial / self-loop semantics)."""
    if isinstance(spec, (tuple, list)):
        spec = ",".join(str(int(o)) for o in spec)
    s = str(spec).strip().lower()
    if s in ("", "ring"):
        return RING
    if world < 1:
        raise ValueError(f"world must be >= 1, got {world}")
    half = world // 2
    if s == "exp":
        offs, o = [], 1
        while o <= max(1, half) and len(offs) < MAX_OFFSETS:
            offs.append(o)
            o *= 2
        return tuple(offs)
    try:
        offs = tuple(int(x) for x in s.split(","))
    except ValueError:
        raise ValueError(f"topology must be ring, exp or comma-separated offsets like '1,3', got {spec!r}") from None
    if world == 1:
        if offs != RING:
            raise ValueError(f"topology {spec!r}: a single rank has no neighbours, only the ring applies")
        return RING
    if len(offs) > MAX_OFFSETS:
        raise ValueError(f"topology {spec!r}: at most {MAX_OFFSETS} offsets (degree <= {2 * MAX_OFFSETS})")
    if list(offs) != sorted(set(offs)):
        raise ValueError(f"topology {spec!r}: offsets must be distinct and ascending")
    if offs[0] < 1 or offs[-1] > half:
        raise ValueError(f"topology {spec!r}: offsets must lie in [1, {half}] for {world} ranks")
    return offs


def check_topology_name(spec) -> None:
    """World-independent syntax check of a topology name (TrainConfig.validate)."""
    s = str(spec).strip().lower()
    if s in ("ring", "exp"):
        return
    try:
        offs = [int(x) for x in s.split(",")]
    except ValueError:
        raise ValueError(f"topology must be ring, exp or comma-separated offsets like '1,3', got {spec!r}") from None
    if not offs or len(offs) > MAX_OFFSETS or offs != sorted(set(offs)) or offs[0] < 1:
        raise ValueError(f"topology {spec!r}: 1 to {MAX_OFFSETS} distinct ascending offsets >= 1")


@dataclass(frozen=True)
class Graph:
    """Circulant gossip graph of one rank (see the module docstring for the slot order)."""
    rank: int
    world: int
    offsets: Tuple[int, ...] = RING

    def __post_init__(self):
        if not (0 <= self.rank < self.world):
            raise ValueError(f"rank {self.rank} outside world {self.world}")
        object.__setattr__(self, "offsets", parse_topology(tuple(self.offsets), self.world))

    @staticmethod
    def build(rank: int, world: int, spec="ring") -> "Graph":
        return Graph(rank, world, parse_topology(spec, world))

    @property
    def is_ring(self) -> bool:
        return self.offsets == RING

    @property
    def serial(self) -> bool:
        return self.world == 1

    @property
    def n_slots(self) -> int:
        return 2 * len(self.offsets)

    def slots(self) -> List[int]:
        """Peer whose pushes land in each of my slots: for o ascending, r-o then r+o."""
        out = []
        for o in self.offsets:
            out += [(self.rank - o) % self.world, (self.rank + o) % self.world]
        return out

    def out_slots(self) -> List[Tuple[int, int]]:
        """For each slot index j, the (peer, peer's slot) I push into.  I am slot 2k ("from p-o") of p = r+o and slot
        2k+1 ("from p+o") of p = r-o, so out-slot j always targets the peer's slot j."""
        out = []
        for k, o in enumerate(self.offsets):
            out += [((self.rank + o) % self.world, 2 * k), ((self.rank - o) % self.world, 2 * k + 1)]
        return out

    def mixing_row(self) -> List[float]:
        """Row of W = (I + sum_o (S^o + S^-o)) / (2|O|+1); a peer reached through two slots counts twice."""
        w = 1.0 / (self.n_slots + 1)
        row = [0.0] * self.world
        row[self.rank] += w
        for p in self.slots():
            row[p] += w
        return row

    # ---- Ring compatibility (offsets == (1,)) ---------------------------------------------
    def _ring_only(self):
        if not self.is_ring:
            raise AttributeError(f"left/right are defined for the ring only (offsets {self.offsets})")

    @property
    def left(self) -> int:
        self._ring_only()
        return (self.rank - 1) % self.world

    @property
    def right(self) -> int:
        self._ring_only()
        return (self.rank + 1) % self.world

    @property
    def degenerate_pair(self) -> bool:
        self._ring_only()
        return self.world == 2

    def neighbours(self):
        return self.left, self.right
