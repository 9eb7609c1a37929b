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

`OnePeerExp` ("onepeer-exp") is the time-varying one-peer exponential graph (Ying et al., NeurIPS 2021).  For R >= 2
let tau = ceil(log2 R) and o_m = 2^m, m = 0 .. tau-1 (every o_m < R).  Steps are 1-based (the device step counter
pass_num + 1); at step k the active index is m = (k-1) mod tau.  Rank r pushes its fired tensors to r + o_m only, and
mixes with slot m, which holds what it last received from r - o_m:
    theta' = (theta + s_m) / 2          (one rounded add, one true division)
so W_k = (I + S^{o_m}) / 2 is doubly stochastic but directed (not symmetric), and a rank sends ONE copy per step.  When
R is a power of two, W_tau ... W_1 = 11^T / R: exact consensus every tau steps.  At R == 2 (tau == 1) the mix is
(theta + theta_peer) / 2, deliberately not the ring's (theta + 2 theta_peer) / 3.  At R == 1 the name resolves to the
ring.  Rank r has tau slots: slot m receives from r - o_m and out-slot m feeds slot m of r + o_m.  In event mode slot m
keeps the last value that arrived from r - o_m, which can be from step k - tau or earlier; the trigger state is per
tensor, not per peer.

`RandomMatch` ("random-match") is randomized pairwise gossip (Boyd et al. 2006): at every step the ranks are split into
pairs by a random perfect matching, and each rank averages with its partner,
    theta' = (theta + theta_partner) / 2          (one rounded add, one true division, as onepeer-exp)
For odd R one rank is idle at each step (its own SGD step only).  The matching is a pure function of (seed, R, k),
`match_pairs` below, so every rank computes it itself; csrc/gossip.cu (EG_MATCH) holds the identical device copy.  W_k
is symmetric, doubly stochastic and idempotent, and lambda_2(E[W]) = (R - 2) / (2 (R - 1)) for even R, 1/2 for odd R.
A rank sends ONE copy per step (none when idle).  At R == 1 the name resolves to the ring; at R == 2 the pair is fixed
and the mix is onepeer-exp's.

`circulant_spectrum` / `chebyshev_coefficients` give the closed-form spectrum of a circulant W on 1^perp and the
coefficients of Chebyshev-accelerated gossip rounds (--gossip-accel chebyshev) fitted to it.  Every backend and the
simulator take the coefficients from here; no other module derives the spectrum.
"""
from __future__ import annotations

import math
import struct
from dataclasses import dataclass
from typing import List, Optional, Tuple

MAX_OFFSETS = 4          # degree <= 8 (csrc/api.h EG_MAX_SLOTS)
MAX_SLOTS = 8            # csrc/api.h EG_MAX_SLOTS: the one-peer graph's period tau <= 8, i.e. R <= 256
RING = (1,)
ONEPEER = "onepeer-exp"
MATCH = "random-match"
MATCH_MAX_WORLD = 1024   # csrc/api.h EG_MATCH_MAX_WORLD: the device copy of the shuffle keeps pi in shared memory
_M64 = (1 << 64) - 1


def is_onepeer(spec) -> bool:
    return isinstance(spec, str) and spec.strip().lower() == ONEPEER


def is_match(spec) -> bool:
    """The random-match topology, by name or by topology object."""
    if isinstance(spec, str):
        return spec.strip().lower() == MATCH
    return getattr(spec, "kind", None) == MATCH


def check_match_seed(seed) -> None:
    """--topology-seed: an int in [0, 2^31) (not a bool)."""
    if isinstance(seed, bool) or not isinstance(seed, int) or not 0 <= seed < (1 << 31):
        raise ValueError(f"--topology-seed must be an integer in [0, 2^31), got {seed!r}")


def _splitmix64(x: int) -> Tuple[int, int]:
    """One step of splitmix64: (new state, output)."""
    x = (x + 0x9E3779B97F4A7C15) & _M64
    z = x
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return x, z ^ (z >> 31)


def match_perm(seed: int, world: int, step: int) -> List[int]:
    """The shuffled rank order pi of 1-based step `step`: x_0 = (seed << 32) ^ step, then Fisher-Yates from the
    identity, for i = R-1 down to 1 swap pi[i] and pi[next() mod (i + 1)]."""
    if step < 1:
        raise ValueError(f"steps are 1-based, got {step}")
    x = ((seed << 32) ^ step) & _M64
    pi = list(range(world))
    for i in range(world - 1, 0, -1):
        x, z = _splitmix64(x)
        j = z % (i + 1)
        pi[i], pi[j] = pi[j], pi[i]
    return pi


def match_pairs(seed: int, world: int, step: int) -> List[Tuple[int, int]]:
    """The pairs (pi[0], pi[1]), (pi[2], pi[3]), ... of step `step`; for odd R, pi[R-1] is idle."""
    pi = match_perm(seed, world, step)
    return [(pi[i], pi[i + 1]) for i in range(0, world - 1, 2)]


def match_partner(seed: int, world: int, step: int, rank: int) -> Optional[int]:
    """The partner of `rank` at step `step`, or None when it is idle."""
    pi = match_perm(seed, world, step)
    pos = pi.index(rank)
    if pos == world - 1 and world % 2 == 1:
        return None
    return pi[pos ^ 1]


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

    @property
    def fanout(self) -> int:
        """Messages one fired tensor costs per step (the event counter's unit)."""
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
    At world == 1 every name resolves to the ring (serial / self-loop semantics).  onepeer-exp is time-varying and
    has no static offsets: at world >= 2 it raises here (OnePeerExp / Graph.build handle it)."""
    if isinstance(spec, (tuple, list)):
        spec = ",".join(str(int(o)) for o in spec)
    s = str(spec).strip().lower()
    if s in ("", "ring"):
        return RING
    if world < 1:
        raise ValueError(f"world must be >= 1, got {world}")
    if s in (ONEPEER, MATCH):
        if world == 1:
            return RING
        raise ValueError(f"{s} is time-varying: it has no static offsets (use Graph.build)")
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
    if s in ("ring", "exp", ONEPEER, MATCH):
        return
    try:
        offs = [int(x) for x in s.split(",")]
    except ValueError:
        raise ValueError(f"topology must be ring, exp, {ONEPEER}, {MATCH} or comma-separated offsets like '1,3', "
                         f"got {spec!r}") from None
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
    def build(rank: int, world: int, spec="ring", seed: int = 0):
        """The graph of `spec` for this rank: a `Graph`, a `OnePeerExp` for onepeer-exp at world >= 2, or a
        `RandomMatch` with matching seed `seed` for random-match at world >= 2."""
        if is_onepeer(spec) and world >= 2:
            return OnePeerExp(rank, world)
        if is_match(spec) and world >= 2:
            return RandomMatch(rank, world, seed)
        return Graph(rank, world, parse_topology(spec, world))

    period = 0               # static graph (OnePeerExp: tau)
    kind = "circulant"       # checkpoint tag (utils/ckpt.py via parallel/base.py)

    @property
    def is_ring(self) -> bool:
        return self.offsets == RING

    @property
    def serial(self) -> bool:
        return self.world == 1

    @property
    def n_slots(self) -> int:
        return 2 * len(self.offsets)

    @property
    def fanout(self) -> int:
        """Messages one fired tensor costs per step: one per slot it lands in."""
        return self.n_slots

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


def onepeer_period(world: int) -> int:
    """tau = ceil(log2 world) for world >= 2."""
    if world < 2:
        raise ValueError(f"{ONEPEER} needs at least 2 ranks, got {world}")
    return (world - 1).bit_length()


@dataclass(frozen=True)
class OnePeerExp:
    """Time-varying one-peer exponential graph of one rank (see the module docstring).  Slot m receives from r - o_m;
    out-slot m feeds slot m of r + o_m; at step k (1-based) only slot active(k) takes part."""
    rank: int
    world: int

    kind = ONEPEER
    is_ring = False

    def __post_init__(self):
        if not (0 <= self.rank < self.world):
            raise ValueError(f"rank {self.rank} outside world {self.world}")
        if onepeer_period(self.world) > MAX_SLOTS:
            raise ValueError(f"{ONEPEER}: at most {2 ** MAX_SLOTS} ranks ({MAX_SLOTS} slots), got {self.world}")

    @property
    def period(self) -> int:
        return onepeer_period(self.world)

    @property
    def offsets(self) -> Tuple[int, ...]:
        return tuple(1 << m for m in range(self.period))

    @property
    def serial(self) -> bool:
        return False

    @property
    def n_slots(self) -> int:
        return self.period

    @property
    def fanout(self) -> int:
        """Messages one fired tensor costs per step: it goes to the single out-peer of the step."""
        return 1

    def active(self, step: int) -> int:
        """Active slot / offset index of 1-based step `step`."""
        if step < 1:
            raise ValueError(f"steps are 1-based, got {step}")
        return (step - 1) % self.period

    def in_peer(self, step: int) -> int:
        return (self.rank - self.offsets[self.active(step)]) % self.world

    def out_peer(self, step: int) -> int:
        return (self.rank + self.offsets[self.active(step)]) % self.world

    def slots(self) -> List[int]:
        """Peer whose pushes land in each of my slots: slot m from r - 2^m."""
        return [(self.rank - o) % self.world for o in self.offsets]

    def out_slots(self) -> List[Tuple[int, int]]:
        """For each slot index m, the (peer, peer's slot) I push into when m is active: slot m of r + 2^m."""
        return [((self.rank + o) % self.world, m) for m, o in enumerate(self.offsets)]

    def mixing_row(self, step: int) -> List[float]:
        """Row of W_step = (I + S^{o_m}) / 2: weight 1/2 on me and on the in-peer of the step."""
        row = [0.0] * self.world
        row[self.rank] += 0.5
        row[self.in_peer(step)] += 0.5
        return row


@dataclass(frozen=True)
class RandomMatch:
    """Random pairwise matchings of one rank (see the module docstring): at step k (1-based) this rank averages with
    match_partner(seed, R, k, rank), or is idle.  One inbox, whoever the sender; no static slots."""
    rank: int
    world: int
    seed: int = 0

    kind = MATCH
    is_ring = False
    period = 0               # not the one-peer graph's slot cycle: the partner comes from the matching
    offsets = ()             # no circulant offsets (checkpoints store the name and the seed)

    def __post_init__(self):
        if not (0 <= self.rank < self.world):
            raise ValueError(f"rank {self.rank} outside world {self.world}")
        if self.world < 2:
            raise ValueError(f"{MATCH} needs at least 2 ranks, got {self.world} (R = 1 resolves to the ring)")
        if self.world > MATCH_MAX_WORLD:
            raise ValueError(f"{MATCH}: at most {MATCH_MAX_WORLD} ranks, got {self.world}")
        check_match_seed(self.seed)

    @property
    def serial(self) -> bool:
        return False

    @property
    def n_slots(self) -> int:
        return 1

    @property
    def fanout(self) -> int:
        """Messages one tensor costs per step on a matched rank: one copy to the partner (an idle rank sends none)."""
        return 1

    def partner(self, step: int) -> Optional[int]:
        return match_partner(self.seed, self.world, step, self.rank)

    def mixing_row(self, step: int) -> List[float]:
        """Row of W_step: 1/2 on me and 1/2 on my partner, or 1 on me when idle."""
        row = [0.0] * self.world
        p = self.partner(step)
        if p is None:
            row[self.rank] = 1.0
        else:
            row[self.rank] += 0.5
            row[p] += 0.5
        return row


# ---- Chebyshev-accelerated gossip rounds (--gossip-accel chebyshev) ---------------------------------------------------
ACCELS = ("none", "chebyshev")
CHEB_POINT = 1e-12       # half-width below which the spectrum on 1^perp is one point (the ring at R = 2 and R = 3)


def _fp32(x: float) -> float:
    """x rounded once to the nearest fp32 (round half to even), as a Python float."""
    return struct.unpack("f", struct.pack("f", x))[0]


def circulant_spectrum(offsets, world: int) -> Tuple[float, float]:
    """(a, b) = (min, max) of W's eigenvalues on 1^perp, in float64, for the circulant graph of `offsets` at `world`
    ranks: lambda_j = (1 + 2 sum_o cos(2 pi j o / R)) / (2|O| + 1), j = 1 .. R - 1.  This is mixing_row()'s W, the
    double count at o = R/2 (and so the ring at R = 2, quirk Q15) included."""
    offs = parse_topology(tuple(offsets), world)
    if world < 2:
        raise ValueError("the spectrum on 1^perp needs at least 2 ranks")
    n = 2 * len(offs)
    lam = [(1.0 + 2.0 * sum(math.cos(2.0 * math.pi * j * o / world) for o in offs)) / (n + 1)
           for j in range(1, world)]
    return min(lam), max(lam)


def chebyshev_coefficients(offsets, world: int, rounds: int, fp32: bool = True) -> List[Tuple[float, float]]:
    """The (alpha_q, omega_q), q = 1 .. `rounds`, of Chebyshev-accelerated gossip on the circulant graph of `offsets`:
    round q mixes w = W x_{q-1} and forms
        x_q = x_{q-1} + alpha_q (w - x_{q-1}) + omega_q (x_{q-1} - x_{q-2})        (no omega term at q = 1)
    so that x_Q = P_Q(W) x_0 with P_Q(W) = T_Q((W - c) / delta) / T_Q(mu), the degree-Q polynomial with P_Q(1) = 1 that
    is smallest on W's spectrum [a, b] (circulant_spectrum): c = (a + b) / 2, delta = (b - a) / 2, mu = (1 - c) / delta,
    rho_1 = 1 / mu, rho_q = 1 / (2 mu - rho_{q-1}); alpha_1 = rho_1 / delta, omega_1 = 0, alpha_q = 2 rho_q / delta,
    omega_q = rho_q rho_{q-1}.  On 1^perp P_Q(W) contracts by 1 / T_Q(mu).  A one-point spectrum (delta <= 1e-12) gives
    alpha_q = 1 / (1 - c) and omega_q = 0: one round is the exact average.  Everything is float64; `fp32` rounds each
    coefficient once to fp32, the values every backend and the simulator use."""
    if isinstance(rounds, bool) or int(rounds) != rounds or rounds < 1:
        raise ValueError(f"rounds must be an integer >= 1, got {rounds!r}")
    a, b = circulant_spectrum(offsets, world)
    c, delta = (a + b) / 2.0, (b - a) / 2.0
    out = []
    if delta <= CHEB_POINT:
        out = [(1.0 / (1.0 - c), 0.0)] * int(rounds)
    else:
        mu = (1.0 - c) / delta
        rho = 1.0 / mu
        out.append((rho / delta, 0.0))
        for _ in range(2, int(rounds) + 1):
            rho_prev, rho = rho, 1.0 / (2.0 * mu - rho)
            out.append((2.0 * rho / delta, rho * rho_prev))
    return [(_fp32(al), _fp32(om)) for al, om in out] if fp32 else out
