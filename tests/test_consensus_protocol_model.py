"""Randomised-interleaving model check of the consensus kernel after the ring step (PROTOCOL.md 1.14).

Each rank has one stream.  Fused step: step kernel k, then the gated consensus kernel of step k.  Split step: the push
of k (it only reads theta), the mix of k, then the consensus kernel of k -- the side stream's push of k + 1 waits for
the main stream, so it follows the consensus kernel of k.  Step kernel warps perform the synchronisation actions of
`gossip_step_kernel` (WAR ack wait, push, flag, flag wait, mix, ticket, ack).  Consensus CTAs do nothing when N does
not divide k; otherwise barrier 0, the owner's reads of every rank's tile (a read spans two scheduler slots, so a write
in between is seen), the broadcast of its partial into every rank's partial buffer, barrier 1, the ticket and, in the
last CTA, the reduction of every partial into the ring row of step k.  A random scheduler interleaves every actor of
every rank.  Checked: no deadlock; every owner reads every rank's theta exactly as step kernel k left it, and no write
lands during a read; every mix reads the neighbours' push of step k; every rank's last CTA sees the partials of step k
for every tile; every rank records exactly the steps N divides.  Mutants: no barrier 0 and no barrier 1 must be
caught."""
import random

import pytest


def run(R, N, steps, seed, split=False, G=2, n_tiles=5, n_warps=2, barrier0=True, barrier1=True,
        max_ticks=600000):
    rng = random.Random(seed)
    iters = -(-n_tiles // G)
    theta = [[[("s", r, 0)] * n_warps for _ in range(n_tiles)] for r in range(R)]
    reading = [[0] * n_tiles for _ in range(R)]                  # owners in the middle of a read of (rank, tile)
    inbox = [{"l": [[0] * n_warps for _ in range(n_tiles)], "r": [[0] * n_warps for _ in range(n_tiles)]}
             for _ in range(R)]
    flag = [{"l": [[0] * n_warps for _ in range(n_tiles)], "r": [[0] * n_warps for _ in range(n_tiles)]}
            for _ in range(R)]
    ack = [{"l": 0, "r": 0} for _ in range(R)]
    ar_flags = [[[[0] * R for _ in range(G)] for _ in range(2)] for _ in range(R)]   # [rank][phase][cta][from]
    part = [[0] * n_tiles for _ in range(R)]                      # step whose partial tile t of rank r holds
    step_ctr = [0] * R
    ticket = [0] * R
    pticket = [0] * R
    ar_ticket = [0] * R
    ring = [[] for _ in range(R)]
    bad = []

    def write_theta(r, t, w, val):
        if reading[r][t]:
            bad.append(("write under a read", r, t, val))
        theta[r][t][w] = val

    def push_warp(r, b, w, k):
        L, Rn = (r - 1) % R, (r + 1) % R
        yield lambda: ack[r]["l"] >= k - 1 and ack[r]["r"] >= k - 1
        for j in range(iters):
            t = b + j * G
            if t < n_tiles:
                if theta[r][t][w] != ("s", r, k - 1):
                    bad.append(("push read", r, t, k, theta[r][t][w]))
                inbox[L]["r"][t][w] = k
                inbox[Rn]["l"][t][w] = k
                yield None
                flag[L]["r"][t][w] = k
                flag[Rn]["l"][t][w] = k
                yield None
        pticket[r] += 1

    def mix_warp(r, b, w, k, push):
        L, Rn = (r - 1) % R, (r + 1) % R
        if push:
            yield from push_warp(r, b, w, k)
        for j in range(iters):
            t = b + j * G
            if t < n_tiles:
                yield lambda t=t: flag[r]["l"][t][w] >= k and flag[r]["r"][t][w] >= k
                for side in ("l", "r"):
                    if inbox[r][side][t][w] != k:
                        bad.append(("inbox", r, side, t, k, inbox[r][side][t][w]))
                write_theta(r, t, w, ("s", r, k))
                yield None
        ticket[r] += 1
        if ticket[r] == G * n_warps * k:
            ack[L]["r"] = k
            ack[Rn]["l"] = k
        yield None

    def cons_cta(r, b, k):
        if k % N:
            return                                               # the gate: no barrier, no counter
        yield None
        seq = step_ctr[r] + 1

        def barrier(ph):
            for q in range(R):
                ar_flags[q][ph][b][r] = seq
            return lambda: all(ar_flags[r][ph][b][q] >= seq for q in range(R))

        if barrier0:
            yield barrier(0)
        for j in range(iters):
            t = b + j * G
            if t >= n_tiles or (b + j) % R != r:
                continue
            for _pass in range(2):                               # theta_bar, then the deviations
                for q in range(R):
                    reading[q][t] += 1
                    yield None
                    if any(x != ("s", q, k) for x in theta[q][t]):
                        bad.append(("owner read", r, q, t, k, theta[q][t]))
                    reading[q][t] -= 1
                    yield None
            for q in range(R):                                   # the partial into every rank's buffer
                part[q][t] = k
                yield None
        if barrier1:
            yield barrier(1)
        ar_ticket[r] += 1
        if ar_ticket[r] % G == 0:                                # last CTA: reduce the partials into the ring
            if any(p != k for p in part[r]):
                bad.append(("partials", r, k, list(part[r])))
            ring[r].append(k)
            step_ctr[r] = seq

    def stream(r):
        """The kernels of rank r in stream order: lists of actors, each list started when the previous has finished."""
        for k in range(1, steps + 1):
            if split:
                yield [push_warp(r, b, w, k) for b in range(G) for w in range(n_warps)]
            yield [mix_warp(r, b, w, k, not split) for b in range(G) for w in range(n_warps)]
            yield [cons_cta(r, b, k) for b in range(G)]

    streams = [stream(r) for r in range(R)]
    running = [[] for _ in range(R)]

    def launch(r):
        while not running[r]:
            try:
                actors = next(streams[r])
            except StopIteration:
                return False
            for a in actors:
                try:
                    running[r].append([a, next(a)])
                except StopIteration:
                    pass
        return True

    live = {r for r in range(R) if launch(r)}
    ticks = 0
    while live and ticks < max_ticks:
        ready = [(r, i) for r in live for i, (_, c) in enumerate(running[r]) if c is None or c()]
        if not ready:
            return "deadlock", bad, ring
        r, i = rng.choice(ready)
        act = running[r][i]
        try:
            act[1] = next(act[0])
        except StopIteration:
            running[r].pop(i)
            if not running[r] and not launch(r):
                live.discard(r)
        ticks += 1
    return ("ok" if not live else "timeout"), bad, ring


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("N", [1, 2])
def test_consensus_protocol_is_deadlock_free_and_reads_what_it_should(N, split):
    steps = 5
    for seed in range(30):
        status, bad, ring = run(3, N, steps, seed, split=split)
        assert status == "ok", (status, seed)
        assert not bad, bad[:3]
        assert all(rr == list(range(N, steps + 1, N)) for rr in ring), ring


@pytest.mark.parametrize("split", [False, True])
def test_mutant_without_barrier_0_is_caught(split):
    """An owner that does not wait for every rank's arrival reads a peer's theta before its step kernel k wrote it."""
    caught = sum(bool(run(3, 1, steps=4, seed=s, split=split, barrier0=False)[1]) for s in range(40))
    assert caught > 0


@pytest.mark.parametrize("split", [False, True])
def test_mutant_without_barrier_1_is_caught(split):
    """A rank that leaves without barrier 1 starts step k + 1 and overwrites theta under a slow owner's read, or reduces
    partials that have not arrived."""
    caught = sum(bool(run(3, 1, steps=4, seed=s, split=split, barrier1=False)[1]) for s in range(60))
    assert caught > 0
