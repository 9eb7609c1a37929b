"""Randomised-interleaving model check of the gossip rounds ahead of the ring step (PROTOCOL.md 1.16).

Each rank has one stream: per step k, the Q - 1 round kernels (h = (Q - 1)(k - 1) + q), the ring step kernel k (the
single-slot inbox with its WAR ack, or the double-buffered inbox, slot k & 1, without one) and, optionally, the consensus
kernel of step k.  Round and step warps perform the synchronisation actions of their kernels: the WAR wait on the
acks, the push of their slice of theta into both out-slots, the (tile, warp) flag, the flag wait of the slice D tiles
back, the mix, the ticket and, in the last warp, the acks.  Consensus CTAs pass barrier 0, read every rank's theta of
the tiles they own (a read spans two scheduler slots, so a write in between is seen) and pass barrier 1.  theta is a
version counter: after step k it is kQ, after round q of step k it is (k - 1)Q + q.  A random scheduler interleaves
every actor of every rank.  Checked: no deadlock; every mix reads the neighbours' theta of exactly the version it
expects, round inbox and step inbox alike, and its own; every consensus read sees version kQ on every rank and no write
lands during it.  Mutant: a round kernel without its WAR guard must be caught."""
import random

import pytest


def run(R, Q, steps, seed, dbuf=False, consensus=False, G=2, n_tiles=5, n_warps=2, D=1, war=True, max_ticks=800000):
    rng = random.Random(seed)
    iters = -(-n_tiles // G)
    slots_of = lambda r: [(r - 1) % R, (r + 1) % R]                      # slot 0 from the left, slot 1 from the right
    outs_of = lambda r: [((r + 1) % R, 0), ((r - 1) % R, 1)]            # out-slot j writes slot j of its peer
    z = lambda: [[0] * n_warps for _ in range(n_tiles)]
    theta = [z() for _ in range(R)]
    reading = [[0] * n_tiles for _ in range(R)]
    rin, rflag, rack = [[z(), z()] for _ in range(R)], [[z(), z()] for _ in range(R)], [[0, 0] for _ in range(R)]
    nb = 2 if dbuf else 1
    sin = [[[z() for _ in range(nb)] for _ in range(2)] for _ in range(R)]
    sflag, sack = [[z(), z()] for _ in range(R)], [[0, 0] for _ in range(R)]
    rticket, sticket = [0] * R, [0] * R
    bar = [[[[0] * R for _ in range(G)] for _ in range(2)] for _ in range(R)]
    cons_ctr = [0] * R
    bad = []

    def write_theta(r, t, w, val):
        if reading[r][t]:
            bad.append(("write under a read", r, t, val))
        theta[r][t][w] = val

    def warp(r, b, w, k, q):
        """q in 1 .. Q - 1: round q of step k; q == 0: the step kernel of step k."""
        rnd = q > 0
        h = (Q - 1) * (k - 1) + q if rnd else k
        want = (k - 1) * Q + q - 1 if rnd else k * Q - 1                # the version every pushed / mixed slice holds
        inbox, flag, ack = (rin, rflag, rack) if rnd else (sin, sflag, sack)
        buf = 0 if rnd or not dbuf else k & 1
        if rnd and war:
            yield lambda: all(rack[r][j] >= h - 1 for j in range(2))
        elif not rnd and not dbuf:
            yield lambda: all(sack[r][j] >= k - 1 for j in range(2))
        for j in range(iters + D):
            t = b + j * G
            if j < iters and t < n_tiles:
                v = theta[r][t][w]
                if v != want:
                    bad.append(("push read", r, t, k, q, v))
                for p, s in outs_of(r):
                    (inbox[p][s] if rnd else inbox[p][s][buf])[t][w] = v
                    yield None
                for p, s in outs_of(r):
                    flag[p][s][t][w] = h
                yield None
            t2 = b + (j - D) * G
            if j >= D and t2 < n_tiles:
                yield lambda t2=t2: all(flag[r][s][t2][w] >= h for s in range(2))
                for s in range(2):
                    got = (inbox[r][s] if rnd else inbox[r][s][buf])[t2][w]
                    if got != want:
                        bad.append(("inbox", "round" if rnd else "step", r, s, t2, k, q, got))
                if theta[r][t2][w] != want:
                    bad.append(("own", r, t2, k, q, theta[r][t2][w]))
                write_theta(r, t2, w, want + 1)
                yield None
        tk = rticket if rnd else sticket
        tk[r] += 1
        if tk[r] == G * n_warps * h and (rnd or not dbuf):
            for s, sender in enumerate(slots_of(r)):
                ack[sender][s] = h
        yield None

    def cons_cta(r, b, k):
        yield None
        seq = cons_ctr[r] + 1

        def barrier(ph):
            for p in range(R):
                bar[p][ph][b][r] = seq
            return lambda: all(bar[r][ph][b][p] >= seq for p in range(R))

        yield barrier(0)
        for j in range(iters):
            t = b + j * G
            if t >= n_tiles or (b + j) % R != r:
                continue
            for p in range(R):
                reading[p][t] += 1
                yield None
                if any(x != k * Q for x in theta[p][t]):
                    bad.append(("consensus read", r, p, t, k, list(theta[p][t])))
                reading[p][t] -= 1
                yield None
        yield barrier(1)
        cons_ctr[r] = seq

    def stream(r):
        for k in range(1, steps + 1):
            for q in range(1, Q):
                yield [warp(r, b, w, k, q) for b in range(G) for w in range(n_warps)]
            yield [warp(r, b, w, k, 0) for b in range(G) for w in range(n_warps)]
            if consensus:
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
            return "deadlock", bad
        r, i = rng.choice(ready)
        act = running[r][i]
        try:
            act[1] = next(act[0])
        except StopIteration:
            running[r].pop(i)
            if not running[r] and not launch(r):
                live.discard(r)
        ticks += 1
    if not live:
        for r in range(R):
            if any(v != steps * Q for row in theta[r] for v in row):
                bad.append(("final", r))
    return ("ok" if not live else "timeout"), bad


@pytest.mark.parametrize("consensus", [False, True])
@pytest.mark.parametrize("dbuf", [False, True])
@pytest.mark.parametrize("Q", [2, 3])
def test_rounds_protocol_is_deadlock_free_and_reads_what_it_should(Q, dbuf, consensus):
    for seed in range(25):
        status, bad = run(3, Q, 4, seed, dbuf=dbuf, consensus=consensus)
        assert status == "ok", (status, seed)
        assert not bad, bad[:3]


@pytest.mark.parametrize("dbuf", [False, True])
def test_mutant_without_the_round_war_guard_is_caught(dbuf):
    """A round that does not wait for its out-peers' acks of round h - 1 overwrites a round inbox a slow peer has not
    read yet."""
    caught = sum(bool(run(3, 3, steps=3, seed=s, dbuf=dbuf, war=False)[1]) for s in range(60))
    assert caught > 0
