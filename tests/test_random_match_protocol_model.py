"""Randomised-interleaving model check of the single-inbox random-match step (PROTOCOL.md 1.17).

Each rank has one stream: per step k, the match step kernel k and, optionally, the consensus kernel of step k.  The
partner of every rank at every step comes from the real matching (parallel/topology.py match_pairs) under a random
seed.  Step warps perform the synchronisation actions of the kernel: the WAR wait on the partner's `done` word, the push
of their slice of theta into the partner's single inbox, the (tile, warp) flag (the step number), the flag wait of the
slice D tiles back, the mix, the ticket and, in the last warp of the grid, `done = k`.  An idle rank (odd R) only
rewrites its own theta and still publishes `done`.  Consensus CTAs pass barrier 0, read every rank's theta of the tiles
they own (a read spans two scheduler slots, so a write in between is seen) and pass barrier 1.  theta holds the step
that produced it; an inbox slice holds (sender, step).  A random scheduler interleaves every actor of every rank.
Checked: no deadlock; every mix reads its partner's theta of exactly this step, and its own theta of the step before;
every consensus read sees step k on every rank and no write lands during it.  Mutants that must be caught: no WAR wait,
the WAR wait on done >= k - 2, and `done` published by the first warp to finish instead of the last."""
import random

import pytest

from eventgrad_b200.parallel.topology import match_pairs


def run(R, steps, seed, consensus=False, G=2, n_tiles=5, n_warps=2, D=1, war=1, done_early=False,
        max_ticks=800000):
    """war: 1 the kernel's WAR wait (done >= k - 1), 2 the mutant done >= k - 2, 0 none."""
    rng = random.Random(seed)
    mseed = rng.randrange(1 << 31)
    partner = {}
    for k in range(1, steps + 1):
        partner[k] = [None] * R
        for a, b in match_pairs(mseed, R, k):
            partner[k][a], partner[k][b] = b, a
    iters = -(-n_tiles // G)
    z = lambda v=0: [[v] * n_warps for _ in range(n_tiles)]
    theta = [z() for _ in range(R)]
    reading = [[0] * n_tiles for _ in range(R)]
    inbox = [z(None) for _ in range(R)]
    flag = [z() for _ in range(R)]
    done = [0] * R
    ticket = [0] * R
    bar = [[[[0] * R for _ in range(G)] for _ in range(2)] for _ in range(R)]
    cons_ctr = [0] * R
    bad = []

    def write_theta(r, t, w, val):
        if reading[r][t]:
            bad.append(("write under a read", r, t, val))
        theta[r][t][w] = val

    def warp(r, b, w, k):
        p = partner[k][r]
        if p is not None and war:
            yield lambda: done[p] >= k - war
        for j in range(iters + D):
            t = b + j * G
            if p is not None and j < iters and t < n_tiles:
                if theta[r][t][w] != k - 1:
                    bad.append(("push read", r, t, k, theta[r][t][w]))
                inbox[p][t][w] = (r, k)
                yield None
                flag[p][t][w] = k
                yield None
            t2 = b + (j - D) * G
            if j >= D and t2 < n_tiles:
                if p is not None:
                    yield lambda t2=t2: flag[r][t2][w] >= k
                    got = inbox[r][t2][w]
                    if got != (p, k):
                        bad.append(("inbox", r, t2, k, got, p))
                if theta[r][t2][w] != k - 1:
                    bad.append(("own", r, t2, k, theta[r][t2][w]))
                write_theta(r, t2, w, k)
                yield None
        ticket[r] += 1
        if done_early and ticket[r] == G * n_warps * (k - 1) + 1:
            done[r] = k                                     # mutant: published before the grid has finished
        if ticket[r] == G * n_warps * k:
            done[r] = k                                     # the last CTA: every inbox read of step k is done
        yield None

    def cons_cta(r, b, k):
        yield None
        seq = cons_ctr[r] + 1

        def barrier(ph):
            for q in range(R):
                bar[q][ph][b][r] = seq
            return lambda: all(bar[r][ph][b][q] >= seq for q in range(R))

        yield barrier(0)
        for j in range(iters):
            t = b + j * G
            if t >= n_tiles or (b + j) % R != r:
                continue
            for q in range(R):
                reading[q][t] += 1
                yield None
                if any(x != k for x in theta[q][t]):
                    bad.append(("consensus read", r, q, t, k, list(theta[q][t])))
                reading[q][t] -= 1
                yield None
        yield barrier(1)
        cons_ctr[r] = seq

    def stream(r):
        for k in range(1, steps + 1):
            yield [warp(r, b, w, k) for b in range(G) for w in range(n_warps)]
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
            if any(v != steps for row in theta[r] for v in row):
                bad.append(("final", r))
    return ("ok" if not live else "timeout"), bad


@pytest.mark.parametrize("consensus", [False, True])
@pytest.mark.parametrize("R", [3, 4, 5, 6])
def test_match_protocol_is_deadlock_free_and_reads_the_partners_step(R, consensus):
    for seed in range(20):
        status, bad = run(R, 5, seed, consensus=consensus)
        assert status == "ok", (status, seed)
        assert not bad, bad[:3]


@pytest.mark.parametrize("mutant", ["no_war", "war_k_minus_2", "done_early"])
def test_mutants_are_caught(mutant):
    """Each weakening lets a new partner overwrite an inbox that its owner is still reading from the previous step."""
    kw = {"no_war": dict(war=0), "war_k_minus_2": dict(war=2), "done_early": dict(done_early=True)}[mutant]
    caught = 0
    for R in (3, 4, 5, 6):
        caught += sum(bool(run(R, 5, s, **kw)[1]) for s in range(40))
    assert caught > 0
