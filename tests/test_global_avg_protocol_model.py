"""Randomised-interleaving model check of periodic global averaging on the ring (PROTOCOL.md 1.11).

Each rank has one stream: step kernel k - 1, then the gated two-shot all-reduce of step k, then step kernel k; a
kernel's CTAs / warps start only when the previous kernel on that stream has finished.  Step kernel warps perform the
synchronisation actions of `gossip_step_kernel` (WAR ack wait, push, flag, flag wait, mix, ticket, ack) at gossip steps
and a plain pass over theta at averaging steps; all-reduce CTAs do nothing when P does not divide k, and otherwise the
barrier-0 arrive / wait, the owner's reads of every rank's tile and broadcast of the mean, and barrier 1, all with
their own launch counter.  A random scheduler interleaves every actor of every rank.  Checked: no deadlock; every
owner reads every rank's theta as left by step kernel k - 1; every averaging step kernel reads the broadcast mean of
step k; every gossip mix reads exactly the neighbours' push of step k (decent fires every tensor).  Mutants: no
barrier 0, a WAR bound of k - 1 (an ack nobody sends) and one of k - 2 at every step (too early) must be caught."""
import random

import pytest


def run(R, P, steps, seed, G=2, n_tiles=5, n_warps=2, depth=2, barrier0=True, war="exact", max_ticks=600000):
    rng = random.Random(seed)
    iters = -(-n_tiles // G)
    theta = [[[("s", r, 0)] * n_warps for _ in range(n_tiles)] for r in range(R)]   # what last wrote slice (t, w)
    inbox = [{"l": [[0] * n_warps for _ in range(n_tiles)], "r": [[0] * n_warps for _ in range(n_tiles)]}
             for _ in range(R)]
    flag = [{"l": [[0] * n_warps for _ in range(n_tiles)], "r": [[0] * n_warps for _ in range(n_tiles)]}
            for _ in range(R)]
    ack = [{"l": 0, "r": 0} for _ in range(R)]
    ar_flags = [[[[0] * R for _ in range(G)] for _ in range(2)] for _ in range(R)]   # [rank][phase][cta][from]
    step_ctr = [0] * R
    ticket = [0] * R
    ar_ticket = [0] * R
    bad = []

    def pga(k):
        return k % P == 0

    def war_bound(k):
        if war == "k-1":
            return k - 1
        if war == "k-2":
            return k - 2
        return k - 2 if pga(k - 1) else k - 1

    def step_warp(r, b, w, k):
        L, Rn = (r - 1) % R, (r + 1) % R
        if pga(k):
            for j in range(iters):
                t = b + j * G
                if t < n_tiles:
                    if theta[r][t][w] != ("avg", k):
                        bad.append(("stale average", r, t, w, k, theta[r][t][w]))
                    theta[r][t][w] = ("s", r, k)
                    yield None
        else:
            bound = max(war_bound(k), 0)
            yield lambda: ack[r]["l"] >= bound and ack[r]["r"] >= bound
            for j in range(iters + depth):
                t = b + j * G
                if j < iters and t < n_tiles:
                    inbox[L]["r"][t][w] = k
                    inbox[Rn]["l"][t][w] = k
                    yield None
                    flag[L]["r"][t][w] = k
                    flag[Rn]["l"][t][w] = k
                    yield None
                t2 = b + (j - depth) * G
                if j >= depth and t2 < n_tiles:
                    yield lambda t2=t2: flag[r]["l"][t2][w] >= k and flag[r]["r"][t2][w] >= k
                    for side in ("l", "r"):
                        if inbox[r][side][t2][w] != k:
                            bad.append(("inbox", r, side, t2, k, inbox[r][side][t2][w]))
                    theta[r][t2][w] = ("s", r, k)
                    yield None
        ticket[r] += 1
        if ticket[r] == G * n_warps * k and not pga(k):
            ack[L]["r"] = k
            ack[Rn]["l"] = k
        yield None

    def ar_cta(r, b, k):
        if not pga(k):
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
            for q in range(R):                                   # rank-ordered reads of every rank's tile
                if any(x != ("s", q, k - 1) for x in theta[q][t]):
                    bad.append(("owner read", r, q, t, k, theta[q][t]))
                yield None
            for q in range(R):                                   # broadcast the mean
                theta[q][t] = [("avg", k)] * n_warps
                yield None
        yield barrier(1)
        ar_ticket[r] += 1
        if ar_ticket[r] % G == 0:
            step_ctr[r] = seq

    def stream(r):
        """The kernels of rank r in stream order: lists of actors, each list started when the previous has finished."""
        for k in range(1, steps + 1):
            yield [ar_cta(r, b, k) for b in range(G)]
            yield [step_warp(r, b, w, k) for b in range(G) for w in range(n_warps)]

    streams = [stream(r) for r in range(R)]
    running = [[] for _ in range(R)]                             # [ (actor, pending condition) ]

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
    return ("ok" if not live else "timeout"), bad


@pytest.mark.parametrize("P", [2, 3])
def test_global_avg_protocol_is_deadlock_free_and_reads_what_it_should(P):
    for seed in range(30):
        status, bad = run(3, P, steps=3 * P + 1, seed=seed)
        assert status == "ok", (status, seed)
        assert not bad, bad[:3]


def test_mutant_without_barrier_0_is_caught():
    """An owner that does not wait for every rank's arrival reads a peer's theta before its step kernel k - 1 wrote it."""
    caught = sum(bool(run(3, 2, steps=5, seed=s, barrier0=False)[1]) for s in range(40))
    assert caught > 0


def test_mutant_war_bound_k_minus_1_deadlocks():
    """After an average the neighbours' last ack is k - 2: waiting for k - 1 waits for an ack nobody sends."""
    for P in (2, 3):
        assert run(3, P, steps=P + 2, seed=0, war="k-1")[0] == "deadlock"


def test_mutant_war_bound_k_minus_2_is_caught():
    """Waiting for k - 2 after a gossip step lets a fast rank overwrite an inbox slice its neighbour has not mixed."""
    caught = sum(bool(run(3, 3, steps=7, seed=s, war="k-2")[1]) for s in range(60))
    assert caught > 0
