"""Randomised-interleaving model check of Chebyshev gossip rounds followed by a step with no handshake (PROTOCOL.md 1.18).

Each rank has one stream: per step k, the Q Chebyshev round kernels (h = Q(k - 1) + q), the serial step kernel k (no
push, no flag, no ack: each warp rewrites its own slices of theta) and, optionally, the consensus kernel of step k.
Round warps perform the synchronisation actions of the round kernel: the WAR wait on the round acks of h - 1, the push
of their slice of theta into both out-slots, the (tile, warp) flag, the flag wait of the slice D tiles back, the mix
with its reads of the round inboxes, of theta and (q >= 2) of `prev`, the stores of `prev` (q < Q) and theta, the ticket
and, in the last warp, the acks.  Consensus CTAs pass barrier 0, read every rank's theta of the tiles they own (a read
spans two scheduler slots, so a write in between is seen) and pass barrier 1.  theta is a version counter: after round
q of step k it is (k - 1)(Q + 1) + q, after the serial step k(Q + 1).  A random scheduler interleaves every actor of
every rank, each rank at its own random speed.  Checked: no deadlock; every mix reads the neighbours' x_{q-1}, its own
x_{q-1} and x_{q-2}; every step reads x_Q; every consensus read sees version k(Q + 1) on every rank and no write lands during it.  Mutant: a round
kernel without its WAR guard must be caught."""
import random

import pytest


def run(R, Q, steps, seed, consensus=False, G=2, n_tiles=5, n_warps=2, D=1, war=True, max_ticks=800000):
    rng = random.Random(seed)
    iters = -(-n_tiles // G)
    slots_of = lambda r: [(r - 1) % R, (r + 1) % R]                      # slot 0 from the left, slot 1 from the right
    outs_of = lambda r: [((r + 1) % R, 0), ((r - 1) % R, 1)]            # out-slot j writes slot j of its peer
    z = lambda: [[0] * n_warps for _ in range(n_tiles)]
    theta, prev = [z() for _ in range(R)], [z() for _ in range(R)]
    reading = [[0] * n_tiles for _ in range(R)]
    rin, rflag, rack = [[z(), z()] for _ in range(R)], [[z(), z()] for _ in range(R)], [[0, 0] for _ in range(R)]
    rticket = [0] * R
    bar = [[[[0] * R for _ in range(G)] for _ in range(2)] for _ in range(R)]
    cons_ctr, cons_ticket = [0] * R, [0] * R
    V = lambda k, q: (k - 1) * (Q + 1) + q                              # theta's version after round q of step k
    bad = []

    def write_theta(r, t, w, val):
        if reading[r][t]:
            bad.append(("write under a read", r, t, val))
        theta[r][t][w] = val

    def round_warp(r, b, w, k, q):
        h = Q * (k - 1) + q
        want = V(k, q - 1)                                              # x_{q-1}: what every pushed / mixed slice holds
        if war:
            yield lambda: all(rack[r][j] >= h - 1 for j in range(2))
        for j in range(iters + D):
            t = b + j * G
            if j < iters and t < n_tiles:
                v = theta[r][t][w]
                if v != want:
                    bad.append(("push read", r, t, k, q, v))
                for p, s in outs_of(r):
                    rin[p][s][t][w] = v
                    yield None
                for p, s in outs_of(r):
                    rflag[p][s][t][w] = h
                yield None
            t2 = b + (j - D) * G
            if j >= D and t2 < n_tiles:
                yield lambda t2=t2: all(rflag[r][s][t2][w] >= h for s in range(2))
                for s in range(2):
                    if rin[r][s][t2][w] != want:
                        bad.append(("inbox", r, s, t2, k, q, rin[r][s][t2][w]))
                if theta[r][t2][w] != want:
                    bad.append(("own", r, t2, k, q, theta[r][t2][w]))
                if q >= 2 and prev[r][t2][w] != want - 1:
                    bad.append(("prev", r, t2, k, q, prev[r][t2][w]))
                if q < Q:
                    prev[r][t2][w] = want
                write_theta(r, t2, w, want + 1)
                yield None
        rticket[r] += 1
        if rticket[r] == G * n_warps * h:
            for s, sender in enumerate(slots_of(r)):
                rack[sender][s] = h
        yield None

    def step_warp(r, b, w, k):
        """The serial step: read x_Q, write theta_{k+1}; nothing crosses ranks."""
        for j in range(iters):
            t = b + j * G
            if t < n_tiles:
                if theta[r][t][w] != V(k, Q):
                    bad.append(("step read", r, t, k, theta[r][t][w]))
                yield None
                write_theta(r, t, w, V(k, Q) + 1)
                yield None

    def cons_cta(r, b, k):
        seq = cons_ctr[r] + 1               # read by every CTA at launch; only the launch's last CTA advances it

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
                if any(x != k * (Q + 1) for x in theta[p][t]):
                    bad.append(("consensus read", r, p, t, k, list(theta[p][t])))
                reading[p][t] -= 1
                yield None
        yield barrier(1)
        cons_ticket[r] += 1
        if cons_ticket[r] == G * seq:
            cons_ctr[r] = seq
        yield None

    def stream(r):
        for k in range(1, steps + 1):
            for q in range(1, Q + 1):
                yield [round_warp(r, b, w, k, q) for b in range(G) for w in range(n_warps)]
            yield [step_warp(r, b, w, k) for b in range(G) for w in range(n_warps)]
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

    # every rank runs at its own random speed, so one rank can fall far behind its peers within a step
    speed = [rng.choice([0.02, 0.2, 1.0]) for _ in range(R)]
    live = {r for r in range(R) if launch(r)}
    ticks = 0
    while live and ticks < max_ticks:
        ready = [(r, i) for r in live for i, (_, c) in enumerate(running[r]) if c is None or c()]
        if not ready:
            return "deadlock", bad
        r, i = rng.choices(ready, weights=[speed[x] for x, _ in ready])[0]
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
            if any(v != steps * (Q + 1) for row in theta[r] for v in row):
                bad.append(("final", r))
    return ("ok" if not live else "timeout"), bad


@pytest.mark.parametrize("consensus", [False, True])
@pytest.mark.parametrize("Q", [1, 2])
def test_cheb_rounds_then_serial_step_are_deadlock_free_and_read_what_they_should(Q, consensus):
    for seed in range(25):
        status, bad = run(3, Q, 4, seed, consensus=consensus)
        assert status == "ok", (status, seed)
        assert not bad, bad[:3]


@pytest.mark.parametrize("Q", [1, 2])
def test_mutant_without_the_round_war_guard_is_caught(Q):
    """A round that does not wait for its out-peers' acks of round h - 1 overwrites a round inbox a slow peer has not
    read yet; with no step handshake behind the rounds, that includes the next step's first round."""
    caught = sum(bool(run(3, Q, steps=3, seed=s, war=False)[1]) for s in range(60))
    assert caught > 0
