"""EventGraD trigger + adaptive threshold state machine -- specification oracle.

This is the vectorised (one lane per parameter tensor) PyTorch statement of the
per-tensor scalar logic in /root/reference/dmnist/event/event.cpp:325-392 and
/root/reference/dcifar10/event/event.cpp:300-365 (SURVEY.md A.1).  The CUDA kernels in
csrc/gossip.cu implement the same arithmetic on the device; tests compare them to this.

Arithmetic types mirror the reference: all state is fp32 (`calloc(sz, 4)`), the slope
average is accumulated in double (`auto slope_avg = 0.0`) and rounded to fp32 when it
becomes the new threshold.

Two trigger metrics (TriggerConfig.metric):
  norm   the reference rule (quirk Q2): fire when | ||theta_i|| - ||theta_i at its last send|| | >= thres_i.  By the
         triangle inequality this only bounds what the receivers miss from below; a sign flip or a permutation never fires.
  drift  fire when ||theta_i - sent_i|| >= thres_i, where sent_i is what the receivers hold of tensor i (the value
         pushed at its last firing; spevent: the element-wise `prev`).  The FSM is unchanged except for its input:
         value_diff is the drift itself, and the slope / threshold history is computed from it.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

METRICS = ("norm", "drift")


@dataclass
class TriggerConfig:
    thres_type: int = 1          # 1 adaptive, 0 constant
    horizon: float = 1.0
    constant: float = 0.0
    sent_history: int = 2
    initial_comm_passes: int = 30
    metric: str = "norm"         # norm (reference: norm difference) | drift (||theta - sent||)

    @staticmethod
    def from_train(cfg) -> "TriggerConfig":
        return TriggerConfig(cfg.thres_type, cfg.horizon, cfg.constant,
                             cfg.sent_history, cfg.initial_comm_passes, getattr(cfg, "trigger", "norm"))


class TriggerState:
    """thres, last_norm, last_iter [sz]; slopes [sz, H]; all fp32, zero-initialised
    (event.cpp:202-220)."""

    def __init__(self, n_tensors: int, history: int = 2, device="cpu"):
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
        self.thres = z(n_tensors)
        self.last_norm = z(n_tensors)
        self.last_iter = z(n_tensors)
        self.slopes = z(n_tensors, history)

    def clone(self) -> "TriggerState":
        c = TriggerState.__new__(TriggerState)
        c.thres, c.last_norm = self.thres.clone(), self.last_norm.clone()
        c.last_iter, c.slopes = self.last_iter.clone(), self.slopes.clone()
        return c

    def state_dict(self):
        return {k: getattr(self, k).cpu().clone() for k in ("thres", "last_norm", "last_iter", "slopes")}

    def load_state_dict(self, sd):
        for k in ("thres", "last_norm", "last_iter", "slopes"):
            getattr(self, k).copy_(sd[k].to(getattr(self, k).device))


@torch.no_grad()
def trigger_step(state: TriggerState, curr_norm: torch.Tensor, pass_num: int,
                 cfg: TriggerConfig) -> torch.Tensor:
    """Advance the FSM one training step. Returns the boolean fire mask [sz].
    `curr_norm`: per-tensor ||theta|| (metric norm) or ||theta - sent|| (metric drift, drift_norms()).
    No host synchronisation: everything stays on curr_norm's device."""
    curr = curr_norm.to(torch.float32)
    if cfg.metric == "drift":
        value_diff = curr.clone()                                     # the drift is the distance itself
    else:
        value_diff = (curr - state.last_norm).abs()                   # fabs(float)
    iter_diff = torch.tensor(float(pass_num), dtype=torch.float32,
                             device=curr.device) - state.last_iter    # int - float -> float
    if cfg.thres_type == 1:
        state.thres.mul_(float(torch.tensor(cfg.horizon, dtype=torch.float32)))  # thres * (float)horizon
    else:
        state.thres.fill_(float(torch.tensor(cfg.constant, dtype=torch.float32)))
    fire = value_diff >= state.thres
    if pass_num < cfg.initial_comm_passes:
        fire = torch.ones_like(fire)
    new_slope = value_diff / iter_diff
    shifted = torch.cat([state.slopes[:, 1:], new_slope[:, None]], dim=1)
    avg = shifted.double().sum(dim=1) / float(cfg.sent_history)
    state.slopes.copy_(torch.where(fire[:, None], shifted, state.slopes))
    if cfg.thres_type == 1:
        state.thres.copy_(torch.where(fire, avg.float(), state.thres))
    state.last_norm.copy_(torch.where(fire, curr, state.last_norm))
    state.last_iter.copy_(torch.where(fire, torch.full_like(curr, float(pass_num)),
                                      state.last_iter))
    return fire


@torch.no_grad()
def drift_norms(theta: torch.Tensor, sent: torch.Tensor, offsets, numels) -> torch.Tensor:
    """Per-tensor ||theta_i - sent_i|| (fp32) of two flat arenas: the drift trigger's input."""
    d = theta - sent
    return torch.stack([torch.linalg.vector_norm(d[o:o + n]) for o, n in zip(offsets, numels)]).float()


# ---------------------------------------------------------------------------------
# Functional pieces of the per-step update, shared by the collective backends and the
# single-process simulator (the CUDA kernels fuse all of them).
# ---------------------------------------------------------------------------------
@torch.no_grad()
def mix3_(theta: torch.Tensor, left: torch.Tensor, right: torch.Tensor) -> torch.Tensor:
    """theta <- (theta + L + R)/3 exactly as add_, add_, div_(3)
    (/root/reference/dcifar10/event/event.cpp:459-461)."""
    return theta.add_(left).add_(right).div_(3)


@torch.no_grad()
def mixk_(theta: torch.Tensor, slots) -> torch.Tensor:
    """theta <- (((theta + s_0) + s_1) + ... + s_{n-1}) / (n+1): the circulant-graph mix (parallel/topology.py), one
    rounded add per inbox slot in slot order, then a true division.  mixk_(theta, [L, R]) == mix3_(theta, L, R)."""
    for s in slots:
        theta.add_(s)
    return theta.div_(len(slots) + 1)


@torch.no_grad()
def cheb_combine_(theta_mixed: torch.Tensor, x: torch.Tensor, x_prev: Optional[torch.Tensor], alpha: torch.Tensor,
                  omega: torch.Tensor) -> torch.Tensor:
    """One Chebyshev-accelerated gossip round (--gossip-accel chebyshev), given theta_mixed = w, the round's mix of x:
        theta_mixed <- (x + alpha * (w - x)) + omega * (x - x_prev)
    with alpha, omega 0-dim fp32 tensors (parallel/topology.py chebyshev_coefficients).  Separate rounded sub, mul and add
    calls in the kernel's order (csrc/gossip_rounds.cu: __fsub_rn, __fmul_rn, __fadd_rn), so nothing fuses into an FMA.
    x_prev None (round 1): the omega term is absent, not multiplied by zero."""
    out = x.add(torch.mul(alpha, theta_mixed.sub(x)))
    if x_prev is not None:
        out.add_(torch.mul(omega, x.sub(x_prev)))
    return theta_mixed.copy_(out)


@torch.no_grad()
def mix2_(theta: torch.Tensor, slot: torch.Tensor) -> torch.Tensor:
    """theta <- (theta + slot) / 2: the one-peer exponential graph's mix (parallel/topology.py OnePeerExp), one rounded
    add and a true division, as the kernel's __fdiv_rn(__fadd_rn(theta, s), 2.f)."""
    return theta.add_(slot).div_(2)


@torch.no_grad()
def rank_mean(thetas) -> torch.Tensor:
    """((theta_0 + theta_1) + ... + theta_{R-1}) / R as a new tensor: one rounded add per rank in rank order, then one
    true division -- reduce_tile of csrc/allreduce.cu, the average of --global-avg-period.  The divisor is a 0-dim
    tensor on the data's device, so CUDA divides instead of multiplying by a rounded 1/R."""
    acc = thetas[0].clone()
    for x in thetas[1:]:
        acc.add_(x)
    return acc.div_(torch.tensor(float(len(thetas)), dtype=acc.dtype, device=acc.device))


@torch.no_grad()
def sgd_(theta: torch.Tensor, grad: torch.Tensor, mom, lr: float, mu: float, wd: float = 0.0,
         nesterov: bool = False) -> None:
    """torch.optim.SGD step with dampening 0 (dcifar10/event/event.cpp:196-200; zero momentum buffer ==
    first-step clone), op for op as torch's single-tensor path, so the rounding is the same:
        d = grad + wd*theta  (wd != 0) ;  m = mu*m + d ;  d = d + mu*m (nesterov) or m ;  theta -= lr*d
    `grad` is not modified.  The reference uses wd = 0, nesterov = False (the defaults)."""
    d = grad.add(theta, alpha=wd) if wd != 0.0 else grad
    if mu != 0.0:
        mom.mul_(mu).add_(d)
        d = d.add(mom, alpha=mu) if nesterov else mom
    theta.add_(d, alpha=-lr)



@torch.no_grad()
def qg_sgd_(theta: torch.Tensor, theta_k: torch.Tensor, grad: torch.Tensor, mom: torch.Tensor, lr: float, mu: float,
            wd: float = 0.0, nesterov: bool = False) -> None:
    """Quasi-global momentum step (QG-DSGDm, Lin, Kong, Stich and Jaggi 2021), op for op as qg_sgd_elem of
    csrc/common.cuh.  `theta` holds the step's mix theta' of `theta_k` (theta_k itself when the step does not mix) and
    receives theta''; `mom` holds m_hat, which is built from the step's own displacement instead of the gradient:
        a = mu*m_hat ;  d = grad + wd*theta' (wd != 0) ;  m = a + d ;  s = d + mu*m (nesterov) or m ;
        theta'' = theta' - lr*s ;  lr != 0: m_hat = a + (1 - mu)*((theta_k - theta') / lr + s), else m_hat is kept
    (theta_k - theta'')/lr is written as mix displacement plus step direction, so lr*s is never subtracted back out of a
    rounded theta''.  1 - mu is formed in the tensors' dtype and the division takes a 0-dim tensor divisor, so CUDA
    divides instead of multiplying by a rounded 1/lr.  At a fixed point the displacement is zero and m_hat decays to 0:
    no 1/(1 - mu) amplification of the heterogeneity bias."""
    d = grad.add(theta, alpha=wd) if wd != 0.0 else grad
    a = mom.mul(mu)
    m = a.add(d)
    s = d.add(m, alpha=mu) if nesterov else m
    q = theta_k.sub(theta)
    theta.add_(s, alpha=-lr)
    if float(torch.tensor(lr, dtype=theta.dtype)) != 0.0:
        q.div_(torch.tensor(lr, dtype=q.dtype, device=q.device)).add_(s)
        c = float(torch.tensor(1.0, dtype=theta.dtype).sub_(mu))
        mom.copy_(a.add_(q.mul_(c)))

@torch.no_grad()
def slowmo_sync_(x: torch.Tensor, u: torch.Tensor, avg: torch.Tensor, lr: float, beta: float, alpha: float) -> None:
    """SlowMo's outer update at a sync step (Wang, Tantia, Ballas and Rabbat 2020), op for op as slowmo_sync_kernel of
    csrc/allreduce.cu.  `avg` is the exact average theta_bar of the ranks' parameters, `x` the outer iterate (where the
    cycle started) and `u` the slow momentum:
        lr != 0:  q = (x - avg) / lr ;  u = beta*u + q ;  x = x - (alpha*lr)*u  (one fma)        lr == 0:  x = avg
    lr, beta and alpha are rounded to the tensors' dtype once; alpha*lr is one rounded product, and the division takes a
    0-dim tensor divisor, so CUDA divides instead of multiplying by a rounded 1/lr.  The caller then sets theta <- x."""
    dt = x.dtype
    lr_t = torch.tensor(lr, dtype=dt)
    if float(lr_t) == 0.0:
        x.copy_(avg)
        return
    b = float(torch.tensor(beta, dtype=dt))
    c = float(torch.tensor(alpha, dtype=dt) * lr_t)
    q = x.sub(avg).div_(lr_t.to(x.device))
    u.mul_(b).add_(q)
    x.add_(u, alpha=-c)


@torch.no_grad()
def consensus_stats(thetas, table):
    """Per-tensor consensus statistics of the ranks' flat arenas `thetas` (--consensus-every), the oracle of
    consensus_kernel in csrc/allreduce.cu.  theta_bar = rank_mean(thetas) in the arenas' dtype (the average that
    Gossip-PGA forms); then, over the numel real elements of tensor i (padding excluded), in float64:
        D_i = sum_r ||theta_r,i - theta_bar_i||^2        A_i = ||theta_bar_i||^2
    Returns (D, A), float64 CPU tensors of length n_tensors."""
    avg = rank_mean(thetas).double()
    xs = [t.double() for t in thetas]
    D = torch.zeros(table.n_tensors, dtype=torch.float64)
    A = torch.zeros(table.n_tensors, dtype=torch.float64)
    for i, (o, n) in enumerate(zip(table.offsets, table.numels)):
        a = avg[o:o + n]
        A[i] = float(a.square().sum())
        D[i] = float(sum(x[o:o + n].sub(a).square().sum() for x in xs))
    return D, A


def consensus_values(D, A, world: int):
    """(distance, relative) of one measurement: distance = sqrt(sum_i D_i / R), relative = distance / sqrt(sum_i A_i),
    the consensus distance sqrt(mean_r ||theta_r - theta_bar||^2) / ||theta_bar||.  relative is 0 when every rank holds
    the zero vector."""
    dist = (float(sum(float(d) for d in D)) / world) ** 0.5
    norm = float(sum(float(a) for a in A)) ** 0.5
    return dist, (dist / norm if norm > 0.0 else (0.0 if dist == 0.0 else float("inf")))


Q8_BLOCK = 256          # elements per int8 scale: one warp's slice of a 2048-float tile (never straddles tensors)
COMPRESS = ("none", "int8", "sign")


def q8_msg_bytes(numel: int) -> int:
    """Logical bytes of one tensor's int8 message: one code per real element + one fp32 scale per block holding any."""
    return numel + 4 * (-(-numel // Q8_BLOCK))


@torch.no_grad()
def q8_encode(d: torch.Tensor):
    """int8 code of a padded flat arena d (length a multiple of Q8_BLOCK), one fp32 scale per block of Q8_BLOCK:
        a = max |d| ; s = a / 127 ; q = s == 0 ? 0 : clamp(rint(d / s), -127, 127)
    IEEE fp32 with round to nearest even throughout, so it matches the q8 step kernel (csrc/gossip.cu, EG_Q8) bit for
    bit.  Both divisions are tensor / tensor: a division by a Python scalar may become a multiply by its reciprocal.
    Returns (q int8 [n], s fp32 [n / Q8_BLOCK])."""
    b = d.reshape(-1, Q8_BLOCK).to(torch.float32)
    a = b.abs().amax(dim=1)
    s = a / torch.full_like(a, 127.0)
    zero = s == 0
    safe = torch.where(zero, torch.ones_like(s), s)
    q = torch.round(b / safe[:, None]).clamp_(-127.0, 127.0)
    q = torch.where(zero[:, None], torch.zeros_like(q), q)
    return q.to(torch.int8).reshape(-1), s


@torch.no_grad()
def q8_decode(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """deq = (float)q * s per block (one rounded multiply): the delta both ends add to prev / their replica."""
    return (q.reshape(-1, Q8_BLOCK).to(torch.float32) * s.reshape(-1, 1)).reshape(-1)


SIGN_LANES = 32         # a block is one warp: lane j holds elements 8j .. 8j + 7 and sends byte j of the block


def sign_msg_bytes(numel: int) -> int:
    """Logical bytes of one tensor's sign message: one bit per real element (rounded up to bytes) + one fp32 scale per
    block holding any."""
    return -(-numel // 8) + 4 * (-(-numel // Q8_BLOCK))


@torch.no_grad()
def sign_encode(d: torch.Tensor):
    """1-bit scaled-sign code of a padded flat arena d (length a multiple of Q8_BLOCK), one scale per block, bit for bit
    the sign path of the q8 step kernel (csrc/gossip.cu, EG_Q8):
        each lane sums its 8 values of |d| left to right; the warp adds a + shfl_xor(a, o) for o = 16, 8, 4, 2, 1 (every
        stage is commutative, so all lanes end with the same value); s = a / 256, a true division;
        bit e of lane j's byte is d_{8j+e} < 0 (+0, -0 and NaN give 0)
    Returns (bytes uint8 [n / 8], s [n / Q8_BLOCK]) in d's dtype (float32 on the wire; float64 for convergence
    studies).  Byte 32 b + j is lane j of block b."""
    b = d.reshape(-1, SIGN_LANES, 8)
    ab = b.abs()
    a = ab[:, :, 0].clone()
    for e in range(1, 8):
        a = a + ab[:, :, e]
    lane = torch.arange(SIGN_LANES, device=d.device)
    o = SIGN_LANES // 2
    while o:
        a = a + a[:, lane ^ o]
        o //= 2
    s = a[:, 0] / torch.full_like(a[:, 0], float(Q8_BLOCK))
    weights = torch.tensor([1 << e for e in range(8)], dtype=torch.int32, device=d.device)
    bits = ((b < 0).to(torch.int32) * weights).sum(dim=2).to(torch.uint8)
    return bits.reshape(-1), s


@torch.no_grad()
def sign_decode(bits: torch.Tensor, s: torch.Tensor, numel=None) -> torch.Tensor:
    """deq_e = bit_e ? -s : s per block, in s's dtype: the delta both ends add to prev / their replica (one rounded
    add each).  `numel`: the decoded span is one tensor's whole tiles, and the elements from `numel` on are its zero
    padding, which decodes to 0 (as in the kernel, which adds nothing there), so padding stays 0."""
    shifts = torch.arange(8, dtype=torch.int32, device=bits.device)
    neg = ((bits.to(torch.int32).reshape(-1, 1) >> shifts) & 1).bool().reshape(-1, Q8_BLOCK)
    sb = s.reshape(-1, 1).expand(-1, Q8_BLOCK)
    deq = torch.where(neg, -sb, sb).reshape(-1)
    if numel is not None:
        deq[numel:] = 0
    return deq


def codec_of(compress: str):
    """(encode(d), decode(code, scales, numel), msg_bytes(numel)) of a --compress codec other than none; decode takes the
    tensor's real element count (int8's padding codes are 0 already)."""
    if compress == "int8":
        return q8_encode, lambda q, s, numel=None: q8_decode(q, s), q8_msg_bytes
    if compress == "sign":
        return sign_encode, sign_decode, sign_msg_bytes
    raise ValueError(f"no codec for compress {compress!r}")


@torch.no_grad()
def choco_mix_(theta: torch.Tensor, prev: torch.Tensor, rep_l: torch.Tensor, rep_r: torch.Tensor,
               gamma: float) -> torch.Tensor:
    """CHOCO-SGD's consensus step (Koloskova, Stich and Jaggi 2019) on the ring, op for op as the q8 step kernel's
    CHOCO mix: t = ((prev + rep_l) + rep_r) / 3 ; theta <- theta + gamma * (t - prev).  `prev` is this rank's public
    copy after this step's push, rep_l / rep_r its replicas of the neighbours' after their deltas arrived.  gamma is
    rounded to theta's dtype once and the division takes a tensor divisor, so every operation is one IEEE rounding.
    Summed over the ranks, t - prev vanishes in exact arithmetic, so the average of theta is kept whatever the codec."""
    g = torch.tensor(gamma, dtype=theta.dtype, device=theta.device)
    t = prev.add(rep_l).add_(rep_r).div_(torch.tensor(3.0, dtype=theta.dtype, device=theta.device))
    return theta.add_(t.sub_(prev).mul_(g))


@torch.no_grad()
def topk_select(theta_flat: torch.Tensor, prev_flat: torch.Tensor, k: int):
    """k indices with the largest |theta - prev| (spevent.cpp:346-349). Ties are broken
    towards the LOWEST index (a deterministic refinement; torch.topk leaves it unspecified).
    Returns (values = theta[idx], idx int64) sorted by (diff desc, index asc)."""
    diff = (theta_flat - prev_flat).abs()
    _, order = torch.sort(diff, descending=True, stable=True)
    idx = order[:k]
    return theta_flat[idx], idx
