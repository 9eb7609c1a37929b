// eventgrad_b200 -- mix-only gossip rounds (--gossip-rounds Q, decent on the ring / a static circulant graph), sm_90a.
//
// One launch is one round q (1 <= q <= Q - 1) of step k = *pass_num + 1: every rank pushes its current theta into every
// out-slot's ROUND inbox, publishes one release flag per (tile, warp) and slot, waits for the flags of its own slots and
// mixes them into theta in place with the step's own mix:
//   theta <- (((theta + in_0) + in_1) + ... + in_{n-1}) / (n + 1)
// which is ((theta + L) + R) / 3 on the ring (slot 0 from the left, slot 1 from the right) and parallel/trigger.py mixk_
// on a static graph.  The Q - 1 launches run after backward and before the unchanged step kernel, which then pushes and
// mixes theta once more and takes the optimizer step: theta_{k+1} = SGD(W^Q theta_k, g_k).
//
// The rounds have their own inboxes, flags, acks and ticket (window sections appended last by parallel/p2p.py
// build_layout), so no step kernel, its layout or its protocol changes.  The handshake counter of round q of step k is
//   h = (Q - 1)(k - 1) + q,
// monotone per flag and per ack across rounds and steps, so one captured CUDA graph replays all Q - 1 launches.  The
// protocol mirrors the step kernel's (PROTOCOL.md 1.16): a WAR guard on the round acks of h - 1, the per-warp push /
// flag / wait / mix pipeline of depth group_iters, and the last CTA acking every slot's sender.  Every wait is bounded
// by timeout_ns and honours the sticky status word.  theta is the only non-handshake state it writes.
//
// gossip_round_cheb_kernel (--gossip-accel chebyshev) is the same round with one more stage after the mix: every one of
// the Q rounds is a launch (`rounds` = Q, so h = Q(k - 1) + q), and round q turns the mix w of x_{q-1} into
//   x_q = (x_{q-1} + alpha_q (w - x_{q-1})) + omega_q (x_{q-1} - x_{q-2})
// with separately rounded sub / mul / add (no FMA), keeping x_{q-2} in the local `prev` buffer.  The difference form
// keeps a consensus vector fixed whatever the fp32 rounding of the coefficients.  x_Q = P_Q(W) x_0, the Chebyshev
// polynomial of W's spectrum (parallel/topology.py chebyshev_coefficients); the step kernel then runs as the serial step.
// The handshake is the power round's word for word (PROTOCOL.md 1.18).
#include "api.h"
#include "common.cuh"

namespace egb {

// push this thread's 8 elements of theta into every out-slot (a null push pointer: the 2-rank ring's single copy)
__device__ __forceinline__ void round_push(const RoundParams& p, size_t base, const F8& th) {
#pragma unroll
  for (int k = 0; k < EG_MAX_SLOTS; ++k)
    if (k < p.n_slots && p.push[k] != nullptr) st_f8(p.push[k] + base, th);
}

// theta of this thread's 8 elements <- the step's mix of the round inboxes.  Slots are added in slot order, two at a
// time, as the graph step kernel does; then one true division by n_slots + 1
__device__ __forceinline__ void round_mix(const RoundParams& p, size_t base) {
  F8 th = ld_f8(p.theta + base);
#pragma unroll
  for (int s = 0; s < EG_MAX_SLOTS; s += 2) {
    if (s < p.n_slots) {
      const F8 A = ld_f8_cg(p.inbox[s] + base), B = ld_f8_cg(p.inbox[s + 1] + base);
#pragma unroll
      for (int e = 0; e < 8; ++e) th.v[e] = __fadd_rn(__fadd_rn(th.v[e], A.v[e]), B.v[e]);
    }
  }
  const float d = (float)(p.n_slots + 1);
#pragma unroll
  for (int e = 0; e < 8; ++e) th.v[e] = __fdiv_rn(th.v[e], d);
  st_f8(p.theta + base, th);
}

// the Chebyshev round on this thread's 8 elements: x = x_{q-1} is the theta it loads, w the mix above in round_mix's
// operand order; theta <- x_q, and prev <- x_{q-1} for q < Q.  Round 1 neither reads prev nor forms the omega term
__device__ __forceinline__ void round_mix_cheb(const RoundParams& p, const ChebParams& c, size_t base, int q,
                                               float alpha, float omega) {
  const F8 x = ld_f8(p.theta + base);
  F8 w = x;
#pragma unroll
  for (int s = 0; s < EG_MAX_SLOTS; s += 2) {
    if (s < p.n_slots) {
      const F8 A = ld_f8_cg(p.inbox[s] + base), B = ld_f8_cg(p.inbox[s + 1] + base);
#pragma unroll
      for (int e = 0; e < 8; ++e) w.v[e] = __fadd_rn(__fadd_rn(w.v[e], A.v[e]), B.v[e]);
    }
  }
  const float d = (float)(p.n_slots + 1);
  F8 y;
#pragma unroll
  for (int e = 0; e < 8; ++e)
    y.v[e] = __fadd_rn(x.v[e], __fmul_rn(alpha, __fsub_rn(__fdiv_rn(w.v[e], d), x.v[e])));
  if (q >= 2) {
    const F8 xp = ld_f8(c.prev + base);
#pragma unroll
    for (int e = 0; e < 8; ++e) y.v[e] = __fadd_rn(y.v[e], __fmul_rn(omega, __fsub_rn(x.v[e], xp.v[e])));
  }
  if (q < p.rounds) st_f8(c.prev + base, x);
  st_f8(p.theta + base, y);
}

template <bool kCheb>
__device__ __forceinline__ void round_body(const RoundParams& p, const ChebParams& c, int q) {
  const int b = blockIdx.x, G = gridDim.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t h = (uint32_t)(p.rounds * *p.pass_num + q);     // (Q - 1)(k - 1) + q with k = *pass_num + 1
  // sticky failure: a peer wait of this or an earlier launch timed out -- store nothing into a peer that may be wedged
  if (*reinterpret_cast<volatile int*>(p.status) != EG_OK) return;
  __shared__ int s_ok;
  if (tid == 0) {
    // WAR guard: every peer I push into has finished reading what I pushed into its round inbox at round h - 1
    bool ok = true;
#pragma unroll
    for (int k = 0; k < EG_MAX_SLOTS; ++k)
      if (k < p.n_slots) ok = wait_ge(p.ack_from[k], h - 1u, p.status, p.timeout_ns) && ok;
    s_ok = ok;
  }
  __syncthreads();
  if (!s_ok) return;
  const int n_tiles = p.n_tiles, D = p.group_iters;
  const int iters = (n_tiles + G - 1) / G;
  float alpha = 0.f, omega = 0.f;
  if constexpr (kCheb) {
    alpha = c.coef[2 * (q - 1)];
    omega = c.coef[2 * (q - 1) + 1];
  }
  for (int j = 0; j < iters + D; ++j) {
    const int t = b + j * G;
    if (j < iters && t < n_tiles) {
      const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
      round_push(p, base, ld_f8(p.theta + base));
      __syncwarp();
      if (lane == 0) {
        fence_sys();                               // my warp's stores are performed before the flags
#pragma unroll
        for (int k = 0; k < EG_MAX_SLOTS; ++k)
          if (k < p.n_slots) st_release_sys(p.flag_to[k] + (size_t)t * EG_WARPS + warp, h);
      }
    }
    const int t2 = b + (j - D) * G;
    if (j >= D && t2 < n_tiles) {
      if (lane == 0) {
#pragma unroll
        for (int s = 0; s < EG_MAX_SLOTS; ++s)
          if (s < p.n_slots) wait_ge(p.flag_from[s] + (size_t)t2 * EG_WARPS + warp, h, p.status, p.timeout_ns);
      }
      __syncwarp();
      if constexpr (kCheb)
        round_mix_cheb(p, c, (size_t)t2 * EG_TILE + (size_t)tid * EG_VEC, q, alpha, omega);
      else
        round_mix(p, (size_t)t2 * EG_TILE + (size_t)tid * EG_VEC);
    }
  }
  // the last CTA: every CTA of this rank has read its round inboxes for h -> ack every slot's sender
  __shared__ int s_last;
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(p.ticket, 1u) == (unsigned)G - 1u;
  }
  __syncthreads();
  if (s_last && tid == 0) {
    *p.ticket = 0u;
    fence_sys();
#pragma unroll
    for (int s = 0; s < EG_MAX_SLOTS; ++s)
      if (s < p.n_slots) st_release_sys(p.ack_to[s], h);
  }
}

__global__ void __launch_bounds__(EG_THREADS, 4) gossip_round_kernel(const RoundParams p, int q) {
  round_body<false>(p, ChebParams{nullptr, nullptr}, q);
}

__global__ void __launch_bounds__(EG_THREADS, 4) gossip_round_cheb_kernel(const RoundParams p, const ChebParams c,
                                                                          int q) {
  round_body<true>(p, c, q);
}

// the smaller of the power and Chebyshev instances' co-resident CTAs: one bound whichever the run launches
int gossip_rounds_max_grid(int device) {
  int sms = 0, a = 0, ac = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, gossip_round_kernel, EG_THREADS, 0);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ac, gossip_round_cheb_kernel, EG_THREADS, 0);
  if (ac < a) a = ac;
  if (a < 1) a = 1;
  return sms * a;
}

static bool round_params_ok(const RoundParams& p) {
  bool ok = p.theta && p.pass_num && p.ticket && p.status && p.rounds >= 1 && p.n_tiles > 0 && p.group_iters >= 0 &&
            p.n_slots >= 2 && p.n_slots <= EG_MAX_SLOTS && !(p.n_slots & 1);
  bool any_push = false;
  for (int k = 0; ok && k < p.n_slots; ++k) {
    ok = p.inbox[k] && p.flag_from[k] && p.flag_to[k] && p.ack_from[k] && p.ack_to[k];
    any_push = any_push || p.push[k] != nullptr;
  }
  return ok && any_push;
}

cudaError_t launch_gossip_rounds(const RoundParams& p, int grid, cudaStream_t s) {
  if (!round_params_ok(p)) return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_GOSSIP, p.rounds);
  for (int q = 1; q <= p.rounds; ++q) {
    gossip_round_kernel<<<grid, EG_THREADS, 0, s>>>(p, q);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t launch_gossip_rounds_cheb(const RoundParams& p, const ChebParams& c, int grid, cudaStream_t s) {
  if (!round_params_ok(p) || !c.prev || !c.coef) return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_GOSSIP, p.rounds);
  for (int q = 1; q <= p.rounds; ++q) {
    gossip_round_cheb_kernel<<<grid, EG_THREADS, 0, s>>>(p, c, q);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace egb
