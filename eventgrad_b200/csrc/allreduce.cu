// eventgrad_b200 -- one-shot / two-shot all-reduce over peer-mapped memory fused with the
// 1/R scale and (cent) the SGD step (K4).  sm_90a.
//
// Replaces the per-tensor MPI_Allreduce(SUM) + grad/numranks + optimizer.step() of
// /root/reference/dmnist/cent/cent.cpp:130-145 and the final parameter averaging of
// /root/reference/dcifar10/event/event.cpp:509-519 with ONE launch over the whole arena.
//
//   one-shot : every rank loads tile t from all R ranks (rank order -> bit-identical result
//              on every rank), scales, applies SGD.  Traffic (R-1)N in; latency-optimal for
//              small arenas (the 407 KB MLP).
//   two-shot : tile t has an owner; the owner reduces it and stores the average into every
//              rank's buffer (reduce-scatter + all-gather in one kernel), then each rank runs
//              SGD on its own copy.  Traffic 2(R-1)N/R; bandwidth-optimal for large arenas.
//
// Cross-rank barriers are per CTA index (CTA b of every rank handles the same tile set), built
// from monotonically increasing release/acquire flags in peer-mapped memory.
//
// Compiled twice: as allreduce.cu (above), and from csrc/allreduce_nvls.cu with EG_NVLS defined, which
// builds the EXPERIMENTAL NVLink-SHARP variant `allreduce_nvls_kernel`: the tile owner reduces with ONE
// `multimem.ld_reduce` on the multicast address (the NVSwitch adds the R copies) and broadcasts the average
// with ONE `multimem.st` -- 2N/R bytes per GPU through the switch instead of 2(R-1)N/R over peer loads.
#include "api.h"
#include "common.cuh"

#ifdef EG_NVLS
#define EG_AR_SYM(name) name##_nvls
#else
#define EG_AR_SYM(name) name
#endif

namespace egb {

// phase-barrier among the CTAs with index b on all ranks
__device__ __forceinline__ void cta_barrier_all_ranks(const AllReduceParams& p, int phase, int b, int G,
                                                      uint32_t seq) {
  __syncthreads();
  const int tid = threadIdx.x;
  if (tid < p.world) {
    fence_sys();
    uint32_t* remote = p.peer_flags[tid] + ((size_t)phase * G + b) * p.world + p.rank;
    st_release_sys(remote, seq);
    wait_ge(p.flags + ((size_t)phase * G + b) * p.world + tid, seq, p.status, p.timeout_ns);
  }
  __syncthreads();
}

template <bool kMom>
__device__ __forceinline__ void sgd_tile(const AllReduceParams& p, size_t base, const F8& g, float lr) {
  F8 th = ld_f8(p.theta + base);
  F8 m;
  if (kMom) m = ld_f8(p.mom + base);
#pragma unroll
  for (int e = 0; e < 8; ++e) th.v[e] = sgd_elem<kMom>(th.v[e], g.v[e], m.v[e], lr, p.mu, p.wd, p.nesterov);
  if (kMom) st_f8(p.mom + base, m);
  st_f8(p.theta + base, th);
  if (p.shadow != nullptr) st_bf16x8(p.shadow + base, th);
}

__device__ __forceinline__ F8 reduce_tile(const AllReduceParams& p, size_t base) {
  F8 acc = ld_f8_cg(p.peer_bufs[0] + base);
  for (int r = 1; r < p.world; ++r) {
    const F8 x = ld_f8_cg(p.peer_bufs[r] + base);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc.v[e] = __fadd_rn(acc.v[e], x.v[e]);
  }
  const float w = (float)p.world;
#pragma unroll
  for (int e = 0; e < 8; ++e) acc.v[e] = __fdiv_rn(acc.v[e], w);   // grad / numranks (cent.cpp:140)
  return acc;
}

#ifdef EG_NVLS
// sum over all ranks' copies of the 8 floats at multicast address `mc` (in-switch reduction), / world
__device__ __forceinline__ F8 nvls_reduce_tile(const float* mc, float world) {
  F8 a;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(a.v[0]), "=f"(a.v[1]), "=f"(a.v[2]), "=f"(a.v[3])
               : "l"(mc)
               : "memory");
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(a.v[4]), "=f"(a.v[5]), "=f"(a.v[6]), "=f"(a.v[7])
               : "l"(mc + 4)
               : "memory");
#pragma unroll
  for (int e = 0; e < 8; ++e) a.v[e] = __fdiv_rn(a.v[e], world);
  return a;
}
// one store, delivered to every rank's copy by the switch
__device__ __forceinline__ void nvls_broadcast_tile(float* mc, const F8& a) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(a.v[0]), "f"(a.v[1]),
               "f"(a.v[2]), "f"(a.v[3])
               : "memory");
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc + 4), "f"(a.v[4]), "f"(a.v[5]),
               "f"(a.v[6]), "f"(a.v[7])
               : "memory");
}
#endif

template <bool kMom>
__global__ void __launch_bounds__(EG_THREADS, 4) EG_AR_SYM(allreduce_kernel)(const AllReduceParams p) {
  const int b = blockIdx.x, G = gridDim.x, tid = threadIdx.x;
  // step gate (--global-avg-period): not an averaging step -> no barrier, no load, no store, no counter; uniform over
  // the grid and, through the equal pass counters, over the ranks (PROTOCOL.md 1.11)
  if (p.gate_period > 0 && (*p.gate_pass + 1) % p.gate_period != 0) return;
  const uint32_t seq = (uint32_t)(*p.step_ctr) + 1u;
  // SGD mode: training step of this launch (the rank's device pass counter, advanced in the tail below)
  const int step = (p.pass_num != nullptr) ? *p.pass_num + 1 : 0;
  const float lr = sched_lr(p.lr_table, p.lr_len, p.lr, step);
  F8 zero;
#pragma unroll
  for (int e = 0; e < 8; ++e) zero.v[e] = 0.f;

  // start: every rank's buffer is final (its producer kernels precede this launch in-stream)
  cta_barrier_all_ranks(p, 0, b, G, seq);

  if (!p.two_shot) {
    for (int t = b; t < p.n_tiles; t += G) {
      const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
      const F8 g = reduce_tile(p, base);
      if (p.mode == 1) sgd_tile<kMom>(p, base, g, lr);
    }
    // nobody may overwrite (or zero) its buffer while a peer is still reading it
    cta_barrier_all_ranks(p, 2, b, G, seq);
    if (p.zero_after)
      for (int t = b; t < p.n_tiles; t += G)
        st_f8(p.local + (size_t)t * EG_TILE + (size_t)tid * EG_VEC, zero);
  } else {
    int j = 0;
    for (int t = b; t < p.n_tiles; t += G, ++j) {
      if ((b + j) % p.world != p.rank) continue;          // tile owner
      const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
#ifdef EG_NVLS
      nvls_broadcast_tile(p.mc_local + base, nvls_reduce_tile(p.mc_local + base, (float)p.world));
#else
      const F8 g = reduce_tile(p, base);
      for (int r = 0; r < p.world; ++r) st_f8(p.peer_bufs[r] + base, g);   // broadcast the average
#endif
    }
    cta_barrier_all_ranks(p, 1, b, G, seq);               // all owners of my tile set have stored
    if (p.mode == 1) {
      for (int t = b; t < p.n_tiles; t += G) {
        const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
        const F8 g = ld_f8_cg(p.local + base);
        sgd_tile<kMom>(p, base, g, lr);
        if (p.zero_after) st_f8(p.local + base, zero);
      }
    }
  }
  // bump the launch counter (and, in SGD mode, the pass counter) once per grid: every CTA has read both before
  // its ticket
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(p.ticket, 1u);
    if (prev == gridDim.x - 1) {
      *p.ticket = 0u;
      *p.step_ctr = (int)seq;
      if (p.pass_num != nullptr) *p.pass_num = step;
    }
  }
}

#ifndef EG_NVLS
// SlowMo sync (--slowmo-period tau): the gated two-shot average of theta, then the outer heavy-ball update of the
// identical x and u on every rank, one persistent launch.  Every op is an fp32 round-to-nearest intrinsic, so nothing
// is contracted and parallel/trigger.py:slowmo_sync_ reproduces it bit for bit.
__global__ void __launch_bounds__(EG_THREADS, 4) slowmo_sync_kernel(const SlowMoParams p) {
  const int b = blockIdx.x, G = gridDim.x, tid = threadIdx.x;
  // step gate: not a sync step -> no barrier, no load, no store, no counter (PROTOCOL.md 1.11, 1.13)
  const int step = *p.gate_pass + 1;
  if (step % p.gate_period != 0) return;
  const uint32_t seq = (uint32_t)(*p.step_ctr) + 1u;
  const float lr = sched_lr(p.lr_table, p.lr_len, p.lr, step);
  const float c = __fmul_rn(p.alpha, lr);

  cta_barrier_all_ranks(p, 0, b, G, seq);                 // every rank's theta is final
  int j = 0;
  for (int t = b; t < p.n_tiles; t += G, ++j) {
    if ((b + j) % p.world != p.rank) continue;            // tile owner
    const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
    const F8 avg = reduce_tile(p, base);
    for (int r = 0; r < p.world; ++r) st_f8(p.peer_bufs[r] + base, avg);
  }
  // every owner has stored theta_bar into my theta, and has finished reading my theta (its reads precede its arrival)
  cta_barrier_all_ranks(p, 1, b, G, seq);
  for (int t = b; t < p.n_tiles; t += G) {
    const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
    F8 x = ld_f8_cg(p.local + base);                      // theta_bar, stored by its owner
    if (lr != 0.f) {
      const F8 xo = ld_f8(p.x + base);
      F8 u = ld_f8(p.u + base);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float q = __fdiv_rn(__fsub_rn(xo.v[e], x.v[e]), lr);
        u.v[e] = __fadd_rn(__fmul_rn(p.beta, u.v[e]), q);
        x.v[e] = __fmaf_rn(u.v[e], -c, xo.v[e]);
      }
      st_f8(p.u + base, u);
    }
    st_f8(p.x + base, x);
    st_f8(p.local + base, x);
    if (p.shadow != nullptr) st_bf16x8(p.shadow + base, x);
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(p.ticket, 1u);
    if (prev == gridDim.x - 1) {
      *p.ticket = 0u;
      *p.step_ctr = (int)seq;
    }
  }
}

cudaError_t launch_slowmo_sync(const SlowMoParams& p, int grid, cudaStream_t s) {
  // the peer-load two-shot average only; tau >= 2 on a pass counter; beta in [0, 1), alpha > 0
  if (p.gate_period < 2 || p.gate_pass == nullptr || !p.two_shot || p.mode != 0 || p.x == nullptr ||
      p.u == nullptr || !(p.beta >= 0.f && p.beta < 1.f) || !(p.alpha > 0.f))
    return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_ALLREDUCE, 1);
  slowmo_sync_kernel<<<grid, EG_THREADS, 0, s>>>(p);
  return cudaGetLastError();
}

// Consensus distance (--consensus-every N): after step k with N dividing k, per tensor
// D_i = sum_r ||theta_r,i - theta_bar_i||^2 and A_i = ||theta_bar_i||^2, one persistent launch after the step kernel.
// theta is only read; the owner of a tile reads it from every rank twice (the mean, then the deviations), so no rank's
// copy is held in registers.  Every sum has a fixed order, so every rank and every run gets the same bits, and
// parallel/trigger.py:consensus_stats is the oracle (fp64 sums in another order: equal to rounding).
__global__ void __launch_bounds__(EG_THREADS, 4) consensus_kernel(const ConsensusParams p) {
  const int b = blockIdx.x, G = gridDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // step gate: not a measurement step -> no barrier, no load, no store, no counter (PROTOCOL.md 1.14)
  const int step = *p.gate_pass;
  if (step % p.gate_period != 0) return;
  const uint32_t seq = (uint32_t)(*p.step_ctr) + 1u;

  cta_barrier_all_ranks(p, 0, b, G, seq);                 // every rank's theta_k is final
  int j = 0;
  for (int t = b; t < p.n_tiles; t += G, ++j) {
    if ((b + j) % p.world != p.rank) continue;            // tile owner
    const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
    const F8 avg = reduce_tile(p, base);
    const int i = p.tile_tensor[t];
    // real elements of the tensor from `base` on (<= 0: all padding)
    const int lim = p.t_numel[i] - (t - p.t_tile_start[i]) * EG_TILE - tid * EG_VEC;
    double d = 0.0, a = 0.0;
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (e < lim) a = fma((double)avg.v[e], (double)avg.v[e], a);
    for (int r = 0; r < p.world; ++r) {
      const F8 x = ld_f8_cg(p.peer_bufs[r] + base);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (e < lim) {
          const double q = (double)x.v[e] - (double)avg.v[e];
          d = fma(q, q, d);
        }
    }
    d = warp_sum_d(d);
    a = warp_sum_d(a);
    if (lane == 0) {
      const size_t o = ((size_t)t * EG_WARPS + warp) * 2;
      for (int r = 0; r < p.world; ++r) {
        p.peer_part[r][o] = d;
        p.peer_part[r][o + 1] = a;
      }
    }
  }
  // every owner of my tile set has stored its partials into my buffer, and no peer reads my theta any more
  cta_barrier_all_ranks(p, 1, b, G, seq);
  __shared__ int s_last;
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(p.ticket, 1u) == (unsigned)G - 1u;
  }
  __syncthreads();
  if (!s_last) return;
  // last CTA: every CTA of this rank has passed barrier 1, so every partial has arrived.  Warp w reduces tensors
  // w, w + 8, ...: lane l sums the tensor's (tile, warp) partials l, l + 32, ..., then the butterfly
  __threadfence();
  const int row = *p.ring_ctr % p.cap;
  for (int i = warp; i < p.n_tensors; i += EG_WARPS) {
    const int lo = p.t_tile_start[i] * EG_WARPS, n = p.t_tile_count[i] * EG_WARPS;
    double d = 0.0, a = 0.0;
    for (int k = lane; k < n; k += 32) {
      d += __ldcg(p.part + (size_t)(lo + k) * 2);
      a += __ldcg(p.part + (size_t)(lo + k) * 2 + 1);
    }
    d = warp_sum_d(d);
    a = warp_sum_d(a);
    if (lane == 0) {
      p.ring[((size_t)row * p.n_tensors + i) * 2] = d;
      p.ring[((size_t)row * p.n_tensors + i) * 2 + 1] = a;
    }
  }
  __syncthreads();
  if (tid == 0) {
    p.ring_step[row] = step;
    *p.ring_ctr += 1;
    *p.ticket = 0u;
    *p.step_ctr = (int)seq;
  }
}

// Co-resident CTAs of the consensus kernel.  The occupancy query also loads the kernel: it is enqueued behind step
// kernels that spin on peer ranks, and a lazy load at its first launch could wait for those kernels to finish
int consensus_max_grid(int device) {
  int sms = 0, per_sm = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, consensus_kernel, EG_THREADS, 0);
  return sms * (per_sm < 1 ? 1 : per_sm);
}

cudaError_t launch_consensus(const ConsensusParams& p, int grid, cudaStream_t s) {
  // the peer-load two-shot tile ownership only; N >= 1 on a pass counter; the partial buffers, the ring and its
  // counters set; a ring of at least one row
  if (p.gate_period < 1 || p.gate_pass == nullptr || !p.two_shot || p.peer_part == nullptr || p.part == nullptr ||
      p.ring == nullptr || p.ring_step == nullptr || p.ring_ctr == nullptr || p.cap < 1 || p.tile_tensor == nullptr ||
      p.t_tile_start == nullptr || p.t_tile_count == nullptr || p.t_numel == nullptr || p.n_tensors < 1)
    return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_ALLREDUCE, 1);
  consensus_kernel<<<grid, EG_THREADS, 0, s>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_allreduce(const AllReduceParams& p, int grid, cudaStream_t s) {
  if (p.gate_period < 0 || (p.gate_period > 0 && p.gate_pass == nullptr)) return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_ALLREDUCE, 1);
  if (p.mode == 1 && p.mu != 0.f && p.mom != nullptr)
    allreduce_kernel<true><<<grid, EG_THREADS, 0, s>>>(p);
  else
    allreduce_kernel<false><<<grid, EG_THREADS, 0, s>>>(p);
  return cudaGetLastError();
}
#else
// two-shot only; p.mc_local = multicast mapping of `local` (torch symmetric memory, see parallel/window.py)
cudaError_t launch_allreduce_nvls(const AllReduceParams& p, int grid, cudaStream_t s) {
  eg_count_launch(EG_FAM_ALLREDUCE, 1);
  if (!p.two_shot || p.mc_local == nullptr) return cudaErrorInvalidValue;
  if (p.gate_period < 0 || (p.gate_period > 0 && p.gate_pass == nullptr)) return cudaErrorInvalidValue;
  if (p.mode == 1 && p.mu != 0.f && p.mom != nullptr)
    allreduce_kernel_nvls<true><<<grid, EG_THREADS, 0, s>>>(p);
  else
    allreduce_kernel_nvls<false><<<grid, EG_THREADS, 0, s>>>(p);
  return cudaGetLastError();
}
#endif

}  // namespace egb
