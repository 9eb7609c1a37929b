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
