// eventgrad_b200 -- common device helpers (sm_90a).
//
// Conventions
//   * EG_TILE fp32 elements per tile; every tile belongs to exactly one parameter tensor
//     (parallel/arena.py pads tensors to whole tiles).  One CTA iteration = one tile:
//     256 threads x 8 floats, moved as two 128-bit LDG/STG (Hopper's widest global access).
//   * Peer memory is reached through CUDA-IPC mapped pointers: a plain st.global on such a
//     pointer travels over NVLink / NVSwitch into the neighbour's HBM.
//   * Cross-GPU ordering: data stores (weak) -> bar.sync -> one thread: fence.acq_rel.sys +
//     st.release.sys flag.  Consumer: ld.acquire.sys spin -> bar.sync -> ld.global.cg data
//     (L1 is bypassed for anything a peer may have written).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "api.h"   // EG_TILE, EG_THREADS
#define EG_WARPS (EG_THREADS / 32)
#define EG_VEC 8  // floats per thread per tile

namespace egb {

struct alignas(32) F8 {
  float v[8];
};

// ---------------------------------------------------------------- 8-float global access (2 x 128 bit)
__device__ __forceinline__ F8 ld_f8(const float* p) {  // default caching (local, private data)
  F8 r;
  asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3])
               : "l"(p));
  asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.v[4]), "=f"(r.v[5]), "=f"(r.v[6]), "=f"(r.v[7])
               : "l"(p + 4));
  return r;
}
// L2-only load: for buffers a peer GPU may be writing (inboxes, peer gradients).
__device__ __forceinline__ F8 ld_f8_cg(const float* p) {
  F8 r;
  asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3])
               : "l"(p));
  asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.v[4]), "=f"(r.v[5]), "=f"(r.v[6]), "=f"(r.v[7])
               : "l"(p + 4));
  return r;
}
__device__ __forceinline__ void st_f8(float* p, const F8& r) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(r.v[0]), "f"(r.v[1]), "f"(r.v[2]),
               "f"(r.v[3])
               : "memory");
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p + 4), "f"(r.v[4]), "f"(r.v[5]),
               "f"(r.v[6]), "f"(r.v[7])
               : "memory");
}
__device__ __forceinline__ void st_bf16x8(__nv_bfloat16* p, const F8& r) {
  __nv_bfloat162 a = __floats2bfloat162_rn(r.v[0], r.v[1]);
  __nv_bfloat162 b = __floats2bfloat162_rn(r.v[2], r.v[3]);
  __nv_bfloat162 c = __floats2bfloat162_rn(r.v[4], r.v[5]);
  __nv_bfloat162 d = __floats2bfloat162_rn(r.v[6], r.v[7]);
  uint4 u;
  u.x = *reinterpret_cast<uint32_t*>(&a);
  u.y = *reinterpret_cast<uint32_t*>(&b);
  u.z = *reinterpret_cast<uint32_t*>(&c);
  u.w = *reinterpret_cast<uint32_t*>(&d);
  *reinterpret_cast<uint4*>(p) = u;
}

// ---------------------------------------------------------------- system-scope signalling
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// status word values (sticky; host raises on non-zero)
enum : int { EG_OK = 0, EG_ERR_TIMEOUT = 1 };

// Spin until *flag >= want (monotonic step counters; no resets -> no ABA). One thread only.
// Returns false on timeout / if a previous kernel already timed out (sticky status): a wedged
// peer must never hang the GPU.
__device__ __forceinline__ bool wait_ge(const uint32_t* flag, uint32_t want, int* status,
                                        uint64_t timeout_ns) {
  if (ld_acquire_sys(flag) >= want) return true;
  if (*reinterpret_cast<volatile int*>(status) != EG_OK) return false;
  const uint64_t t0 = globaltimer_ns();
  unsigned backoff = 32;
  while (true) {
    if (ld_acquire_sys(flag) >= want) return true;
    __nanosleep(backoff);
    if (backoff < 1024) backoff <<= 1;
    if (globaltimer_ns() - t0 > timeout_ns) {
      atomicExch(status, EG_ERR_TIMEOUT);
      return false;
    }
  }
}

// ---------------------------------------------------------------- warp reductions
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------- optimizer (torch.optim.SGD, dampening 0)
// Learning rate of training step `step` (1-based): table[min(step-1, len-1)] (engine/lr_schedule.py), or the
// scalar lr when no table is set.  `step` comes from the device-resident pass counter, so a captured CUDA graph
// follows the schedule on every replay.
__device__ __forceinline__ float sched_lr(const float* table, int len, float lr, int step) {
  if (table == nullptr || len <= 0) return lr;
  const int i = step < 1 ? 0 : (step > len ? len - 1 : step - 1);
  return __ldg(table + i);
}

// One element of the update, rounded as torch.optim.SGD rounds it (parallel/trigger.py:sgd_ is the oracle):
//   d = wd != 0 ? fma(theta, wd, g) : g;   m = m*mu + d;   d = nesterov ? fma(m, mu, d) : m;   theta = fma(d, -lr, theta)
// wd == 0 and nesterov == 0 give exactly the plain heavy-ball step.  All branches are uniform across the grid.
template <bool kMom>
__device__ __forceinline__ float sgd_elem(float th, float g, float& m, float lr, float mu, float wd, int nesterov) {
  float d = (wd != 0.f) ? __fmaf_rn(th, wd, g) : g;
  if (kMom) {
    m = __fadd_rn(__fmul_rn(m, mu), d);
    d = nesterov ? __fmaf_rn(m, mu, d) : m;
  }
  return __fmaf_rn(d, -lr, th);
}

// Quasi-global momentum (QG-DSGDm, Lin et al. 2021; parallel/trigger.py:qg_sgd_ is the oracle).  `th` is the step's
// mix theta' of theta_k (theta_k when the step does not mix), `dk` = theta_k - theta' (rounded), `mh` the buffer m_hat,
// c = 1 - mu in fp32:
//   a = mu*m_hat;  d as sgd_elem;  m = a + d;  s = nesterov ? fma(m, mu, d) : m;  theta'' = fma(s, -lr, theta')
//   lr != 0: m_hat = a + c*((theta_k - theta') / lr + s), the step's own displacement (theta_k - theta'') / lr written as
//   mix displacement plus step direction, so lr*s is never subtracted back out of a rounded theta''
__device__ __forceinline__ float qg_sgd_elem(float dk, float th, float g, float& mh, float lr, float mu, float c,
                                             float wd, int nesterov) {
  const float a = __fmul_rn(mh, mu);
  const float d = (wd != 0.f) ? __fmaf_rn(th, wd, g) : g;
  const float m = __fadd_rn(a, d);
  const float s = nesterov ? __fmaf_rn(m, mu, d) : m;
  if (lr != 0.f) mh = __fadd_rn(a, __fmul_rn(c, __fadd_rn(__fdiv_rn(dk, lr), s)));
  return __fmaf_rn(s, -lr, th);
}
}  // namespace egb
