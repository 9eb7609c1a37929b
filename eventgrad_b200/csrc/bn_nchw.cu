// eventgrad_b200 -- fused BatchNorm2d (+ residual add) (+ ReLU) for fp32 NCHW activations, training forward +
// backward.  sm_90a.
//
// Why a second layout: the headline runs at the reference's precision (IEEE fp32, event.cpp:279), and cuDNN's
// fp32 convolutions are NCHW kernels -- handed NHWC tensors they transpose around every conv.  So the fp32 path
// keeps activations NCHW and these kernels replace cuDNN's BN + ATen's add / ReLU (separate batch-norm forward,
// batch-norm backward and elementwise kernels) with the same 2 + 2 launch structure as csrc/bn_act.cu (NHWC, bf16 /
// fp32):
//   forward : stats kernel (per-channel sum / sum-of-squares, last CTA of a channel finalises mean, invstd and
//             the running statistics) -> apply kernel  y = relu(x * sc + sh (+ res))
//   backward: reduce kernel (dbeta = sum dz, dgamma = sum dz * xhat with dz = dy * (y > 0))
//             -> dx kernel  dx = gamma * invstd * (dz - dbeta/M - xhat * dgamma/M), dres = dz
// Geometry: channel c of image n is HW contiguous floats at ((n*C + c) * HW).  Reductions: grid (C, S); CTA (c, s)
// walks the float4 items of channel c assigned to split s.  Elementwise kernels: flat grid-stride over float4 items
// (every float4 lies inside one channel because HW % 4 == 0).
#include "api.h"
#include "common.cuh"

namespace egb {

#define BNC_THREADS 256

struct BncGeom {
  long long items;      // float4 items per channel = N * HW / 4
  int hw4;              // HW / 4
  int hw4_shift;        // log2(hw4) if hw4 is a power of two, else -1
  long long chw4;       // C * HW / 4  (float4 stride between images)
};

__device__ __forceinline__ long long bnc_addr4(const BncGeom& g, int c, long long item) {
  long long n, q;
  if (g.hw4_shift >= 0) {
    n = item >> g.hw4_shift;
    q = item & (long long)(g.hw4 - 1);
  } else {
    n = item / g.hw4;
    q = item - n * g.hw4;
  }
  return n * g.chw4 + (long long)c * g.hw4 + q;      // in float4 units
}

// block reduction of two per-thread floats; result valid in thread 0
__device__ __forceinline__ void bnc_block_sum2(float& a, float& b) {
  __shared__ float sa[BNC_THREADS / 32], sb[BNC_THREADS / 32];
  a = warp_sum(a);
  b = warp_sum(b);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) {
    sa[warp] = a;
    sb[warp] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float x = 0.f, y = 0.f;
#pragma unroll
    for (int w = 0; w < BNC_THREADS / 32; ++w) {
      x += sa[w];
      y += sb[w];
    }
    a = x;
    b = y;
  }
}

// last CTA of channel c combines the S partial pairs in fixed order, in double
__device__ __forceinline__ bool bnc_elect_and_combine(const BnParams& p, int c, int S, float a, float b, double* ta,
                                                      double* tb) {
  __shared__ int s_last;
  float* part = p.partial + ((size_t)c * S + blockIdx.y) * 2;
  if (threadIdx.x == 0) {
    part[0] = a;
    part[1] = b;
    __threadfence();
    const unsigned prev = atomicAdd(p.ticket + c, 1u);
    s_last = (prev == (unsigned)S - 1) ? 1 : 0;
    if (s_last) p.ticket[c] = 0u;
  }
  __syncthreads();
  if (!s_last) return false;
  if (threadIdx.x == 0) {
    __threadfence();
    double x = 0.0, y = 0.0;
    const float* base = p.partial + (size_t)c * S * 2;
    for (int s = 0; s < S; ++s) {
      x += (double)__ldcg(base + 2 * s);
      y += (double)__ldcg(base + 2 * s + 1);
    }
    *ta = x;
    *tb = y;
  }
  return true;    // totals valid in thread 0 only
}

// ------------------------------------------------------------------------------------------------ forward
__global__ void __launch_bounds__(BNC_THREADS, 4) bnc_fwd_stats_kernel(const BnParams p, const BncGeom g) {
  const int c = blockIdx.x, S = gridDim.y;
  const float4* x4 = reinterpret_cast<const float4*>(p.x);
  float s = 0.f, q = 0.f;
  const long long stride = (long long)S * BNC_THREADS;
  long long it = (long long)blockIdx.y * BNC_THREADS + threadIdx.x;
  for (; it + 3 * stride < g.items; it += 4 * stride) {        // 4 x 16 B in flight per thread
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = __ldg(x4 + bnc_addr4(g, c, it + u * stride));
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      s += (v[u].x + v[u].y) + (v[u].z + v[u].w);
      q = fmaf(v[u].x, v[u].x, q); q = fmaf(v[u].y, v[u].y, q); q = fmaf(v[u].z, v[u].z, q); q = fmaf(v[u].w, v[u].w, q);
    }
  }
  for (; it < g.items; it += stride) {
    const float4 v = __ldg(x4 + bnc_addr4(g, c, it));
    s += (v.x + v.y) + (v.z + v.w);
    q = fmaf(v.x, v.x, q); q = fmaf(v.y, v.y, q); q = fmaf(v.z, v.z, q); q = fmaf(v.w, v.w, q);
  }
  bnc_block_sum2(s, q);
  double ts, tq;
  if (!bnc_elect_and_combine(p, c, S, s, q, &ts, &tq)) return;
  if (threadIdx.x == 0) {
    const double invM = 1.0 / (double)p.M;
    const double mean = ts * invM;
    double var = tq * invM - mean * mean;      // biased
    if (var < 0.0) var = 0.0;
    p.mean[c] = (float)mean;
    p.invstd[c] = rsqrtf((float)var + p.eps);
    if (p.run_mean != nullptr) {
      const double unb = p.M > 1 ? var * (double)p.M / (double)(p.M - 1) : var;
      p.run_mean[c] = (float)((1.0 - p.momentum) * (double)p.run_mean[c] + p.momentum * mean);
      p.run_var[c] = (float)((1.0 - p.momentum) * (double)p.run_var[c] + p.momentum * unb);
    }
    if (c == 0 && p.nbt != nullptr) *p.nbt += 1;
  }
}

__global__ void __launch_bounds__(BNC_THREADS, 4) bnc_fwd_apply_kernel(const BnParams p, const BncGeom g, long long total4) {
  const float4* x4 = reinterpret_cast<const float4*>(p.x);
  const float4* r4 = reinterpret_cast<const float4*>(p.res);
  float4* y4 = reinterpret_cast<float4*>(p.y);
  const long long stride = (long long)gridDim.x * BNC_THREADS;
  for (long long i = (long long)blockIdx.x * BNC_THREADS + threadIdx.x; i < total4; i += 2 * stride) {
    float4 v[2], r[2];
    int ch[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long long j = i + u * stride;
      if (j < total4) {
        v[u] = __ldg(x4 + j);
        if (r4 != nullptr) r[u] = __ldg(r4 + j);
        ch[u] = (int)((g.hw4_shift >= 0 ? (j >> g.hw4_shift) : (j / g.hw4)) % p.C);
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long long j = i + u * stride;
      if (j >= total4) continue;
      const float sc = __ldg(p.gamma + ch[u]) * __ldg(p.invstd + ch[u]);
      const float sh = __ldg(p.beta + ch[u]) - __ldg(p.mean + ch[u]) * sc;
      float4 o;
      o.x = fmaf(v[u].x, sc, sh); o.y = fmaf(v[u].y, sc, sh); o.z = fmaf(v[u].z, sc, sh); o.w = fmaf(v[u].w, sc, sh);
      if (r4 != nullptr) { o.x += r[u].x; o.y += r[u].y; o.z += r[u].z; o.w += r[u].w; }
      if (p.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
      y4[j] = o;
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward
__global__ void __launch_bounds__(BNC_THREADS, 3) bnc_bwd_reduce_kernel(const BnParams p, const BncGeom g) {
  const int c = blockIdx.x, S = gridDim.y;
  const float4* x4 = reinterpret_cast<const float4*>(p.x);
  const float4* y4 = reinterpret_cast<const float4*>(p.y);
  const float4* d4 = reinterpret_cast<const float4*>(p.dy);
  const float mu = p.mean[c], is = p.invstd[c];
  float s1 = 0.f, s2 = 0.f;
  const long long stride = (long long)S * BNC_THREADS;
  for (long long it = (long long)blockIdx.y * BNC_THREADS + threadIdx.x; it < g.items; it += 2 * stride) {
    float4 d[2], x[2], y[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long long j = it + u * stride;
      if (j < g.items) {
        const long long a = bnc_addr4(g, c, j);
        d[u] = __ldg(d4 + a);
        x[u] = __ldg(x4 + a);
        if (p.relu) y[u] = __ldg(y4 + a);
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (it + u * stride >= g.items) continue;
      float dz0 = d[u].x, dz1 = d[u].y, dz2 = d[u].z, dz3 = d[u].w;
      if (p.relu) {
        if (!(y[u].x > 0.f)) dz0 = 0.f;
        if (!(y[u].y > 0.f)) dz1 = 0.f;
        if (!(y[u].z > 0.f)) dz2 = 0.f;
        if (!(y[u].w > 0.f)) dz3 = 0.f;
      }
      s1 += (dz0 + dz1) + (dz2 + dz3);
      s2 = fmaf(dz0, (x[u].x - mu) * is, s2); s2 = fmaf(dz1, (x[u].y - mu) * is, s2);
      s2 = fmaf(dz2, (x[u].z - mu) * is, s2); s2 = fmaf(dz3, (x[u].w - mu) * is, s2);
    }
  }
  bnc_block_sum2(s1, s2);
  double t1, t2;
  if (!bnc_elect_and_combine(p, c, S, s1, s2, &t1, &t2)) return;
  if (threadIdx.x == 0) {
    p.dbeta[c] = (float)t1;
    p.dgamma[c] = (float)t2;
  }
}

__global__ void __launch_bounds__(BNC_THREADS, 3) bnc_bwd_dx_kernel(const BnParams p, const BncGeom g, long long total4) {
  const float4* x4 = reinterpret_cast<const float4*>(p.x);
  const float4* y4 = reinterpret_cast<const float4*>(p.y);
  const float4* d4 = reinterpret_cast<const float4*>(p.dy);
  float4* dx4 = reinterpret_cast<float4*>(p.dx);
  float4* dr4 = reinterpret_cast<float4*>(p.dres);
  const float invM = 1.f / (float)p.M;
  const long long stride = (long long)gridDim.x * BNC_THREADS;
  for (long long i = (long long)blockIdx.x * BNC_THREADS + threadIdx.x; i < total4; i += 2 * stride) {
    float4 d[2], x[2], y[2];
    int ch[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long long j = i + u * stride;
      if (j < total4) {
        d[u] = __ldg(d4 + j);
        x[u] = __ldg(x4 + j);
        if (p.relu) y[u] = __ldg(y4 + j);
        ch[u] = (int)((g.hw4_shift >= 0 ? (j >> g.hw4_shift) : (j / g.hw4)) % p.C);
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long long j = i + u * stride;
      if (j >= total4) continue;
      const float mu = __ldg(p.mean + ch[u]), is = __ldg(p.invstd + ch[u]);
      const float k0 = __ldg(p.gamma + ch[u]) * is;
      const float k1 = __ldcg(p.dbeta + ch[u]) * invM, k2 = __ldcg(p.dgamma + ch[u]) * invM;
      float4 dz = d[u];
      if (p.relu) {
        if (!(y[u].x > 0.f)) dz.x = 0.f;
        if (!(y[u].y > 0.f)) dz.y = 0.f;
        if (!(y[u].z > 0.f)) dz.z = 0.f;
        if (!(y[u].w > 0.f)) dz.w = 0.f;
      }
      float4 o;
      o.x = k0 * (dz.x - k1 - (x[u].x - mu) * is * k2);
      o.y = k0 * (dz.y - k1 - (x[u].y - mu) * is * k2);
      o.z = k0 * (dz.z - k1 - (x[u].z - mu) * is * k2);
      o.w = k0 * (dz.w - k1 - (x[u].w - mu) * is * k2);
      dx4[j] = o;
      if (dr4 != nullptr) dr4[j] = dz;
    }
  }
}

// ------------------------------------------------------------------------------------------------ launcher
static inline long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

// p.M = N*H*W rows per channel, p.C channels, `hw` = H*W (multiple of 4); workspace: partial >= C * S * 2 floats
// (S <= 64), ticket >= C words.  which: 0 training forward, 1 apply only (eval), 2 backward.
cudaError_t launch_bn_nchw(const BnParams& p, int hw, int which, int sm_count, cudaStream_t s) {
  if (!p.fp32 || hw < 4 || hw % 4 != 0 || p.C < 1 || p.C > 2048 || p.M < 1 || p.M % hw != 0) return cudaErrorInvalidValue;
  BncGeom g;
  g.hw4 = hw / 4;
  g.items = p.M / 4;
  g.chw4 = (long long)p.C * g.hw4;
  g.hw4_shift = -1;
  if ((g.hw4 & (g.hw4 - 1)) == 0) {
    int sh = 0;
    while ((1 << sh) < g.hw4) ++sh;
    g.hw4_shift = sh;
  }
  const long long total4 = g.items * p.C;
  // reductions: ~8 float4 per thread per tensor, at most 64 splits, at least ~2 waves of CTAs when possible
  long long S = cdiv(g.items, (long long)BNC_THREADS * 8);
  const long long want = cdiv(2LL * sm_count * 4, p.C);
  if (S < want) S = want;
  const long long smax = cdiv(g.items, BNC_THREADS);
  if (S > smax) S = smax;
  if (S > 64) S = 64;
  if (S < 1) S = 1;
  long long eg = cdiv(total4, (long long)BNC_THREADS * 2);
  const long long cap = (long long)sm_count * 16;
  if (eg > cap) eg = cap;
  if (eg < 1) eg = 1;
  if (which == 0) {
    eg_count_launch(EG_FAM_BN, 2);
    bnc_fwd_stats_kernel<<<dim3((unsigned)p.C, (unsigned)S), BNC_THREADS, 0, s>>>(p, g);
    bnc_fwd_apply_kernel<<<(unsigned)eg, BNC_THREADS, 0, s>>>(p, g, total4);
  } else if (which == 1) {
    eg_count_launch(EG_FAM_BN, 1);
    bnc_fwd_apply_kernel<<<(unsigned)eg, BNC_THREADS, 0, s>>>(p, g, total4);
  } else if (which == 2) {
    eg_count_launch(EG_FAM_BN, 2);
    bnc_bwd_reduce_kernel<<<dim3((unsigned)p.C, (unsigned)S), BNC_THREADS, 0, s>>>(p, g);
    bnc_bwd_dx_kernel<<<(unsigned)eg, BNC_THREADS, 0, s>>>(p, g, total4);
  } else {
    return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace egb
