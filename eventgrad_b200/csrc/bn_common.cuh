// eventgrad_b200 -- device helpers shared by the fused BatchNorm kernels (csrc/bn_act.cu, csrc/bn_act_v2.cu).
// Geometry: NHWC == row-major [M, C]; a CTA owns one 64-channel slice (blockIdx.x) and one row split
// (blockIdx.y); 8 threads x 8 channels (one 128-byte line) per row, 32 rows per pass.
#pragma once
#include "api.h"
#include "common.cuh"

namespace egb {

#define BN_THREADS 256
#define BN_RPP 32            // rows per pass (256 threads / 8 threads per row)
#define BN_SLICE 64          // channels per slice
#define BN_FWD_PASSES 8      // slab depth held in registers by the fused forward
#define BN_BWD_PASSES 4      // ... by the fused backward (3 tensors)

struct V8 {
  float v[8];
};
__device__ __forceinline__ V8 unpack_bf16x8(const uint4& u) {
  V8 r;
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    r.v[2 * i] = f.x;
    r.v[2 * i + 1] = f.y;
  }
  return r;
}
__device__ __forceinline__ uint4 pack_bf16x8(const V8& r) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(r.v[2 * i], r.v[2 * i + 1]);
  return u;
}
// fp32 -> three bf16 planes (x = a + b + c to 2^-24 |x|; both residuals are exact in fp32) for 8 values; `base` points at
// plane 0 of these 8 elements, the other planes are `plane` elements further (csrc/conv_tc.cu operand format)
__device__ __forceinline__ void store_planes8(const V8& x, __nv_bfloat16* base, size_t plane) {
  __nv_bfloat16 a[8], b[8], c[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    a[e] = __float2bfloat16_rn(x.v[e]);
    const float r1 = __fsub_rn(x.v[e], __bfloat162float(a[e]));
    b[e] = __float2bfloat16_rn(r1);
    c[e] = __float2bfloat16_rn(__fsub_rn(r1, __bfloat162float(b[e])));
  }
  *reinterpret_cast<uint4*>(base) = *reinterpret_cast<const uint4*>(a);
  *reinterpret_cast<uint4*>(base + plane) = *reinterpret_cast<const uint4*>(b);
  *reinterpret_cast<uint4*>(base + 2 * plane) = *reinterpret_cast<const uint4*>(c);
}
__device__ __forceinline__ uint4 ldg16(const __nv_bfloat16* p) { return *reinterpret_cast<const uint4*>(p); }
__device__ __forceinline__ void stg16(__nv_bfloat16* p, const uint4& u) { *reinterpret_cast<uint4*>(p) = u; }

// Element-type abstraction: Raw8<T> = 8 consecutive channels of one row as they sit in memory
// (bf16: one 16-byte word; fp32: two 16-byte words -- the reference's precision, event.cpp:279).
template <typename T> struct Raw8;
template <> struct Raw8<__nv_bfloat16> { uint4 u; };
template <> struct Raw8<float> { float4 a, b; };

__device__ __forceinline__ Raw8<__nv_bfloat16> ld8(const __nv_bfloat16* p) {
  Raw8<__nv_bfloat16> r; r.u = *reinterpret_cast<const uint4*>(p); return r;
}
__device__ __forceinline__ Raw8<float> ld8(const float* p) {
  Raw8<float> r;
  r.a = *reinterpret_cast<const float4*>(p);
  r.b = *reinterpret_cast<const float4*>(p + 4);
  return r;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const Raw8<__nv_bfloat16>& r) { *reinterpret_cast<uint4*>(p) = r.u; }
__device__ __forceinline__ void st8(float* p, const Raw8<float>& r) {
  *reinterpret_cast<float4*>(p) = r.a;
  *reinterpret_cast<float4*>(p + 4) = r.b;
}
__device__ __forceinline__ void zero8(Raw8<__nv_bfloat16>& r) { r.u = make_uint4(0, 0, 0, 0); }
__device__ __forceinline__ void zero8(Raw8<float>& r) { r.a = r.b = make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ V8 unpack8(const Raw8<__nv_bfloat16>& r) { return unpack_bf16x8(r.u); }
__device__ __forceinline__ V8 unpack8(const Raw8<float>& r) {
  V8 o;
  o.v[0] = r.a.x; o.v[1] = r.a.y; o.v[2] = r.a.z; o.v[3] = r.a.w;
  o.v[4] = r.b.x; o.v[5] = r.b.y; o.v[6] = r.b.z; o.v[7] = r.b.w;
  return o;
}
__device__ __forceinline__ void pack8(const V8& v, Raw8<__nv_bfloat16>& r) { r.u = pack_bf16x8(v); }
__device__ __forceinline__ void pack8(const V8& v, Raw8<float>& r) {
  r.a = make_float4(v.v[0], v.v[1], v.v[2], v.v[3]);
  r.b = make_float4(v.v[4], v.v[5], v.v[6], v.v[7]);
}
// d[e] = 0 where y[e] <= 0 (ReLU mask folded into the incoming gradient, done on the raw words)
__device__ __forceinline__ void mask_le0(Raw8<__nv_bfloat16>& d, const Raw8<__nv_bfloat16>& y) {
  const unsigned short* ys = reinterpret_cast<const unsigned short*>(&y.u);
  unsigned short* ds = reinterpret_cast<unsigned short*>(&d.u);
#pragma unroll
  for (int e = 0; e < 8; ++e)
    if ((ys[e] & 0x8000u) || (ys[e] & 0x7fffu) == 0u) ds[e] = 0;   // bf16 sign / zero test
}
__device__ __forceinline__ void mask_le0(Raw8<float>& d, const Raw8<float>& y) {
  if (!(y.a.x > 0.f)) d.a.x = 0.f;
  if (!(y.a.y > 0.f)) d.a.y = 0.f;
  if (!(y.a.z > 0.f)) d.a.z = 0.f;
  if (!(y.a.w > 0.f)) d.a.w = 0.f;
  if (!(y.b.x > 0.f)) d.b.x = 0.f;
  if (!(y.b.y > 0.f)) d.b.y = 0.f;
  if (!(y.b.z > 0.f)) d.b.z = 0.f;
  if (!(y.b.w > 0.f)) d.b.w = 0.f;
}

// ReLU mask sources of the split backward kernels (BnParams::mask_mode)
#define BN_MASK_Y 0
#define BN_MASK_X 1
#define BN_MASK_BITS 2

// y = fmaf(x, sc, sh) (+ residual): the forward apply kernel and the "mask from x" backward share this expression, so
// the backward's fmaf(x, sc, sh) > 0 is bit for bit the forward's decision
__device__ __forceinline__ void bn_affine(const BnParams& p, int c, float& sc, float& sh) {
  sc = p.gamma[c] * p.invstd[c];
  sh = p.beta[c] - p.mean[c] * sc;
}

// ReLU mask of 8 channels as bits (bit e = channel e), from whichever source p.mask_mode names
template <typename T>
__device__ __forceinline__ unsigned relu_bits(const BnParams& p, const Raw8<T>& yr, unsigned char mb, const V8& x,
                                              const float (&sc)[8], const float (&sh)[8]) {
  if (p.mask_mode == BN_MASK_BITS) return mb;
  unsigned m = 0u;
  if (p.mask_mode == BN_MASK_X) {
#pragma unroll
    for (int e = 0; e < 8; ++e) m |= (fmaf(x.v[e], sc[e], sh[e]) > 0.f ? 1u : 0u) << e;
  } else {
    const V8 y = unpack8(yr);
#pragma unroll
    for (int e = 0; e < 8; ++e) m |= (y.v[e] > 0.f ? 1u : 0u) << e;
  }
  return m;
}

// -------------------------------------------------------------------------------------------
// Reduce the per-thread 2x8 accumulators over the 32 row lanes, write this CTA's partial row
// [128] = {sum a[64] | sum b[64]} for its slice.
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ void block_partials(const float (&a)[8], const float (&b)[8], float* smem /*[32][128]*/,
                                               int tx, int ty, float* partial_row) {
  float* row = smem + ty * 128;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    row[tx * 8 + e] = a[e];
    row[64 + tx * 8 + e] = b[e];
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    float s = 0.f;
#pragma unroll 8
    for (int r = 0; r < BN_RPP; ++r) s += smem[r * 128 + threadIdx.x];
    partial_row[threadIdx.x] = s;
  }
}

// Last CTA of a slice: tot[c] = sum_r partial[r][c], fixed order, double.  256 threads = 32 float4
// columns x 8 row lanes, 8 loads in flight each; lanes folded through smem (8 x 128 doubles).
__device__ __forceinline__ void slice_combine(const float* partial, int nrows, double* sm /*[8][128]*/) {
  const int col = threadIdx.x & 31, bl = threadIdx.x >> 5;
  const float4* p4 = reinterpret_cast<const float4*>(partial) + col;
  double a0 = 0, a1 = 0, a2 = 0, a3 = 0;
  int r = bl;
  for (; r + 56 < nrows; r += 64) {
    float4 x[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) x[u] = __ldcg(p4 + (size_t)(r + 8 * u) * 32);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      a0 += (double)x[u].x; a1 += (double)x[u].y; a2 += (double)x[u].z; a3 += (double)x[u].w;
    }
  }
  for (; r < nrows; r += 8) {
    const float4 x0 = __ldcg(p4 + (size_t)r * 32);
    a0 += (double)x0.x; a1 += (double)x0.y; a2 += (double)x0.z; a3 += (double)x0.w;
  }
  __syncthreads();                                        // smem is being re-purposed
  double* dst = sm + bl * 128 + col * 4;
  dst[0] = a0; dst[1] = a1; dst[2] = a2; dst[3] = a3;
  __syncthreads();
  if (threadIdx.x < 128) {
    double t = sm[threadIdx.x];
#pragma unroll
    for (int l = 1; l < 8; ++l) t += sm[l * 128 + threadIdx.x];
    sm[threadIdx.x] = t;                                  // row 0 = totals
  }
  __syncthreads();
}

__device__ __forceinline__ bool elect_last_of_slice(unsigned int* ticket, unsigned int n) {
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(ticket, 1u);
    s_last = (prev == n - 1) ? 1 : 0;
    if (s_last) *ticket = 0u;
  }
  __syncthreads();
  if (s_last) __threadfence();
  return s_last != 0;
}

// mean / invstd / running stats for one slice from its totals (tot[0..63] = sum x, [64..127] = sum x^2)
__device__ __forceinline__ void finalize_stats(const BnParams& p, int slice, const double* tot) {
  if (threadIdx.x < BN_SLICE) {
    const int c = slice * BN_SLICE + threadIdx.x;
    const double invM = 1.0 / (double)p.M;
    const double mean = tot[threadIdx.x] * invM;
    double var = tot[64 + threadIdx.x] * invM - mean * mean;   // biased
    if (var < 0.0) var = 0.0;
    p.mean[c] = (float)mean;
    p.invstd[c] = rsqrtf((float)var + p.eps);
    if (p.run_mean != nullptr) {
      const double unb = p.M > 1 ? var * (double)p.M / (double)(p.M - 1) : var;
      p.run_mean[c] = (float)((1.0 - p.momentum) * (double)p.run_mean[c] + p.momentum * mean);
      p.run_var[c] = (float)((1.0 - p.momentum) * (double)p.run_var[c] + p.momentum * unb);
    }
  }
  if (threadIdx.x == 0 && slice == 0 && p.nbt != nullptr) *p.nbt += 1;
}

// epoch flag: slice-last CTA publishes, everyone else of the slice spins (bounded)
__device__ __forceinline__ void publish_flag(unsigned int* flag, unsigned int value) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flag), "r"(value) : "memory");
  }
}
__device__ __forceinline__ void wait_flag(const unsigned int* flag, unsigned int value, int* status) {
  if (threadIdx.x == 0) {
    const uint64_t t0 = globaltimer_ns();
    unsigned v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
      if ((int)(v - value) >= 0) break;
      if (globaltimer_ns() - t0 > 2000000000ull) {       // 2 s: co-residency assumption violated
        if (status != nullptr) atomicExch(status, 2);
        break;
      }
    } while (true);
  }
  __syncthreads();
}

}  // namespace egb
