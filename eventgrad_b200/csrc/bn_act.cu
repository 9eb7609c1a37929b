// eventgrad_b200 -- fused BatchNorm2d (+ residual add) (+ ReLU), training forward + backward,
// channels-last activations in fp32 (the reference's precision, event.cpp:279) or bf16 -- every kernel is a
// template over the element type -- fp32 statistics/parameters.  sm_90a.
//
// Why: a launch-level profile of the flagship step (CIFAR ResNet, bf16 autocast)
// shows ATen's batch-norm + elementwise kernels taking ~2/3 of the GPU time while the tensor-core
// convolutions take under 1/3.  The block pattern of the reference's ResNet
// (/root/reference/dcifar10/common/resnet.hpp:39-52: bn -> relu, bn -> += residual -> relu) is
// memory-bound glue.
//
// Geometry.  NHWC == row-major [M = N*H*W, C].  The tensor is cut into C/64 channel SLICES; a CTA
// works on one slice (blockIdx.x, fastest) and one row split (blockIdx.y): 8 threads x 8 channels (one
// 128-byte line) per row, 32 rows per pass.  Per-slice partial sums are combined in fixed order by
// the last CTA *of that slice*, so the combine work is spread over C/64 CTAs and is tiny.
//
// Two code paths, chosen per call by the tensor size:
//   * FUSED (small/medium tensors -- the per-GPU tensors of the 8-GPU configuration): ONE kernel.
//     Each CTA keeps its slab in registers, publishes its partials, waits on a per-slice epoch flag
//     written by the slice's last CTA (all CTAs co-resident: grid <= 2 x SMs), then normalises the
//     registers and stores.  x is read exactly once; forward = 1 launch, backward = 1 launch.
//   * SPLIT (large tensors): stats kernel -> apply kernel; reduce kernel -> dx kernel.
#include "bn_common.cuh"

namespace egb {

// typed views of the type-erased BnParams pointers
// loads in flight per thread in the stats loop: 8 x 16 B (bf16) / 4 x 32 B (fp32)
#define BN_STATS_UNROLL(T) (sizeof(T) == 2 ? 8 : 4)
#define BN_APPLY_UNROLL(T) (sizeof(T) == 2 ? 4 : 2)
#define BN_RED_UNROLL(T) (sizeof(T) == 2 ? 3 : 2)
#define BN_DX_UNROLL(T) (sizeof(T) == 2 ? 2 : 1)
#define BN_PTRS(T)                                                              \
  const T* __restrict__ px = static_cast<const T*>(p.x);                        \
  const T* __restrict__ pres = static_cast<const T*>(p.res);                    \
  T* __restrict__ py = static_cast<T*>(p.y);                                    \
  const T* __restrict__ pdy = static_cast<const T*>(p.dy);                      \
  T* __restrict__ pdx = static_cast<T*>(p.dx);                                  \
  T* __restrict__ pdres = static_cast<T*>(p.dres);                              \
  (void)px; (void)pres; (void)py; (void)pdy; (void)pdx; (void)pdres;

// ===========================================================================================
// FUSED forward: stats + normalise (+res)(+relu) in one launch, x read once
// ===========================================================================================
template <typename T>
__global__ void __launch_bounds__(BN_THREADS, 2) bn_fwd_fused_kernel(const BnParams p) {
  BN_PTRS(T)
  __shared__ __align__(16) float smem[BN_RPP * 128];
  const int slice = blockIdx.x, rs = blockIdx.y, RS = gridDim.y;   // slice fastest: CTAs scheduled together read adjacent 128 B of the same rows
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const unsigned epoch = *reinterpret_cast<volatile unsigned int*>(p.epoch);
  const size_t coff = (size_t)slice * BN_SLICE + tx * 8;
  Raw8<T> xr[BN_FWD_PASSES];
  float s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
  const long long row0 = (long long)rs * (BN_FWD_PASSES * BN_RPP) + ty;
#pragma unroll
  for (int u = 0; u < BN_FWD_PASSES; ++u) {
    const long long row = row0 + u * BN_RPP;
    if (row < p.M) xr[u] = ld8(px + row * p.C + coff); else zero8(xr[u]);
  }
#pragma unroll
  for (int u = 0; u < BN_FWD_PASSES; ++u) {
    const V8 x = unpack8(xr[u]);                           // rows beyond M contribute exact zeros
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      s[e] += x.v[e];
      q[e] = fmaf(x.v[e], x.v[e], q[e]);
    }
  }
  float* prow = p.partial + ((size_t)slice * RS + rs) * 128;
  block_partials(s, q, smem, tx, ty, prow);
  if (elect_last_of_slice(p.ticket + slice, RS)) {
    double* tot = reinterpret_cast<double*>(smem);          // 8*128 doubles = 8 KB <= 16 KB
    slice_combine(p.partial + (size_t)slice * RS * 128, RS, tot);
    finalize_stats(p, slice, tot);
    publish_flag(p.flag + slice, epoch + 1u);
    if (threadIdx.x == 0) {                                 // global epoch bump by the last slice to finish
      const unsigned prev = atomicAdd(p.ticket + 63, 1u);
      if (prev == gridDim.x - 1) {
        p.ticket[63] = 0u;
        *p.epoch = epoch + 1u;
      }
    }
  }
  wait_flag(p.flag + slice, epoch + 1u, p.status);
  float sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = slice * BN_SLICE + tx * 8 + e;
    const float mean = __ldcg(p.mean + c), is = __ldcg(p.invstd + c);
    sc[e] = p.gamma[c] * is;
    sh[e] = p.beta[c] - mean * sc[e];
  }
  const bool has_res = pres != nullptr;
#pragma unroll
  for (int u = 0; u < BN_FWD_PASSES; ++u) {
    const long long row = row0 + u * BN_RPP;
    if (row >= p.M) continue;
    V8 x = unpack8(xr[u]);
    V8 r;
    if (has_res) r = unpack8(ld8(pres + row * p.C + coff));
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float v = fmaf(x.v[e], sc[e], sh[e]);
      if (has_res) v += r.v[e];
      x.v[e] = p.relu ? fmaxf(v, 0.f) : v;
    }
    Raw8<T> o;
    pack8(x, o);
    st8(py + row * p.C + coff, o);
  }
}

// ===========================================================================================
// FUSED backward: reduce + dx (+dres) in one launch
// ===========================================================================================
template <typename T>
__global__ void __launch_bounds__(BN_THREADS, 2) bn_bwd_fused_kernel(const BnParams p) {
  BN_PTRS(T)
  __shared__ __align__(16) float smem[BN_RPP * 128];
  const int slice = blockIdx.x, rs = blockIdx.y, RS = gridDim.y;   // slice fastest: CTAs scheduled together read adjacent 128 B of the same rows
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const unsigned epoch = *reinterpret_cast<volatile unsigned int*>(p.epoch);
  const size_t coff = (size_t)slice * BN_SLICE + tx * 8;
  float mu[8], is[8], s1[8], s2[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    mu[e] = p.mean[slice * BN_SLICE + tx * 8 + e];
    is[e] = p.invstd[slice * BN_SLICE + tx * 8 + e];
    s1[e] = s2[e] = 0.f;
  }
  Raw8<T> dzr[BN_BWD_PASSES], xr[BN_BWD_PASSES];
  const long long row0 = (long long)rs * (BN_BWD_PASSES * BN_RPP) + ty;
#pragma unroll
  for (int u = 0; u < BN_BWD_PASSES; ++u) {
    const long long row = row0 + u * BN_RPP;
    const bool ok = row < p.M;
    Raw8<T> d;
    if (ok) {
      d = ld8(pdy + row * p.C + coff);
      xr[u] = ld8(px + row * p.C + coff);
      if (p.relu) mask_le0(d, ld8(py + row * p.C + coff));  // dz = dy * (y > 0): fold the mask into dz now
    } else {
      zero8(d);
      zero8(xr[u]);
    }
    dzr[u] = d;
  }
#pragma unroll
  for (int u = 0; u < BN_BWD_PASSES; ++u) {
    const V8 dz = unpack8(dzr[u]), x = unpack8(xr[u]);
    const bool ok = (row0 + u * BN_RPP) < p.M;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      s1[e] += dz.v[e];
      s2[e] = fmaf(dz.v[e], ok ? (x.v[e] - mu[e]) * is[e] : 0.f, s2[e]);
    }
  }
  float* prow = p.partial + ((size_t)slice * RS + rs) * 128;
  block_partials(s1, s2, smem, tx, ty, prow);
  if (elect_last_of_slice(p.ticket + slice, RS)) {
    double* tot = reinterpret_cast<double*>(smem);
    slice_combine(p.partial + (size_t)slice * RS * 128, RS, tot);
    if (threadIdx.x < BN_SLICE) {
      p.dbeta[slice * BN_SLICE + threadIdx.x] = (float)tot[threadIdx.x];
      p.dgamma[slice * BN_SLICE + threadIdx.x] = (float)tot[64 + threadIdx.x];
    }
    publish_flag(p.flag + slice, epoch + 1u);
    if (threadIdx.x == 0) {
      const unsigned prev = atomicAdd(p.ticket + 63, 1u);
      if (prev == gridDim.x - 1) {
        p.ticket[63] = 0u;
        *p.epoch = epoch + 1u;
      }
    }
  }
  wait_flag(p.flag + slice, epoch + 1u, p.status);
  float k0[8], k1[8], k2[8];
  const float invM = 1.f / (float)p.M;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = slice * BN_SLICE + tx * 8 + e;
    k0[e] = p.gamma[c] * is[e];
    k1[e] = __ldcg(p.dbeta + c) * invM;
    k2[e] = __ldcg(p.dgamma + c) * invM;
  }
  const bool want_dres = pdres != nullptr;
#pragma unroll
  for (int u = 0; u < BN_BWD_PASSES; ++u) {
    const long long row = row0 + u * BN_RPP;
    if (row >= p.M) continue;
    const V8 dz = unpack8(dzr[u]);
    V8 x = unpack8(xr[u]);
#pragma unroll
    for (int e = 0; e < 8; ++e) x.v[e] = k0[e] * (dz.v[e] - k1[e] - (x.v[e] - mu[e]) * is[e] * k2[e]);
    Raw8<T> o;
    pack8(x, o);
    st8(pdx + row * p.C + coff, o);
    if (want_dres) st8(pdres + row * p.C + coff, dzr[u]);
  }
}

// ===========================================================================================
// SPLIT path (large tensors)
// ===========================================================================================
template <typename T>
__global__ void __launch_bounds__(BN_THREADS, 3) bn_fwd_stats_kernel(const BnParams p) {
  BN_PTRS(T)
  __shared__ __align__(16) float smem[BN_RPP * 128];
  const int slice = blockIdx.x, rs = blockIdx.y, RS = gridDim.y;   // slice fastest: CTAs scheduled together read adjacent 128 B of the same rows
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const size_t coff = (size_t)slice * BN_SLICE + tx * 8;
  float s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
  const long long stride = (long long)RS * BN_RPP;
  long long row = (long long)rs * BN_RPP + ty;
  for (; row + (BN_STATS_UNROLL(T) - 1) * stride < p.M; row += BN_STATS_UNROLL(T) * stride) {
    Raw8<T> xr[BN_STATS_UNROLL(T)];
#pragma unroll
    for (int u = 0; u < BN_STATS_UNROLL(T); ++u) xr[u] = ld8(px + (row + u * stride) * p.C + coff);
#pragma unroll
    for (int u = 0; u < BN_STATS_UNROLL(T); ++u) {
      const V8 x = unpack8(xr[u]);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        s[e] += x.v[e];
        q[e] = fmaf(x.v[e], x.v[e], q[e]);
      }
    }
  }
  for (; row < p.M; row += stride) {
    const V8 x = unpack8(ld8(px + row * p.C + coff));
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      s[e] += x.v[e];
      q[e] = fmaf(x.v[e], x.v[e], q[e]);
    }
  }
  block_partials(s, q, smem, tx, ty, p.partial + ((size_t)slice * RS + rs) * 128);
  if (!elect_last_of_slice(p.ticket + slice, RS)) return;
  double* tot = reinterpret_cast<double*>(smem);
  slice_combine(p.partial + (size_t)slice * RS * 128, RS, tot);
  finalize_stats(p, slice, tot);
}

template <typename T>
__global__ void __launch_bounds__(BN_THREADS, 3) bn_fwd_apply_kernel(const BnParams p) {
  BN_PTRS(T)
  const int slice = blockIdx.x, rs = blockIdx.y, RS = gridDim.y;   // slice fastest: CTAs scheduled together read adjacent 128 B of the same rows
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const size_t coff = (size_t)slice * BN_SLICE + tx * 8;
  float sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) bn_affine(p, slice * BN_SLICE + tx * 8 + e, sc[e], sh[e]);
  const long long stride = (long long)RS * BN_RPP;
  const bool has_res = pres != nullptr;
  for (long long row = (long long)rs * BN_RPP + ty; row < p.M; row += BN_APPLY_UNROLL(T) * stride) {
    Raw8<T> xr[BN_APPLY_UNROLL(T)], rr[BN_APPLY_UNROLL(T)];
#pragma unroll
    for (int u = 0; u < BN_APPLY_UNROLL(T); ++u) {
      const long long r2 = row + u * stride;
      if (r2 < p.M) {
        xr[u] = ld8(px + r2 * p.C + coff);
        if (has_res) rr[u] = ld8(pres + r2 * p.C + coff);
      }
    }
#pragma unroll
    for (int u = 0; u < BN_APPLY_UNROLL(T); ++u) {
      const long long r2 = row + u * stride;
      if (r2 >= p.M) continue;
      V8 x = unpack8(xr[u]);
      V8 r;
      if (has_res) r = unpack8(rr[u]);
      unsigned m = 0u;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float v = fmaf(x.v[e], sc[e], sh[e]);
        if (has_res) v += r.v[e];
        m |= (v > 0.f ? 1u : 0u) << e;
        x.v[e] = p.relu ? fmaxf(v, 0.f) : v;
      }
      Raw8<T> o;
      pack8(x, o);
      st8(py + r2 * p.C + coff, o);
      if (p.mask != nullptr) p.mask[(r2 * p.C + coff) >> 3] = (unsigned char)m;
      if (p.y_planes != nullptr) store_planes8(x, p.y_planes + r2 * p.C + coff, (size_t)p.M * p.C);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(BN_THREADS, 2) bn_bwd_reduce_kernel(const BnParams p) {
  BN_PTRS(T)
  __shared__ __align__(16) float smem[BN_RPP * 128];
  const int slice = blockIdx.x, rs = blockIdx.y, RS = gridDim.y;   // slice fastest: CTAs scheduled together read adjacent 128 B of the same rows
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const size_t coff = (size_t)slice * BN_SLICE + tx * 8;
  float mu[8], is[8], s1[8], s2[8], sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    mu[e] = p.mean[slice * BN_SLICE + tx * 8 + e];
    is[e] = p.invstd[slice * BN_SLICE + tx * 8 + e];
    s1[e] = s2[e] = 0.f;
    if (p.mask_mode == BN_MASK_X) bn_affine(p, slice * BN_SLICE + tx * 8 + e, sc[e], sh[e]);
  }
  const long long stride = (long long)RS * BN_RPP;
  for (long long row = (long long)rs * BN_RPP + ty; row < p.M; row += BN_RED_UNROLL(T) * stride) {
    Raw8<T> dr[BN_RED_UNROLL(T)], xr[BN_RED_UNROLL(T)], yr[BN_RED_UNROLL(T)];
    unsigned char mb[BN_RED_UNROLL(T)];
#pragma unroll
    for (int u = 0; u < BN_RED_UNROLL(T); ++u) {
      const long long r2 = row + u * stride;
      if (r2 < p.M) {
        dr[u] = ld8(pdy + r2 * p.C + coff);
        xr[u] = ld8(px + r2 * p.C + coff);
        if (p.relu && p.mask_mode == BN_MASK_Y) yr[u] = ld8(py + r2 * p.C + coff);
        if (p.relu && p.mask_mode == BN_MASK_BITS) mb[u] = p.mask[(r2 * p.C + coff) >> 3];
      }
    }
#pragma unroll
    for (int u = 0; u < BN_RED_UNROLL(T); ++u) {
      if (row + u * stride >= p.M) continue;
      const V8 d = unpack8(dr[u]), x = unpack8(xr[u]);
      const unsigned m = p.relu ? relu_bits<T>(p, yr[u], mb[u], x, sc, sh) : 0xffu;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float dz = ((m >> e) & 1u) ? d.v[e] : 0.f;
        s1[e] += dz;
        s2[e] = fmaf(dz, (x.v[e] - mu[e]) * is[e], s2[e]);
      }
    }
  }
  block_partials(s1, s2, smem, tx, ty, p.partial + ((size_t)slice * RS + rs) * 128);
  if (!elect_last_of_slice(p.ticket + slice, RS)) return;
  double* tot = reinterpret_cast<double*>(smem);
  slice_combine(p.partial + (size_t)slice * RS * 128, RS, tot);
  if (threadIdx.x < BN_SLICE) {
    p.dbeta[slice * BN_SLICE + threadIdx.x] = (float)tot[threadIdx.x];
    p.dgamma[slice * BN_SLICE + threadIdx.x] = (float)tot[64 + threadIdx.x];
  }
}

template <typename T>
__global__ void __launch_bounds__(BN_THREADS, 2) bn_bwd_dx_kernel(const BnParams p) {
  BN_PTRS(T)
  const int slice = blockIdx.x, rs = blockIdx.y, RS = gridDim.y;   // slice fastest: CTAs scheduled together read adjacent 128 B of the same rows
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const size_t coff = (size_t)slice * BN_SLICE + tx * 8;
  float mu[8], is[8], k0[8], k1[8], k2[8], sc[8], sh[8];
  const float invM = 1.f / (float)p.M;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = slice * BN_SLICE + tx * 8 + e;
    mu[e] = p.mean[c];
    is[e] = p.invstd[c];
    k0[e] = p.gamma[c] * is[e];              // dx = k0*(dz - k1 - xhat*k2)
    k1[e] = p.dbeta[c] * invM;
    k2[e] = p.dgamma[c] * invM;
    if (p.mask_mode == BN_MASK_X) bn_affine(p, c, sc[e], sh[e]);
  }
  const long long stride = (long long)RS * BN_RPP;
  const bool want_dres = pdres != nullptr;
  for (long long row = (long long)rs * BN_RPP + ty; row < p.M; row += BN_DX_UNROLL(T) * stride) {
    Raw8<T> dr[BN_DX_UNROLL(T)], xr[BN_DX_UNROLL(T)], yr[BN_DX_UNROLL(T)];
    unsigned char mb[BN_DX_UNROLL(T)];
#pragma unroll
    for (int u = 0; u < BN_DX_UNROLL(T); ++u) {
      const long long r2 = row + u * stride;
      if (r2 < p.M) {
        dr[u] = ld8(pdy + r2 * p.C + coff);
        xr[u] = ld8(px + r2 * p.C + coff);
        if (p.relu && p.mask_mode == BN_MASK_Y) yr[u] = ld8(py + r2 * p.C + coff);
        if (p.relu && p.mask_mode == BN_MASK_BITS) mb[u] = p.mask[(r2 * p.C + coff) >> 3];
      }
    }
#pragma unroll
    for (int u = 0; u < BN_DX_UNROLL(T); ++u) {
      const long long r2 = row + u * stride;
      if (r2 >= p.M) continue;
      V8 d = unpack8(dr[u]), x = unpack8(xr[u]);
      const unsigned m = p.relu ? relu_bits<T>(p, yr[u], mb[u], x, sc, sh) : 0xffu;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float dz = ((m >> e) & 1u) ? d.v[e] : 0.f;
        d.v[e] = dz;
        x.v[e] = k0[e] * (dz - k1[e] - (x.v[e] - mu[e]) * is[e] * k2[e]);
      }
      Raw8<T> o;
      pack8(x, o);
      if (pdx != nullptr) st8(pdx + r2 * p.C + coff, o);
      if (p.dx_planes != nullptr) store_planes8(x, p.dx_planes + r2 * p.C + coff, (size_t)p.M * p.C);
      if (want_dres) {
        pack8(d, o);
        st8(pdres + r2 * p.C + coff, o);
      }
    }
  }
}

// -------------------------------------------------------------------------------------------
int bn_partial_rows(int sm_count) { return sm_count * 4 + 64; }   // max total CTAs of a reduction launch

static inline long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }

// which: 0 training forward (stats [+ apply]), 1 apply only (eval), 2 backward
template <typename T>
static cudaError_t launch_bn_t(const BnParams& p, int which, int sm_count, cudaStream_t s) {
  if (p.C % BN_SLICE != 0 || p.C / BN_SLICE > 32 || p.M < 1) return cudaErrorInvalidValue;
  const int slices = p.C / BN_SLICE;
  const long long passes = ceil_div(p.M, BN_RPP);
  const int max_ctas = 2 * sm_count;                       // co-residency bound of the fused kernels
  const int split_cap = 2 * sm_count;                      // reductions: ONE wave of fat CTAs (2 resident per SM)
  auto map_grid = [&](int rows_per_cta_passes) {
    long long rsn = ceil_div(passes, rows_per_cta_passes);
    const long long cap = (long long)(8 * sm_count) / slices;
    if (rsn > cap) rsn = cap;
    if (rsn < 1) rsn = 1;
    return dim3((unsigned)slices, (unsigned)rsn);
  };
  auto red_grid = [&]() {
    long long rsn = ceil_div(passes, 8);
    const long long cap = (long long)split_cap / slices;
    if (rsn > cap) rsn = cap;
    if (rsn < 1) rsn = 1;
    return dim3((unsigned)slices, (unsigned)rsn);
  };
  if (which == 0) {
    const long long rs_f = ceil_div(passes, BN_FWD_PASSES);
    if (p.fused_ok && p.y_planes == nullptr && p.mask == nullptr && rs_f * slices <= max_ctas) {
      eg_count_launch(EG_FAM_BN, 1);
      bn_fwd_fused_kernel<T><<<dim3((unsigned)slices, (unsigned)rs_f), BN_THREADS, 0, s>>>(p);
    } else {
      eg_count_launch(EG_FAM_BN, 2);
      bn_fwd_stats_kernel<T><<<red_grid(), BN_THREADS, 0, s>>>(p);
      bn_fwd_apply_kernel<T><<<map_grid(BN_APPLY_UNROLL(T)), BN_THREADS, 0, s>>>(p);
    }
  } else if (which == 1) {
    eg_count_launch(EG_FAM_BN, 1);
    bn_fwd_apply_kernel<T><<<map_grid(BN_APPLY_UNROLL(T)), BN_THREADS, 0, s>>>(p);
  } else if (which == 2) {
    const long long rs_b = ceil_div(passes, BN_BWD_PASSES);
    if (p.fused_ok && p.dx_planes == nullptr && p.mask_mode == BN_MASK_Y && rs_b * slices <= max_ctas) {
      eg_count_launch(EG_FAM_BN, 1);
      bn_bwd_fused_kernel<T><<<dim3((unsigned)slices, (unsigned)rs_b), BN_THREADS, 0, s>>>(p);
    } else {
      eg_count_launch(EG_FAM_BN, 2);
      bn_bwd_reduce_kernel<T><<<red_grid(), BN_THREADS, 0, s>>>(p);
      bn_bwd_dx_kernel<T><<<map_grid(BN_DX_UNROLL(T)), BN_THREADS, 0, s>>>(p);
    }
  } else {
    return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t launch_bn(const BnParams& p, int which, int sm_count, cudaStream_t s) {
  return p.fp32 ? launch_bn_t<float>(p, which, sm_count, s) : launch_bn_t<__nv_bfloat16>(p, which, sm_count, s);
}

}  // namespace egb
