// eventgrad_b200 -- the convolutions of the ResNet family (3x3 stride 1/2, 1x1 stride 1/2, 3-channel stem: forward, data
// gradient, weight gradient) on the Hopper tensor cores (wgmma) at fp32 accuracy (sm_90a).
//
// The reference trains in fp32 (dcifar10/event/event.cpp:259-276 feeds fp32 tensors to torch::nn::Conv2d,
// resnet.hpp:3-9), and fp32 has no tensor-core path: cuDNN's fp32 kernels are SIMT (67 TFLOP/s peak on an H100 SXM).
// These kernels keep fp32 STORAGE and fp32 ACCURACY but do the multiply-accumulate work with wgmma.mma_async:
//
//   every fp32 operand is split once into three bf16 planes  x = x0 + x1 + x2  (8+8+8 mantissa bits: exact up to
//   2^-24 |x|), and the product is accumulated in fp32 from the six significant cross terms
//       x0*w0 + x0*w1 + x1*w0 + x1*w1 + x0*w2 + x2*w0        (dropped: x1*w2, x2*w1, x2*w2 <= 2^-25 |x*w|)
//   so one "fp32 MMA" costs six bf16 MMAs: 989 TFLOP/s / 6 = 165 TFLOP/s of fp32-equivalent peak, 2.5x the SIMT
//   peak.  tests/test_gpu_conv_tc.py measures the error against an fp64 convolution next to cuDNN's fp32 error.
//
// Implicit GEMM, no im2col buffer: activations are NHWC planes [3][N][H][W][C]; the A tile of filter tap (r,s) is a
// SHIFTED window of the input, which a tiled 5-D TMA load fetches directly -- coordinates (c0, s-1, h0+r-1, n0, plane)
// with the hardware zero-filling everything outside the image (that IS the padding).
//
//   conv3x3_fprop_kernel   Y[pix, co] = sum_{tap,ci} X[pix+tap, ci] * Wt[co, tap, ci]        (forward; also the data
//                          gradient: X := dY planes, Wt := flipped/transposed weights [ci][8-tap][co])
//       persistent CTAs, tile 128 pixels x NT channels (NT = 128 or 64: conv_fprop_ntile), K loop = 9 taps x
//       Cin/64; warpgroup 0 is the TMA producer (at NT = 128 it gives most of its registers to the MMA warpgroups,
//       setmaxnreg), warpgroups 1 and 2 each own 64 rows of the tile: 24 wgmma per stage into five FRESH register
//       accumulators, each added into the fp32 tile sum (round-to-nearest adds: the tensor core itself truncates).
//   conv3x3_wgrad_kernel   dW[tap, ci, co] = sum_pix X[pix+tap, ci] * dY[pix, co]            (weight gradient)
//       both operands are "MN-major" (the contiguous dimension is the channel, K = pixels), expressed with MN-major
//       SWIZZLE_128B descriptors over the very same TMA boxes; split over pixel ranges, partial sums in a workspace
//       (one split: dW is written directly).  N tile 64 (see CV_WGRAD_NT).
//   conv_wgrad_reduce_kernel   fixed-tree (bitwise reproducible) sum of the partials + transpose to the OHWI layout.
//   conv_fprop_reduce_kernel   sum of the K-split partial tiles of the forward kernel on small grids (per-GPU batch 32).
//   split3_kernel          fp32 -> three bf16 planes (flat; "parity" variant: the four (h%2, w%2) sub-images of the
//                          input of a STRIDE-2 conv, so that its taps become unit-stride boxes; "stem" variant: the 27
//                          (tap, rgb) values of the 3-channel stem gathered into one 64-wide K block = a 1x1 conv)
//   conv_wprep_kernel      weights fp32 [Co][T][Ci] -> planes [3][Co][T*Ci] (forward) and [3][Ci][T*Co] (data gradient).
//
// One kernel pair serves every convolution of the network through a TAP TABLE (ConvTcParams.dh/dw/src/wk): tap t
// reads source sub-image src[t] shifted by (dh[t], dw[t]) and the weight slice wk[t]:
//   3x3 stride 1      9 taps, shift (r-1, s-1)                      dgrad: same taps, weight slice 8-t of W^T
//   3x3 stride 2      9 taps over the parity images, shift in {-1,0}   dgrad: 4 launches, one per INPUT parity class
//                                                                   (1/2/2/4 taps over dY, scattered with stride 2)
//   1x1 stride 2      1 tap over parity image (0,0)                 dgrad: class (0,0) only, the rest is zero
//   stem (3 -> 64)    1 tap over the gathered 64-wide patches       (no data gradient: the input is the image)
#include "api.h"
#include "common.cuh"
#include "tc_common.cuh"

namespace egb {
using namespace tc;

#define CV_THREADS 384     // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + epilogue, 64 rows of the tile each
#define CV_CONSUMERS 256   // threads that arrive on an empty[] barrier (every MMA thread, after its wgmma wait)
#define CV_APLANE 16384u   // one bf16 plane of an operand tile with 128 rows: 128 x 128 B
#define CV_SMS 132         // grid cap of the element-wise launches (H100 SXM: 132 SMs)
// N tile of the forward / data-gradient kernel: 128 or 64 output channels, chosen per launch by conv_fprop_ntile.
// An MMA warpgroup holds three accumulator sets of NT/2 floats per thread (the sum + two in flight): 192 registers
// at NT = 128, more than the 168 a thread of a 384-thread CTA launches with.  So at NT = 128 the producer warpgroup,
// whose one working thread only issues TMA, drops to CV_PRODUCER_REGS and the MMA warpgroups rise to CV_MMA_REGS
// (128 x 40 + 256 x 232 = 64512 = 384 x 168).  The wider tile reads A from shared memory once per 128
// output channels instead of 64, and spreads the per-k-block barriers and descriptors over twice the MMA work.
#define CV_PRODUCER_REGS 40
#define CV_MMA_REGS 232
// N tile of the weight-gradient kernel: 64.  At 128 its MMA warpgroups need more than 232 registers (ptxas spills
// about 400 bytes per thread, also at a 24 / 240 split), so it stays at 64.
#define CV_WGRAD_NT 64
// operand stages in the 227 KB of shared memory: NT = 64: 3 x 72 KB (A 3 x 16 KB + B 3 x 8 KB); NT = 128: 2 x 96 KB
#define CV_STAGES(NT) ((NT) == 128 ? 2 : 3)

// the six cross terms (plane of A, plane of B), largest last so that the small corrections are summed first
#define CV_TERM_A(t) ((t) == 0 ? 2 : ((t) == 2 || (t) == 3) ? 1 : 0)
#define CV_TERM_B(t) ((t) == 1 ? 2 : ((t) == 2 || (t) == 4) ? 1 : 0)

template <int NT, int TA, int TB>
__device__ __forceinline__ void mma_nt(float (&d)[NT / 2], uint64_t da, uint64_t db, uint32_t acc) {
  if constexpr (NT == 128)
    wgmma_m64n128<TA, TB>(d, da, db, acc);
  else
    wgmma_m64n64<TA, TB>(d, da, db, acc);
}

// One k-block of the six-term product for this warpgroup's 64 rows.  The tensor core TRUNCATES every accumulation
// to fp32, relative to the largest magnitude in it; a chain of MMAs onto a full-magnitude accumulator therefore drifts
// towards zero (with one accumulator per 24-MMA k-block, results shrank by ~6e-8 relative on H100).  So: the five small correction terms (20 MMAs) go into one
// fresh accumulator, and every 16-K MMA of the main term x0*w0 into a fresh accumulator of its own; each is added
// into the fp32 sum `acc` with round-to-nearest.  Two accumulator sets (d, e) alternate so that one MMA group is
// always queued on the tensor core while the previous one is being added.
// k_step: byte offset of 16 K elements inside an operand plane.
template <int NT, int TA, int TB>
__device__ __forceinline__ void term_mma(float (&d)[NT / 2], uint32_t sa, uint32_t sb, uint32_t lbo, uint32_t scale_d) {
  const uint64_t da = TA ? desc_mn_sw128(sa, lbo) : desc_k_sw128(sa);
  const uint64_t db = TB ? desc_mn_sw128(sb, lbo) : desc_k_sw128(sb);
  mma_nt<NT, TA, TB>(d, da, db, scale_d);
}
// acc += d, and half an ulp of d back with d's sign: the MMA's final rounding is towards zero (it loses half an ulp on
// average, a bias that a deep network amplifies), the correction makes each partial unbiased.
template <int R>
__device__ __forceinline__ void add_group(float (&acc)[R], float (&d)[R]) {
  wgmma_fence_regs(d);
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const float half_ulp = __int_as_float(__float_as_int(d[j]) & 0xff800000) * 5.9604645e-8f;   // sign * 2^(e-24)
    acc[j] += d[j];
    acc[j] += half_ulp;
  }
}
template <int NT, int TA, int TB>
__device__ __forceinline__ void six_term_kblock(float (&acc)[NT / 2], float (&d)[NT / 2], float (&e)[NT / 2],
                                                uint32_t a0, uint32_t a_plane, uint32_t b0, uint32_t b_plane,
                                                uint32_t lbo, uint32_t k_step) {
  wgmma_fence();
#pragma unroll
  for (int t = 0; t < 5; ++t)
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4)
      term_mma<NT, TA, TB>(d, a0 + CV_TERM_A(t) * a_plane + k4 * k_step, b0 + CV_TERM_B(t) * b_plane + k4 * k_step, lbo,
                           (t > 0 || k4 > 0) ? 1u : 0u);
  wgmma_commit();
  // main term (plane 0 of both operands), one fresh accumulator per K step
  wgmma_fence();
  term_mma<NT, TA, TB>(e, a0, b0, lbo, 0u);
  wgmma_commit();
  wgmma_wait<1>();
  add_group(acc, d);
  wgmma_fence();
  term_mma<NT, TA, TB>(d, a0 + k_step, b0 + k_step, lbo, 0u);
  wgmma_commit();
  wgmma_wait<1>();
  add_group(acc, e);
  wgmma_fence();
  term_mma<NT, TA, TB>(e, a0 + 2 * k_step, b0 + 2 * k_step, lbo, 0u);
  wgmma_commit();
  wgmma_wait<1>();
  add_group(acc, d);
  wgmma_fence();
  term_mma<NT, TA, TB>(d, a0 + 3 * k_step, b0 + 3 * k_step, lbo, 0u);
  wgmma_commit();
  wgmma_wait<1>();
  add_group(acc, e);
  wgmma_wait<0>();
  add_group(acc, d);
}

// ------------------------------------------------------------------------------------------------ forward / dgrad
// ADD: the epilogue adds the masked skip-connection gradient (p.addend / p.addmask); only launched un-split.  A separate
// instantiation, so that the k-loop of the plain kernel is compiled exactly as without the option.
template <int NT, int STAGES, bool ADD>
__global__ void __launch_bounds__(CV_THREADS, 1)
conv3x3_fprop_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const ConvTcParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  constexpr uint32_t A_BYTES = 3u * CV_APLANE, B_PLANE = (uint32_t)NT * 128u, STAGE = A_BYTES + 3u * B_PLANE;
  const int tid = threadIdx.x, wg = tid >> 7;
  const uint32_t smem_unaligned = s_u32(smem_raw);
  const uint32_t smem0 = (smem_unaligned + 1023u) & ~1023u;
  unsigned char* smem_al = smem_raw + (smem0 - smem_unaligned);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_al + STAGES * STAGE);
  const uint32_t full0 = s_u32(bars), empty0 = full0 + 8u * STAGES;
  const int cpb = p.Ca / 64, num_kb_all = p.ntaps * cpb;
  const int n_tiles = p.Cb / NT;
  const int ksplits = p.ksplits;                           // > 1: few tiles (small batch): split the K loop over CTAs,
  const int kper = (num_kb_all + ksplits - 1) / ksplits;   //      partial tiles go to a workspace (launcher reduces)
  const int total = p.m_tiles * n_tiles * ksplits;
  const int tpi = p.bn == 1 ? p.H / p.bh : 1;              // tiles per image
#define CV_DECODE_WORK                                                         \
  const int ks = work % ksplits, tile_ = work / ksplits;                       \
  const int mt = tile_ / n_tiles, nt = tile_ - mt * n_tiles;                   \
  const int kb_lo = ks * kper, kb_hi = min(num_kb_all, kb_lo + kper);

  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      bar_init(full0 + 8u * i, 1);
      bar_init(empty0 + 8u * i, CV_CONSUMERS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA PRODUCER (one thread) =====================
    if constexpr (NT == 128) setmaxnreg_dec<CV_PRODUCER_REGS>();
    if (tid == 0) {
      uint32_t it = 0;
      for (int work = blockIdx.x; work < total; work += gridDim.x) {
        CV_DECODE_WORK
        const int n0 = p.bn == 1 ? mt / tpi : mt * p.bn;
        const int h0 = p.bn == 1 ? (mt - n0 * tpi) * p.bh : 0;
        for (int kb = kb_lo; kb < kb_hi; ++kb, ++it) {
          const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
          const int tap = kb / cpb, cc = kb - tap * cpb;
          const int dh = p.dh[tap], dw = p.dw[tap], src = p.src[tap], wk = p.wk[tap];
          bar_wait(empty0 + 8u * s, ph ^ 1u);
          bar_expect_tx(full0 + 8u * s, STAGE);
          const uint32_t sa = smem0 + s * STAGE;
#pragma unroll
          for (int pl = 0; pl < 3; ++pl)      // shifted window; rows outside the image arrive as zeros (= padding)
            tma_load_5d(sa + pl * CV_APLANE, &tmA, full0 + 8u * s, cc * 64, dw, h0 + dh, n0, pl * p.nsrc + src);
#pragma unroll
          for (int pl = 0; pl < 3; ++pl)
            tma_load_2d(sa + A_BYTES + pl * B_PLANE, &tmB, full0 + 8u * s, wk * p.Ca + cc * 64, pl * p.Cb + nt * NT);
        }
      }
    }
  } else {
    // ===================== MMA + EPILOGUE (rows 64g .. 64g+63 of every tile) =====================
    if constexpr (NT == 128) setmaxnreg_inc<CV_MMA_REGS>();
    const int g = wg - 1, warp = (tid >> 5) & 3, lane = tid & 31;
    const long long M = (long long)p.N * p.H * p.W;
    float d[NT / 2], e[NT / 2];
#pragma unroll
    for (int j = 0; j < NT / 2; ++j) d[j] = e[j] = 0.f;
    uint32_t it = 0;
    for (int work = blockIdx.x; work < total; work += gridDim.x) {
      CV_DECODE_WORK
      float acc[NT / 2];
#pragma unroll
      for (int j = 0; j < NT / 2; ++j) acc[j] = 0.f;
      for (int kb = kb_lo; kb < kb_hi; ++kb, ++it) {
        const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
        bar_wait(full0 + 8u * s, ph);                          // operands have landed
        const uint32_t sa = smem0 + s * STAGE;
        // K-major operands: +16 K elements = +32 bytes inside the 128-byte swizzled row
        six_term_kblock<NT, 0, 0>(acc, d, e, sa + (uint32_t)g * 8192u, CV_APLANE, sa + A_BYTES, B_PLANE, 0u, 32u);
        bar_arrive(empty0 + 8u * s);                           // this thread's MMAs no longer read the stage
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long row = (long long)mt * 128 + g * 64 + warp * 16 + (lane >> 2) + h * 8;
        float* dst;
        if (ksplits > 1) {                                     // partial tile, dense rows: ws[ks][m_tiles*128][Cb]
          dst = p.ws + (((size_t)ks * p.m_tiles * 128) + (size_t)row) * p.Cb + nt * NT;
        } else if (row < M) {
          long long opix = row;
          if (p.os != 1 || p.OH != p.H || p.OW != p.W) {        // strided scatter (data gradient of a stride-2 conv)
            const int hw = p.H * p.W;
            const int n = (int)(row / hw), rem = (int)(row - (long long)n * hw);
            const int i = rem / p.W, j = rem - i * p.W;
            opix = ((long long)n * p.OH + i * p.os + p.op) * p.OW + j * p.os + p.oq;
          }
          dst = p.out + (size_t)opix * p.Cb + nt * NT;
        } else {
          continue;
        }
        dst += 2 * (lane & 3);
        if constexpr (ADD) {                                   // skip-connection gradient: + (mask ? addend : 0.f)
          // Every load of the row segment is issued before the first store, so the thread waits out one load latency
          // per row instead of one per 8 channels.  Column j's 2 channels sit in mask byte (off >> 3) + j: the NT/8
          // bytes are consecutive and NT/8-aligned (Cb and nt*NT are multiples of NT), one vector load.
          const size_t off = (size_t)(dst - p.out);
          const float* __restrict__ src = p.addend + off;
          uint32_t mw[NT / 32];
          if constexpr (NT == 128) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(p.addmask + (off >> 3)));
            mw[0] = v.x; mw[1] = v.y; mw[2] = v.z; mw[3] = v.w;
          } else {
            const uint2 v = __ldg(reinterpret_cast<const uint2*>(p.addmask + (off >> 3)));
            mw[0] = v.x; mw[1] = v.y;
          }
          float2 a[NT / 8];
#pragma unroll
          for (int j = 0; j < NT / 8; ++j) a[j] = __ldg(reinterpret_cast<const float2*>(src + 8 * j));
#pragma unroll
          for (int j = 0; j < NT / 8; ++j) {
            const unsigned m = (mw[j >> 2] >> (8 * (j & 3) + 2 * (lane & 3))) & 3u;
            *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h] + ((m & 1u) ? a[j].x : 0.f),
                                                                  acc[4 * j + 2 * h + 1] + ((m & 2u) ? a[j].y : 0.f));
          }
          continue;
        }
#pragma unroll
        for (int j = 0; j < NT / 8; ++j)
          *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
  }
}

// out[pixel(row)][c] = sum_ks ws[ks][row][c] (fixed order), with the same output mapping as the un-split epilogue
__global__ void __launch_bounds__(256) conv_fprop_reduce_kernel(const ConvTcParams p) {
  const long long M = (long long)p.N * p.H * p.W;
  const int c4n = p.Cb / 4;
  const size_t zs = (size_t)p.m_tiles * 128 * p.Cb;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M * c4n; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / c4n;
    const int c4 = (int)(i - row * c4n);
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int z = 0; z < p.ksplits; ++z) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(p.ws + z * zs + (size_t)row * p.Cb) + c4);
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    long long opix = row;
    if (p.os != 1 || p.OH != p.H || p.OW != p.W) {
      const int hw = p.H * p.W;
      const int n = (int)(row / hw), rem = (int)(row - (long long)n * hw);
      const int ii = rem / p.W, j = rem - ii * p.W;
      opix = ((long long)n * p.OH + ii * p.os + p.op) * p.OW + j * p.os + p.oq;
    }
    if (p.addend != nullptr) {                                 // skip-connection gradient, as in the un-split epilogue
      const size_t off = (size_t)opix * p.Cb + 4 * c4;
      const float4 v = __ldg(reinterpret_cast<const float4*>(p.addend + off));
      const unsigned m = (unsigned)p.addmask[off >> 3] >> (off & 7);
      a.x += (m & 1u) ? v.x : 0.f;
      a.y += (m & 2u) ? v.y : 0.f;
      a.z += (m & 4u) ? v.z : 0.f;
      a.w += (m & 8u) ? v.w : 0.f;
    }
    reinterpret_cast<float4*>(p.out + (size_t)opix * p.Cb)[c4] = a;
  }
}

// ------------------------------------------------------------------------------------------------ weight gradient
// grid (ceil(U/2), Cb/NT, splits); U = ntaps * Ca/64 "units" (tap, 64-channel block of the input); one CTA accumulates
// D[128 = two units][NT] over its range of 64-pixel K blocks and writes the partial to ws[split][unit*64 + ci][co].
// MMA warpgroup g owns unit g of the pair (tile rows 64g .. 64g+63).
template <int NT, int STAGES>
__global__ void __launch_bounds__(CV_THREADS, 1)
conv3x3_wgrad_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmG,
                     const ConvTcParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  constexpr uint32_t A_BYTES = 3u * CV_APLANE, B_PLANE = (uint32_t)NT * 128u, STAGE = A_BYTES + 3u * B_PLANE;
  constexpr uint32_t BLK = 8192u;                           // one [64 pixels][64 channels] block
  const int tid = threadIdx.x, wg = tid >> 7;
  const uint32_t smem_unaligned = s_u32(smem_raw);
  const uint32_t smem0 = (smem_unaligned + 1023u) & ~1023u;
  unsigned char* smem_al = smem_raw + (smem0 - smem_unaligned);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_al + STAGES * STAGE);
  const uint32_t full0 = s_u32(bars), empty0 = full0 + 8u * STAGES;
  const int cpb = p.Ca / 64, U = p.ntaps * cpb;
  const int u0 = 2 * blockIdx.x, u1 = (u0 + 1 < U) ? u0 + 1 : u0;
  const int per = (p.k_blocks + (int)gridDim.z - 1) / (int)gridDim.z;
  const int kb0 = blockIdx.z * per, kb1 = min(p.k_blocks, kb0 + per);
  const int nkb = kb1 > kb0 ? kb1 - kb0 : 0;
  const int bpi = p.bn == 1 ? p.H / p.bh : 1;              // 64-pixel blocks per image

  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      bar_init(full0 + 8u * i, 1);
      bar_init(empty0 + 8u * i, CV_CONSUMERS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    if (tid == 0) {
      int tap[2], cb64[2];
      tap[0] = u0 / cpb; cb64[0] = u0 - tap[0] * cpb;
      tap[1] = u1 / cpb; cb64[1] = u1 - tap[1] * cpb;
      for (int i = 0; i < nkb; ++i) {
        const int kb = kb0 + i;
        const uint32_t s = (uint32_t)i % STAGES, ph = ((uint32_t)i / STAGES) & 1u;
        const int n0 = p.bn == 1 ? kb / bpi : kb * p.bn;
        const int h0 = p.bn == 1 ? (kb - n0 * bpi) * p.bh : 0;
        bar_wait(empty0 + 8u * s, ph ^ 1u);
        bar_expect_tx(full0 + 8u * s, STAGE);
        const uint32_t sa = smem0 + s * STAGE;
#pragma unroll
        for (int pl = 0; pl < 3; ++pl)
#pragma unroll
          for (int blk = 0; blk < 2; ++blk) {
            const int t = tap[blk];
            tma_load_5d(sa + pl * CV_APLANE + blk * BLK, &tmX, full0 + 8u * s, cb64[blk] * 64, p.dw[t], h0 + p.dh[t], n0,
                        pl * p.nsrc + p.src[t]);
          }
#pragma unroll
        for (int pl = 0; pl < 3; ++pl)
#pragma unroll
          for (int blk = 0; blk < NT / 64; ++blk)
            tma_load_5d(sa + A_BYTES + pl * B_PLANE + blk * BLK, &tmG, full0 + 8u * s, blockIdx.y * NT + blk * 64, 0, h0,
                        n0, pl);
      }
    }
  } else {
    const int g = wg - 1, warp = (tid >> 5) & 3, lane = tid & 31;
    const int unit = g == 0 ? u0 : u1;
    const bool store = (g == 0) || (u1 != u0);
    float acc[NT / 2], d[NT / 2], e[NT / 2];
#pragma unroll
    for (int j = 0; j < NT / 2; ++j) acc[j] = d[j] = e[j] = 0.f;
    for (int i = 0; i < nkb; ++i) {
      const uint32_t s = (uint32_t)i % STAGES, ph = ((uint32_t)i / STAGES) & 1u;
      bar_wait(full0 + 8u * s, ph);
      const uint32_t sa = smem0 + s * STAGE;
      // MN-major operands: 16 pixels = two 8-row atoms = +2048 bytes; the next 64 channels of B are one BLK further
      six_term_kblock<NT, 1, 1>(acc, d, e, sa + (uint32_t)g * BLK, CV_APLANE, sa + A_BYTES, B_PLANE, BLK, 2048u);
      bar_arrive(empty0 + 8u * s);
    }
    if (store) {
      const size_t rows_all = (size_t)p.ntaps * p.Ca;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const size_t my_row = (size_t)unit * 64 + warp * 16 + (lane >> 2) + h * 8;
        const int c0 = blockIdx.y * NT + 2 * (lane & 3);
        if (gridDim.z == 1) {
          // one pixel split: this tile IS the result -- write dW[co][row] (OHWI) directly
#pragma unroll
          for (int j = 0; j < NT / 8; ++j) {
            p.dwout[(size_t)(c0 + 8 * j) * rows_all + my_row] = acc[4 * j + 2 * h];
            p.dwout[(size_t)(c0 + 8 * j + 1) * rows_all + my_row] = acc[4 * j + 2 * h + 1];
          }
        } else {
          float* dst = p.out + ((size_t)blockIdx.z * rows_all + my_row) * p.Cb + c0;
#pragma unroll
          for (int j = 0; j < NT / 8; ++j)
            *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
    }
  }
}

// dw[co][row] = sum_z ws[z][row][co]   (row = tap*Ca + ci; fixed summation order => bitwise reproducible)
__global__ void __launch_bounds__(256) conv_wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw,
                                                                int rows, int Cb, int splits) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8
  const int row0 = blockIdx.x * 32, co0 = blockIdx.y * 32;
  // sum over the splits as four interleaved chains (z mod 4) combined by a fixed tree: 16 loads in flight per thread
  // instead of 4 (the kernel is latency bound), and still bitwise reproducible
  float a4[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < 4; ++c) a4[i][c] = 0.f;
  const size_t zs = (size_t)rows * Cb;
  for (int z0 = 0; z0 < splits; z0 += 4) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (z0 + c < splits) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = row0 + ty + 8 * i;
          if (r < rows) a4[i][c] += __ldg(ws + (size_t)(z0 + c) * zs + (size_t)r * Cb + co0 + tx);
        }
      }
    }
  }
  float acc[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) acc[i] = (a4[i][0] + a4[i][1]) + (a4[i][2] + a4[i][3]);
#pragma unroll
  for (int i = 0; i < 4; ++i) tile[ty + 8 * i][tx] = acc[i];
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + ty + 8 * i, r = row0 + tx;
    if (r < rows) dw[(size_t)co * rows + r] = tile[tx][ty + 8 * i];
  }
}

// ------------------------------------------------------------------------------------------------ fp32 -> 3 x bf16
__device__ __forceinline__ void split3(float x, __nv_bfloat16& a, __nv_bfloat16& b, __nv_bfloat16& c) {
  a = __float2bfloat16_rn(x);
  const float r1 = __fsub_rn(x, __bfloat162float(a));        // exact
  b = __float2bfloat16_rn(r1);
  const float r2 = __fsub_rn(r1, __bfloat162float(b));       // exact
  c = __float2bfloat16_rn(r2);
}

__global__ void __launch_bounds__(256) split3_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                     size_t n8, size_t plane) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
    const F8 x = ld_f8(src + i * 8);
    __nv_bfloat16 a[8], b[8], c[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) split3(x.v[j], a[j], b[j], c[j]);
    *reinterpret_cast<uint4*>(dst + i * 8) = *reinterpret_cast<const uint4*>(a);
    *reinterpret_cast<uint4*>(dst + plane + i * 8) = *reinterpret_cast<const uint4*>(b);
    *reinterpret_cast<uint4*>(dst + 2 * plane + i * 8) = *reinterpret_cast<const uint4*>(c);
  }
}

// Input of a stride-2 conv: x [N][H][W][C] fp32 -> planes [3][4][N][H/2][W/2][C]; sub-image (h%2)*2 + (w%2) holds the
// pixels of that parity, so tap (r,s) of the strided conv is a UNIT-stride box of one sub-image shifted by -1 or 0.
__global__ void __launch_bounds__(256) split3_parity_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                            int N, int H, int W, int C) {
  const int c8 = C / 8;
  const size_t n8 = (size_t)N * H * W * c8, plane = (size_t)N * H * W * C;
  const int H2 = H / 2, W2 = W / 2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
    const size_t pix = i / c8;
    const int cg = (int)(i - pix * c8);
    const int w = (int)(pix % W);
    const size_t t = pix / W;
    const int h = (int)(t % H), n = (int)(t / H);
    const int sub = (h & 1) * 2 + (w & 1);
    const size_t o = ((((size_t)sub * N + n) * H2 + (h >> 1)) * W2 + (w >> 1)) * C + (size_t)cg * 8;
    const F8 x = ld_f8(src + i * 8);
    __nv_bfloat16 a[8], b[8], c[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) split3(x.v[j], a[j], b[j], c[j]);
    *reinterpret_cast<uint4*>(dst + o) = *reinterpret_cast<const uint4*>(a);
    *reinterpret_cast<uint4*>(dst + plane + o) = *reinterpret_cast<const uint4*>(b);
    *reinterpret_cast<uint4*>(dst + 2 * plane + o) = *reinterpret_cast<const uint4*>(c);
  }
}

// Stem (Cin = 3): gather the 27 values (tap, rgb) of every output pixel's 3x3 window into ONE 64-wide K block
// (k = (r*3+s)*3 + c, zero beyond 27 and outside the image): the stem becomes a 1x1 convolution with K = 64.
// x [N][H][W][3] fp32 -> planes [3][N][H][W][64].
__global__ void __launch_bounds__(256) split3_stem_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                          int N, int H, int W) {
  const size_t n8 = (size_t)N * H * W * 8, plane = (size_t)N * H * W * 64;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
    const size_t pix = i >> 3;
    const int g = (int)(i & 7);
    const int w = (int)(pix % W);
    const size_t t = pix / W;
    const int h = (int)(t % H), n = (int)(t / H);
    __nv_bfloat16 a[8], b[8], c[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = g * 8 + j;
      float v = 0.f;
      if (k < 27) {
        const int tap = k / 3, ch = k - tap * 3;
        const int r = tap / 3, sx = tap - r * 3;
        const int hh = h + r - 1, ww = w + sx - 1;
        if (hh >= 0 && hh < H && ww >= 0 && ww < W) v = __ldg(src + (((size_t)n * H + hh) * W + ww) * 3 + ch);
      }
      split3(v, a[j], b[j], c[j]);
    }
    *reinterpret_cast<uint4*>(dst + i * 8) = *reinterpret_cast<const uint4*>(a);
    *reinterpret_cast<uint4*>(dst + plane + i * 8) = *reinterpret_cast<const uint4*>(b);
    *reinterpret_cast<uint4*>(dst + 2 * plane + i * 8) = *reinterpret_cast<const uint4*>(c);
  }
}

// Weights, once per step: w fp32 [Co][T][Ci] (OHWI) -> wp planes [3][Co][T*Ci] (same order: the forward's B operand)
// and, when wtp != null, wtp planes [3][Ci][T*Co] (wt[ci][t][co] = w[co][t][ci]: the data gradient's B operand).
// grid (Ci/32, Co/32, T), 256 threads (32 x 8).
__global__ void __launch_bounds__(256) conv_wprep_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ wp,
                                                         __nv_bfloat16* __restrict__ wtp, int Co, int T, int Ci) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int ci0 = blockIdx.x * 32, co0 = blockIdx.y * 32, t = blockIdx.z;
  const size_t plane = (size_t)Co * T * Ci;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + ty + 8 * i;
    const size_t idx = ((size_t)co * T + t) * Ci + ci0 + tx;
    const float v = __ldg(w + idx);
    tile[ty + 8 * i][tx] = v;
    __nv_bfloat16 a, b, c;
    split3(v, a, b, c);
    wp[idx] = a;
    wp[plane + idx] = b;
    wp[2 * plane + idx] = c;
  }
  if (wtp == nullptr) return;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int ci = ci0 + ty + 8 * i;
    const size_t idx = ((size_t)ci * T + t) * Co + co0 + tx;
    __nv_bfloat16 a, b, c;
    split3(tile[tx][ty + 8 * i], a, b, c);
    wtp[idx] = a;
    wtp[plane + idx] = b;
    wtp[2 * plane + idx] = c;
  }
}

// ------------------------------------------------------------------------------------------------ host side
static bool make_map_act(CUtensorMap* m, const void* base, int C, int W, int H, int N, int planes, int box_w, int box_h,
                         int box_n) {
  EgEncodeTiledFn enc = eg_get_encode_tiled();
  if (enc == nullptr) return false;
  const cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N, (cuuint64_t)planes};
  const cuuint64_t strides[4] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2,
                                 (cuuint64_t)N * H * W * C * 2};
  const cuuint32_t box[5] = {64, (cuuint32_t)box_w, (cuuint32_t)box_h, (cuuint32_t)box_n, 1};
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
static bool make_map_w(CUtensorMap* m, const void* base, uint64_t K, uint64_t rows, uint32_t box_rows) {
  EgEncodeTiledFn enc = eg_get_encode_tiled();
  if (enc == nullptr) return false;
  const cuuint64_t dims[2] = {K, rows};
  const cuuint64_t strides[1] = {K * 2};
  const cuuint32_t box[2] = {64, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// pixel tile of `rows` (128 or 64) rows: full image rows, bh of them, or bn whole images when an image is smaller
static bool tile_geometry(int N, int H, int W, int rows, int* bh, int* bn, int* tiles) {
  if (W < 1 || W > rows || rows % W) return false;
  int h = rows / W;
  if (h > H) h = H;
  if (H % h) return false;
  const int n = rows / (W * h);
  if (W * h * n != rows) return false;
  if (n > 1 && h != H) return false;
  *bh = h;
  *bn = n;
  *tiles = n == 1 ? N * (H / h) : (N + n - 1) / n;
  return true;
}

// (N, H, W) = the pixel grid of the GEMM rows (the conv's OUTPUT grid; dY's grid for a stride-2 data gradient)
bool conv_tc_supported(int N, int H, int W, int Ca, int Cb) {
  int bh, bn, t;
  return N >= 1 && Ca % 64 == 0 && Cb % 64 == 0 && Ca >= 64 && Cb >= 64 && tile_geometry(N, H, W, 128, &bh, &bn, &t) &&
         tile_geometry(N, H, W, 64, &bh, &bn, &t);
}

int conv_wgrad_splits(int N, int H, int W, int Ca, int Cb, int ntaps, int sm_count) {
  int bh, bn, kblocks;
  if (!tile_geometry(N, H, W, 64, &bh, &bn, &kblocks)) return 0;
  const int NT = CV_WGRAD_NT;
  const int U = ntaps * (Ca / 64);
  const int work = ((U + 1) / 2) * (Cb / NT);
  int s = sm_count / work;
  if (s < 1) s = 1;
  if (s > kblocks) s = kblocks;
  return s;
}

static bool taps_ok(const ConvTcParams& p) {
  if (p.ntaps < 1 || p.ntaps > 9 || p.nsrc < 1 || p.nsrc > 4 || p.wtaps < 1 || p.wtaps > 9) return false;
  for (int t = 0; t < p.ntaps; ++t)
    if (p.src[t] < 0 || p.src[t] >= p.nsrc || p.wk[t] < 0 || p.wk[t] >= p.wtaps) return false;
  return true;
}

// K-loop splits of the forward kernel: only when the tiles alone leave most SMs idle (small per-GPU batch).  Counted
// at the 64-wide N tile, which is the one a split launch runs.
int conv_fprop_ksplits(int N, int H, int W, int Ca, int Cb, int ntaps, int sm_count) {
  int bh, bn, m_tiles;
  if (!tile_geometry(N, H, W, 128, &bh, &bn, &m_tiles)) return 0;
  const int NT = 64;
  const int tiles = m_tiles * (Cb / NT), num_kb = ntaps * (Ca / 64);
  if (tiles * 2 > sm_count || num_kb < 4) return 1;
  int ks = sm_count / tiles;
  if (ks > num_kb / 2) ks = num_kb / 2;                     // at least two k-blocks per split
  if (ks < 2) return 1;
  const int per = (num_kb + ks - 1) / ks;
  return (num_kb + per - 1) / per;                          // no empty split
}

int conv_fprop_mtiles(int N, int H, int W) {
  int bh, bn, m_tiles;
  return tile_geometry(N, H, W, 128, &bh, &bn, &m_tiles) ? m_tiles : 0;
}

// N tile of the forward / data-gradient launch.  128 needs Cb % 128 == 0 and an un-split K loop, and the busiest SM
// of the persistent grid must get no more MMA work than at 64: 2 * waves(t) <= waves(2t), t = 128-wide tiles.  A
// 128 x 128 tile does twice the work of a 128 x 64 one at about 1.15x the rate (H100 SXM at 700 W, batch 256:
// 82-84 -> 94-97 fp32-equivalent TFLOP/s), so when the 128-wide grid fills fewer SMs, 64 is faster.  That happens
// to the small grids of the multi-GPU per-GPU batches, e.g. 16x16x128 at batch 32: 64 tiles at 128 vs 128 at 64 on
// 132 SMs, 40 against 64 TFLOP/s measured at 400 W (DESIGN.md section 5a).
int conv_fprop_ntile(int N, int H, int W, int Ca, int Cb, int ntaps, int sm_count) {
  if (Cb % 128 != 0 || sm_count < 1 || conv_fprop_ksplits(N, H, W, Ca, Cb, ntaps, sm_count) != 1) return 64;
  const int t = conv_fprop_mtiles(N, H, W) * (Cb / 128);
  const int waves128 = (t + sm_count - 1) / sm_count, waves64 = (2 * t + sm_count - 1) / sm_count;
  return 2 * waves128 <= waves64 ? 128 : 64;
}

template <int NT, int STAGES, bool ADD>
static cudaError_t fprop_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvTcParams& p, int grid,
                                cudaStream_t s) {
  const size_t smem = (size_t)STAGES * (3 * CV_APLANE + 3 * NT * 128) + 256 + 1024;
  cudaError_t e = cudaFuncSetAttribute(conv3x3_fprop_kernel<NT, STAGES, ADD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  conv3x3_fprop_kernel<NT, STAGES, ADD><<<grid, CV_THREADS, smem, s>>>(tmA, tmB, p);
  return cudaGetLastError();
}

// p.a = activation planes [3][nsrc][N][H][W][Ca], p.b = weight planes [3][Cb][wtaps*Ca], p.out fp32 [N][OH][OW][Cb]
cudaError_t launch_conv_fprop(const ConvTcParams& p0, int sm_count, cudaStream_t s) {
  ConvTcParams p = p0;
  if (!conv_tc_supported(p.N, p.H, p.W, p.Ca, p.Cb) || !taps_ok(p)) return cudaErrorInvalidValue;
  if (p.os < 1 || p.op < 0 || p.oq < 0 || p.op >= p.os || p.oq >= p.os || p.OH < p.H * p.os || p.OW < p.W * p.os)
    return cudaErrorInvalidValue;
  tile_geometry(p.N, p.H, p.W, 128, &p.bh, &p.bn, &p.m_tiles);
  if (p.ksplits < 1 || p.ws == nullptr) p.ksplits = 1;
  if (p.ksplits > 1) {                                      // the caller sized ws with conv_fprop_ksplits()
    const int want = conv_fprop_ksplits(p.N, p.H, p.W, p.Ca, p.Cb, p.ntaps, sm_count);
    if (p.ksplits != want) return cudaErrorInvalidValue;
  }
  CUtensorMap tmA, tmB;
  const int NT = conv_fprop_ntile(p.N, p.H, p.W, p.Ca, p.Cb, p.ntaps, sm_count);
  if (!make_map_w(&tmB, p.b, (uint64_t)p.wtaps * p.Ca, (uint64_t)3 * p.Cb, (uint32_t)NT)) return cudaErrorNotSupported;
  const int total = p.m_tiles * (p.Cb / NT) * p.ksplits;
  const int grid = total < sm_count ? total : sm_count;
  if (!make_map_act(&tmA, p.a, p.Ca, p.W, p.H, p.N, 3 * p.nsrc, p.W, p.bh, p.bn)) return cudaErrorNotSupported;
  eg_count_launch(EG_FAM_CONV, p.ksplits > 1 ? 2 : 1);
  if ((p.addend == nullptr) != (p.addmask == nullptr)) return cudaErrorInvalidValue;
  const bool add = p.addend != nullptr && p.ksplits == 1;   // K-split: the reduce kernel adds it
  cudaError_t e = NT == 128 ? (add ? fprop_launch<128, CV_STAGES(128), true>(tmA, tmB, p, grid, s)
                                   : fprop_launch<128, CV_STAGES(128), false>(tmA, tmB, p, grid, s))
                            : (add ? fprop_launch<64, CV_STAGES(64), true>(tmA, tmB, p, grid, s)
                                   : fprop_launch<64, CV_STAGES(64), false>(tmA, tmB, p, grid, s));
  if (e != cudaSuccess || p.ksplits == 1) return e;
  const long long n4 = (long long)p.N * p.H * p.W * (p.Cb / 4);
  long long blocks = (n4 + 255) / 256;
  if (blocks > sm_count * 8) blocks = sm_count * 8;
  conv_fprop_reduce_kernel<<<(unsigned)blocks, 256, 0, s>>>(p);
  return cudaGetLastError();
}

// The weight gradient runs at the device's lowest priority, also as a node of a captured graph (the attribute is
// recorded on the kernel node).  It is off the critical path: nothing reads dw before the optimizer step, so when an
// SM frees up, a pending CTA of the higher-priority work on the main stream (data gradients, BatchNorm) takes it first.
static cudaLaunchConfig_t low_priority_config(dim3 grid, unsigned block, size_t smem, cudaStream_t s,
                                              cudaLaunchAttribute* attr) {
  int least = 0, greatest = 0;
  cudaDeviceGetStreamPriorityRange(&least, &greatest);
  attr->id = cudaLaunchAttributePriority;
  attr->val.priority = least;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cfg;
}

template <int NT, int STAGES>
static cudaError_t wgrad_launch(const CUtensorMap& tmX, const CUtensorMap& tmG, const ConvTcParams& p, dim3 grid,
                                cudaStream_t s) {
  const size_t smem = (size_t)STAGES * (3 * CV_APLANE + 3 * NT * 128) + 256 + 1024;
  cudaError_t e = cudaFuncSetAttribute(conv3x3_wgrad_kernel<NT, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  cudaLaunchAttribute prio;
  cudaLaunchConfig_t cfg = low_priority_config(grid, CV_THREADS, smem, s, &prio);
  return cudaLaunchKernelEx(&cfg, conv3x3_wgrad_kernel<NT, STAGES>, tmX, tmG, p);
}

// p.a = input planes [3][nsrc][N][H][W][Ca], p.b = dY planes [3][N][H][W][Cb], p.out = workspace
// [splits][ntaps*Ca][Cb], dw = [Cb][ntaps][Ca] (OHWI)
cudaError_t launch_conv_wgrad(const ConvTcParams& p0, float* dw, int splits, cudaStream_t s) {
  ConvTcParams p = p0;
  if (!conv_tc_supported(p.N, p.H, p.W, p.Ca, p.Cb) || !taps_ok(p) || splits < 1) return cudaErrorInvalidValue;
  tile_geometry(p.N, p.H, p.W, 64, &p.bh, &p.bn, &p.k_blocks);
  if (splits > p.k_blocks) splits = p.k_blocks;
  CUtensorMap tmX, tmG;
  const int NT = CV_WGRAD_NT;
  if (!make_map_act(&tmX, p.a, p.Ca, p.W, p.H, p.N, 3 * p.nsrc, p.W, p.bh, p.bn)) return cudaErrorNotSupported;
  if (!make_map_act(&tmG, p.b, p.Cb, p.W, p.H, p.N, 3, p.W, p.bh, p.bn)) return cudaErrorNotSupported;
  const int U = p.ntaps * (p.Ca / 64);
  const dim3 grid((U + 1) / 2, p.Cb / NT, splits);
  p.dwout = dw;
  eg_count_launch(EG_FAM_CONV, splits > 1 ? 2 : 1);
  cudaError_t e = wgrad_launch<CV_WGRAD_NT, CV_STAGES(CV_WGRAD_NT)>(tmX, tmG, p, grid, s);
  if (e != cudaSuccess || splits == 1) return e;
  const int rows = p.ntaps * p.Ca;
  cudaLaunchAttribute prio;
  cudaLaunchConfig_t cfg = low_priority_config(dim3((rows + 31) / 32, p.Cb / 32), 256, 0, s, &prio);
  return cudaLaunchKernelEx(&cfg, conv_wgrad_reduce_kernel, (const float*)p.out, dw, rows, p.Cb, splits);
}

// (kind, priority) of every kernel node of a captured graph; kind: 1 = weight gradient (or its reduce), 2 = forward /
// data gradient (or its reduce), 0 = any other kernel.  For tests: the priorities must be in the graph, not only in
// eager launches.
cudaError_t conv_graph_kernel_priorities(cudaGraph_t g, std::vector<std::pair<int, int>>* out) {
  size_t n = 0;
  cudaError_t e = cudaGraphGetNodes(g, nullptr, &n);
  if (e != cudaSuccess) return e;
  std::vector<cudaGraphNode_t> nodes(n);
  if (n && (e = cudaGraphGetNodes(g, nodes.data(), &n)) != cudaSuccess) return e;
  const void* wgrad_fns[] = {(const void*)conv3x3_wgrad_kernel<CV_WGRAD_NT, CV_STAGES(CV_WGRAD_NT)>,
                             (const void*)conv_wgrad_reduce_kernel};
  const void* fprop_fns[] = {(const void*)conv3x3_fprop_kernel<128, CV_STAGES(128), true>,
                             (const void*)conv3x3_fprop_kernel<128, CV_STAGES(128), false>,
                             (const void*)conv3x3_fprop_kernel<64, CV_STAGES(64), true>,
                             (const void*)conv3x3_fprop_kernel<64, CV_STAGES(64), false>,
                             (const void*)conv_fprop_reduce_kernel};
  auto is = [](const void* f, const void* const* fns, int k) {
    for (int i = 0; i < k; ++i) {
      cudaFunction_t h = nullptr;
      if (f == fns[i] || (cudaGetFuncBySymbol(&h, fns[i]) == cudaSuccess && f == (const void*)h)) return true;
    }
    return false;
  };
  for (size_t i = 0; i < n; ++i) {
    cudaGraphNodeType t;
    if ((e = cudaGraphNodeGetType(nodes[i], &t)) != cudaSuccess) return e;
    if (t != cudaGraphNodeTypeKernel) continue;
    cudaLaunchAttributeValue v = {};
    if ((e = cudaGraphKernelNodeGetAttribute(nodes[i], cudaLaunchAttributePriority, &v)) != cudaSuccess) return e;
    // a kernel that another library launched through the driver API has no runtime entry: it is none of ours
    cudaKernelNodeParams kp = {};
    int kind = 0;
    if (cudaGraphKernelNodeGetParams(nodes[i], &kp) == cudaSuccess)
      kind = is(kp.func, wgrad_fns, 2) ? 1 : is(kp.func, fprop_fns, 5) ? 2 : 0;
    else
      cudaGetLastError();
    out->emplace_back(kind, v.priority);
  }
  return cudaSuccess;
}

static unsigned split_blocks(size_t n8) {
  size_t blocks = (n8 + 255) / 256;
  if (blocks > CV_SMS * 16) blocks = CV_SMS * 16;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

cudaError_t launch_split3(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t s) {
  if (n % 8) return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_CONV, 1);
  split3_kernel<<<split_blocks(n / 8), 256, 0, s>>>(src, dst, n / 8, n);
  return cudaGetLastError();
}

cudaError_t launch_split3_parity(const float* src, __nv_bfloat16* dst, int N, int H, int W, int C, cudaStream_t s) {
  if (C % 8 || H % 2 || W % 2) return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_CONV, 1);
  split3_parity_kernel<<<split_blocks((size_t)N * H * W * C / 8), 256, 0, s>>>(src, dst, N, H, W, C);
  return cudaGetLastError();
}

cudaError_t launch_split3_stem(const float* src, __nv_bfloat16* dst, int N, int H, int W, cudaStream_t s) {
  eg_count_launch(EG_FAM_CONV, 1);
  split3_stem_kernel<<<split_blocks((size_t)N * H * W * 8), 256, 0, s>>>(src, dst, N, H, W);
  return cudaGetLastError();
}

cudaError_t launch_conv_wprep(const float* w, __nv_bfloat16* wp, __nv_bfloat16* wtp, int Co, int T, int Ci, cudaStream_t s) {
  if (Co % 32 || Ci % 32 || T < 1) return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_CONV, 1);
  conv_wprep_kernel<<<dim3(Ci / 32, Co / 32, T), 256, 0, s>>>(w, wp, wtp, Co, T, Ci);
  return cudaGetLastError();
}

}  // namespace egb
