// eventgrad_b200 -- wgmma fused Linear+bias(+ReLU): TMA + 128-byte swizzle, persistent CTAs, warp-specialised
// (sm_90a).
//
// A single thread issues `cp.async.bulk.tensor.2d` (TMA) for 128-byte-wide boxes into a 128B-swizzled ring; two MMA
// warpgroups each own 64 rows of the 128-row tile, run wgmma.mma_async against SWIZZLE_128B descriptors with the
// accumulator in registers, and apply bias + ReLU in the register epilogue:
//
//   warpgroup 0    TMA producer   full[s]  <- expect_tx + 2 bulk tensor loads (A 128x64, B Nx64 bf16)
//   warpgroup 1-2  MMA            wait full[s]; 4 K steps x NC wgmma (K=16 each, +32 B inside the swizzle atom);
//                                 keep one k-block in flight, release the previous stage -> empty[s];
//                                 per tile: bias + ReLU on the registers, stores
//
// N is covered by NC wgmma of width CH (N <= 64: one n64; N <= 128: one n128; N <= 256: two n128).  B rows past N are
// never loaded; the columns they produce are computed from stale shared memory and discarded.
#include <cuda.h>

#include "api.h"
#include "common.cuh"
#include "tc_common.cuh"

namespace egb {
using namespace tc;

#define TM_ROWS 128
#define TM_BK 64
#define TM_STAGES 4
#define TM_THREADS 384
#define TM_CONSUMERS 256

template <int CH, int NC, bool kOutBf16>
__global__ void __launch_bounds__(TM_THREADS, 1)
linear_tma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const LinearParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  constexpr uint32_t A_BYTES = TM_ROWS * TM_BK * 2, B_BYTES = CH * NC * TM_BK * 2, STAGE = A_BYTES + B_BYTES;
  const int tid = threadIdx.x, wg = tid >> 7;
  const int N = p.N;
  const uint32_t tx_bytes = A_BYTES + (uint32_t)N * TM_BK * 2;
  // SWIZZLE_128B atoms (TMA destination and wgmma descriptors, base offset 0) need 1024-byte aligned tiles;
  // the dynamic-smem base is only guaranteed 16-byte aligned, so round up (the launcher adds 1 KB of slack)
  const uint32_t smem_unaligned = s_u32(smem_raw);
  const uint32_t smem0 = (smem_unaligned + 1023u) & ~1023u;
  unsigned char* smem_al = smem_raw + (smem0 - smem_unaligned);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_al + TM_STAGES * STAGE);
  const uint32_t full0 = s_u32(bars), empty0 = full0 + 8u * TM_STAGES;
  const int n_tiles = (p.M + TM_ROWS - 1) / TM_ROWS;
  const int num_kb = (p.K + TM_BK - 1) / TM_BK;

  if (tid == 0) {
    for (int i = 0; i < TM_STAGES; ++i) {
      bar_init(full0 + 8u * i, 1);                 // producer's arrive.expect_tx (+ transaction bytes)
      bar_init(empty0 + 8u * i, TM_CONSUMERS);     // every MMA thread, once its wgmma reading the stage completed
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA PRODUCER (one thread) =====================
    if (tid == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const uint32_t s = it % TM_STAGES, ph = (it / TM_STAGES) & 1u;
          bar_wait(empty0 + 8u * s, ph ^ 1u);                   // slot free (fresh barrier: passes at once)
          bar_expect_tx(full0 + 8u * s, tx_bytes);
          const uint32_t sa = smem0 + s * STAGE;
          tma_load_2d(sa, &tmA, full0 + 8u * s, kb * TM_BK, tile * TM_ROWS);   // OOB rows / K tail are zero-filled
          tma_load_2d(sa + A_BYTES, &tmB, full0 + 8u * s, kb * TM_BK, 0);
        }
      }
    }
  } else {
    // ===================== MMA + EPILOGUE (rows 64g .. 64g+63 of every tile) =====================
    const int g = wg - 1, warp = (tid >> 5) & 3, lane = tid & 31;
    float d[NC][CH / 2];
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      uint32_t prev = 0;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const uint32_t s = it % TM_STAGES, ph = (it / TM_STAGES) & 1u;
        bar_wait(full0 + 8u * s, ph);                           // TMA bytes have landed
        const uint32_t sa = smem0 + s * STAGE;
        wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < TM_BK / 16; ++k4) {
          const uint64_t da = desc_k_sw128(sa + (uint32_t)g * 8192u) + (uint64_t)(k4 * 2);   // +32 B in the atom
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            const uint64_t db = desc_k_sw128(sa + A_BYTES + (uint32_t)c * CH * 128u) + (uint64_t)(k4 * 2);
            const uint32_t accum = (kb > 0 || k4 > 0) ? 1u : 0u;
            if constexpr (CH == 128) wgmma_m64n128<0, 0>(d[c], da, db, accum);
            else wgmma_m64n64<0, 0>(d[c], da, db, accum);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                                        // the k-block before this one has completed
        if (kb > 0) bar_arrive(empty0 + 8u * prev);
        prev = s;
      }
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < NC; ++c) wgmma_fence_regs(d[c]);
      bar_arrive(empty0 + 8u * prev);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = tile * TM_ROWS + g * 64 + warp * 16 + (lane >> 2) + h * 8;
        if (row >= p.M) continue;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
#pragma unroll
          for (int j = 0; j < CH / 8; ++j) {
            const int col = c * CH + 8 * j + 2 * (lane & 3);
            if (col >= N) continue;
            float v0 = d[c][4 * j + 2 * h], v1 = d[c][4 * j + 2 * h + 1];
            if (p.bias) { v0 += __ldg(p.bias + col); v1 += __ldg(p.bias + col + 1); }
            if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (kOutBf16)
              *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.y) + (size_t)row * N + col) =
                  __floats2bfloat162_rn(v0, v1);
            else
              *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.y) + (size_t)row * N + col) = make_float2(v0, v1);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
static bool make_map(CUtensorMap* m, const void* base, uint64_t rows, uint64_t K, uint32_t box_rows) {
  EgEncodeTiledFn enc = eg_get_encode_tiled();
  if (enc == nullptr) return false;
  const cuuint64_t dims[2] = {K, rows};                    // innermost first
  const cuuint64_t strides[1] = {K * 2};                   // bytes, dims 1..rank-1
  const cuuint32_t box[2] = {TM_BK, box_rows};             // 64 elements = 128 B == the swizzle span
  const cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int CH, int NC>
static cudaError_t linear_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const LinearParams& p, int grid,
                                 cudaStream_t s) {
  const size_t smem = (size_t)TM_STAGES * ((size_t)TM_ROWS * TM_BK * 2 + (size_t)CH * NC * TM_BK * 2) + 256 + 1024;
  cudaError_t e;
  if (p.out_bf16) {
    e = cudaFuncSetAttribute(linear_tma_kernel<CH, NC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    linear_tma_kernel<CH, NC, true><<<grid, TM_THREADS, smem, s>>>(tmA, tmB, p);
  } else {
    e = cudaFuncSetAttribute(linear_tma_kernel<CH, NC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    linear_tma_kernel<CH, NC, false><<<grid, TM_THREADS, smem, s>>>(tmA, tmB, p);
  }
  return cudaGetLastError();
}

cudaError_t launch_linear_tc_tma(const LinearParams& p, int sm_count, cudaStream_t s) {
  if (p.N % 16 != 0 || p.N < 16 || p.N > 256 || p.K % 8 != 0 || p.M < 1) return cudaErrorInvalidValue;
  CUtensorMap tmA, tmB;
  if (!make_map(&tmA, p.x, (uint64_t)p.M, (uint64_t)p.K, TM_ROWS)) return cudaErrorNotSupported;
  if (!make_map(&tmB, p.w, (uint64_t)p.N, (uint64_t)p.K, (uint32_t)p.N)) return cudaErrorNotSupported;
  const int n_tiles = (p.M + TM_ROWS - 1) / TM_ROWS;
  const int grid = n_tiles < sm_count ? n_tiles : sm_count;
  eg_count_launch(EG_FAM_LINEAR, 1);
  if (p.N <= 64) return linear_launch<64, 1>(tmA, tmB, p, grid, s);
  if (p.N <= 128) return linear_launch<128, 1>(tmA, tmB, p, grid, s);
  return linear_launch<128, 2>(tmA, tmB, p, grid, s);
}

}  // namespace egb
