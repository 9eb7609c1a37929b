// eventgrad_b200 -- fused decode + augmentation of a uint8 image batch (sm_90a).
// ConstantPad(4) -> RandomHorizontalFlip -> RandomCrop(HxW) of the reference
// (/root/reference/dcifar10/common/transform.hpp:68-101) collapse into one gather, fused with
// the uint8->float conversion, normalisation, optional bf16 cast and NCHW->NHWC relayout:
//   out[b,c,y,x] = padded[b,c, y+oy_b, flip_b ? (W+2p-1)-(x+ox_b) : x+ox_b]
#include "api.h"
#include "common.cuh"

namespace egb {

template <bool kBf16, bool kNhwc>
__global__ void __launch_bounds__(256) decode_augment_kernel(const uint8_t* __restrict__ in, void* out,
                                                             const int* __restrict__ oy,
                                                             const int* __restrict__ ox,
                                                             const int* __restrict__ flip, int B, int C,
                                                             int H, int W, int pad, float scale,
                                                             float mean, float inv_std) {
  const int n = B * H * W;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    const int x = p % W, y = (p / W) % H, b = p / (W * H);
    int sy = y, sx = x;
    if (oy != nullptr) {
      sy = y + oy[b] - pad;
      int px = x + ox[b];
      if (flip[b]) px = (W + 2 * pad - 1) - px;
      sx = px - pad;
    }
    const bool inside = (sy >= 0) && (sy < H) && (sx >= 0) && (sx < W);
    for (int c = 0; c < C; ++c) {
      float v = 0.f;
      if (inside) v = (float)in[(((size_t)b * C + c) * H + sy) * W + sx];
      v = (v * scale - mean) * inv_std;
      const size_t o = kNhwc ? ((((size_t)b * H + y) * W + x) * C + c) : ((((size_t)b * C + c) * H + y) * W + x);
      if (kBf16)
        reinterpret_cast<__nv_bfloat16*>(out)[o] = __float2bfloat16_rn(v);
      else
        reinterpret_cast<float*>(out)[o] = v;
    }
  }
}

cudaError_t launch_decode_augment(const uint8_t* in, void* out, const int* oy, const int* ox,
                                  const int* flip, int B, int C, int H, int W, int pad, float scale,
                                  float mean, float inv_std, int out_bf16, int nhwc, cudaStream_t s) {
  const int n = B * H * W;
  if (n == 0) return cudaSuccess;
  const int grid = (n + 255) / 256;
  eg_count_launch(EG_FAM_DATA, 1);
#define EG_AUG(BF, NH) \
  decode_augment_kernel<BF, NH><<<grid, 256, 0, s>>>(in, out, oy, ox, flip, B, C, H, W, pad, scale, mean, inv_std)
  if (out_bf16) {
    if (nhwc) EG_AUG(true, true); else EG_AUG(true, false);
  } else {
    if (nhwc) EG_AUG(false, true); else EG_AUG(false, false);
  }
#undef EG_AUG
  return cudaGetLastError();
}

}  // namespace egb
