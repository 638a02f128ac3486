// Decoded video samples -> the bytes the reference writes: src/utils/util.py:87-104 save_videos_grid does
// `(x * 255).numpy().astype(np.uint8)`, after `(x + 1) / 2` if rescale, on an fp32 host tensor (the fp16 video widened,
// or the frame interpolator's fp32 output). Same fp32 operations in the same order (no fma contraction), truncation
// toward zero -> bit-identical bytes for values in range; out-of-range values saturate (the numpy cast is undefined
// there), NaN -> 0. Shared by ap_pack_frames_u8 and ap_video_grid_u8.
#pragma once
#include <cuda_fp16.h>

namespace ap {

__device__ __forceinline__ unsigned to_u8(float x, int rescale) {
  if (rescale) x = __fmul_rn(__fadd_rn(x, 1.f), 0.5f);
  return min(__float2uint_rz(__fmul_rn(x, 255.f)), 255u);   // cvt.rzi.u32.f32 saturates: negative and NaN -> 0
}

__device__ __forceinline__ unsigned to_u8(__half h, int rescale) { return to_u8(__half2float(h), rescale); }

}  // namespace ap
