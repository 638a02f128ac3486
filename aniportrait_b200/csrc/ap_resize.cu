// cv2.resize(img, (W, H)) with the default INTER_LINEAR on uint8 3-channel frames, byte-identical to OpenCV's fixed-point
// kernel: what the reference's FaceMeshVisualizer.draw_landmarks (src/utils/draw_util.py:146) does to its 512 x 512 canvas,
// and what scripts/vid2vid.py:199-200 does once more to the result. tests/resize_reference.py states the arithmetic.
#include <limits.h>
#include <stdint.h>

#include "ap_host.h"
#include "ap_ptx.cuh"

namespace ap {

// ---------------------------------------------------------------------------------------------------------
// One CTA per (frame, band of kResizeRows destination rows), frame-major on a 1-D grid, one thread per destination pixel
// (all three channels). The row taps of the band are computed once into shared memory, the column taps per thread.
// Two-stage mode (src -> mid -> dst): each of the 2 x 2 mid pixels a destination pixel reads is recomputed from its own
// 2 x 2 source texels and rounded to uint8 exactly as the stored mid image would be; neighbouring threads read the same
// source rows, which stay in L1 / L2.
// ---------------------------------------------------------------------------------------------------------
constexpr int kResizeRows = 8;
constexpr int kResizeThreads = 256;
constexpr int kCoefScale = 2048;   // INTER_RESIZE_COEF_SCALE: 11-bit coefficients

struct Tap {
  int i0, i1;   // the two source indices (clipped to [0, n - 1])
  int c0, c1;   // their fixed-point weights
};

// Destination index d of an axis resized from n samples with scale = 1 / (dst / n). Every operation is rounded on its own
// (no FMA contraction): f = (float)((d + 0.5) * scale - 0.5), s = floor(f), f -= s. Columns (clamp_f) pin s and f = 0 at
// both borders; rows keep f and only clip the two indices.
__device__ __forceinline__ Tap linear_tap(int d, int n, double scale, bool clamp_f) {
  const float fd = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
  int s = __float2int_rd(fd);
  float f = __fsub_rn(fd, (float)s);
  if (clamp_f) {
    if (s < 0) s = 0, f = 0.f;
    if (s >= n - 1) s = n - 1, f = 0.f;
  }
  Tap t;
  t.c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), (float)kCoefScale));
  t.c1 = __float2int_rn(__fmul_rn(f, (float)kCoefScale));
  t.i0 = min(max(s, 0), n - 1);
  t.i1 = min(max(s + 1, 0), n - 1);
  return t;
}

// cv2's vectorised vertical pass (VResizeLinearVec_32s8u): int16 high halves of (H >> 4) * beta, then (sum + 2) >> 2,
// saturated. Every term is >= 0.
__device__ __forceinline__ int vertical(int h0, int h1, int b0, int b1) {
  return min(((((h0 >> 4) * b0) >> 16) + (((h1 >> 4) * b1) >> 16) + 2) >> 2, 255);
}

// One resized pixel (3 channels) of the uint8 image `img` (w pixels per row) under column tap x and row tap y.
__device__ __forceinline__ void sample(const uint8_t* __restrict__ img, int w, const Tap& x, const Tap& y, int out[3]) {
  const uint8_t* r0 = img + (long long)y.i0 * w * 3;
  const uint8_t* r1 = img + (long long)y.i1 * w * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = __ldg(r0 + x.i0 * 3 + c) * x.c0 + __ldg(r0 + x.i1 * 3 + c) * x.c1;
    const int h1 = __ldg(r1 + x.i0 * 3 + c) * x.c0 + __ldg(r1 + x.i1 * 3 + c) * x.c1;
    out[c] = vertical(h0, h1, y.c0, y.c1);
  }
}

struct ResizeStage {
  int w, h;            // source size of the stage
  double sx, sy;       // 1 / (dst / src) per axis
};

template <bool kChain>
__global__ void __launch_bounds__(kResizeThreads)
resize_linear_u8_kernel(const uint8_t* __restrict__ src, ResizeStage first, ResizeStage second, int dst_w, int dst_h,
                        uint8_t* __restrict__ dst) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  // the last stage's row taps and, chained, the first stage's row taps of its two mid rows
  __shared__ Tap rows[kResizeRows][3];
  const int bands = (dst_h + kResizeRows - 1) / kResizeRows;
  const int f = blockIdx.x / bands;
  const int y0 = blockIdx.x % bands * kResizeRows;
  const int nrows = min(kResizeRows, dst_h - y0);
  const ResizeStage& last = kChain ? second : first;
  if (threadIdx.x < nrows) {
    const Tap t = linear_tap(y0 + threadIdx.x, last.h, last.sy, false);
    rows[threadIdx.x][0] = t;
    if (kChain) {
      rows[threadIdx.x][1] = linear_tap(t.i0, first.h, first.sy, false);
      rows[threadIdx.x][2] = linear_tap(t.i1, first.h, first.sy, false);
    }
  }
  __syncthreads();
  griddep_wait();

  const uint8_t* img = src + (long long)f * first.h * first.w * 3;
  uint8_t* out = dst + ((long long)f * dst_h + y0) * dst_w * 3;
  for (int x = threadIdx.x; x < dst_w; x += kResizeThreads) {
    const Tap tx = linear_tap(x, last.w, last.sx, true);
    Tap ta, tb;   // chained: the first stage's column taps of the two mid columns
    if (kChain) {
      ta = linear_tap(tx.i0, first.w, first.sx, true);
      tb = linear_tap(tx.i1, first.w, first.sx, true);
    }
    for (int r = 0; r < nrows; ++r) {
      int v[3];
      if (kChain) {
        int m00[3], m01[3], m10[3], m11[3];   // mid pixels (row tap, column tap)
        sample(img, first.w, ta, rows[r][1], m00);
        sample(img, first.w, tb, rows[r][1], m01);
        sample(img, first.w, ta, rows[r][2], m10);
        sample(img, first.w, tb, rows[r][2], m11);
#pragma unroll
        for (int c = 0; c < 3; ++c)
          v[c] = vertical(m00[c] * tx.c0 + m01[c] * tx.c1, m10[c] * tx.c0 + m11[c] * tx.c1, rows[r][0].c0, rows[r][0].c1);
      } else {
        sample(img, first.w, tx, rows[r][0], v);
      }
      uint8_t* o = out + ((long long)r * dst_w + x) * 3;
      o[0] = (uint8_t)v[0];
      o[1] = (uint8_t)v[1];
      o[2] = (uint8_t)v[2];
    }
  }
}

static ResizeStage make_stage(int w, int h, int to_w, int to_h) {
  return ResizeStage{w, h, 1.0 / ((double)to_w / w), 1.0 / ((double)to_h / h)};
}

static bool side_ok(int v) { return v >= 1 && v <= AP_RESIZE_MAX_SIDE; }

}  // namespace ap

extern "C" int ap_resize_linear_u8(const void* src, int L, int src_w, int src_h, int mid_w, int mid_h, int dst_w,
                                   int dst_h, void* dst, void* stream) {
  AP_REQUIRE(src && dst && L > 0, "resize_linear_u8: bad arguments");
  AP_REQUIRE(ap::side_ok(src_w) && ap::side_ok(src_h) && ap::side_ok(dst_w) && ap::side_ok(dst_h),
             "resize_linear_u8: %dx%d -> %dx%d: every side must lie in [1, %d]", src_w, src_h, dst_w, dst_h,
             AP_RESIZE_MAX_SIDE);
  const bool chain = mid_w != 0 || mid_h != 0;
  AP_REQUIRE(!chain || (ap::side_ok(mid_w) && ap::side_ok(mid_h)),
             "resize_linear_u8: intermediate size %dx%d: both sides 0 (one resize) or in [1, %d]", mid_w, mid_h,
             AP_RESIZE_MAX_SIDE);
  const long long ctas = (long long)L * ((dst_h + ap::kResizeRows - 1) / ap::kResizeRows);
  AP_REQUIRE(ctas <= INT_MAX, "resize_linear_u8: %d frames of %d rows exceed one launch", L, dst_h);
  if (chain) {
    const ap::ResizeStage first = ap::make_stage(src_w, src_h, mid_w, mid_h);
    const ap::ResizeStage second = ap::make_stage(mid_w, mid_h, dst_w, dst_h);
    AP_LAUNCH((ap::resize_linear_u8_kernel<true>), (unsigned)ctas, ap::kResizeThreads, 0, (cudaStream_t)stream,
              (const uint8_t*)src, first, second, dst_w, dst_h, (uint8_t*)dst);
  } else {
    const ap::ResizeStage first = ap::make_stage(src_w, src_h, dst_w, dst_h);
    AP_LAUNCH((ap::resize_linear_u8_kernel<false>), (unsigned)ctas, ap::kResizeThreads, 0, (cudaStream_t)stream,
              (const uint8_t*)src, first, first, dst_w, dst_h, (uint8_t*)dst);
  }
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}
