// Pillow's Image.resize(size, Image.BILINEAR) on RGB frames, byte-identical to its 8-bit resampler (libImaging/Resample.c):
// what the scripts' transforms.Resize((height, width)) does to every frame of the comparison grid (reference
// scripts/audio2vid.py:207-210, vid2vid.py:147-162, pose2vid.py:146-151). tests/pil_resize_reference.py states the
// arithmetic.
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include "ap_host.h"
#include "ap_ptx.cuh"

namespace ap {

// ---------------------------------------------------------------------------------------------------------
// One CTA per (frame, band of kPilRows output rows, tile of kPilCols output columns), on a 1-D grid. The CTA computes the
// coefficients of its columns and rows into shared memory, runs the horizontal pass over the source rows its band reads
// into a shared uint8 tile (Pillow stores that intermediate as uint8, and the rounding is part of the result), then the
// vertical pass. Neighbouring bands recompute the few source rows they share.
// Coefficients are computed on the device in double, each operation rounded on its own (no FMA contraction), in Pillow's
// order: the C ABI then needs no coefficient table from its caller, and the cost is a few hundred double operations per
// CTA against tens of thousands of pixel products.
// ---------------------------------------------------------------------------------------------------------
constexpr int kPilRows = 16;
constexpr int kPilCols = 64;
constexpr int kPilThreads = 256;
constexpr int kPilBits = 22;   // PRECISION_BITS = 32 - 8 - 2

struct PilAxis {
  int in, out;
  double scale;   // in / out
  double fs;      // max(scale, 1): the filter scale, also the support (bilinear support 1)
  double ss;      // 1 / fs
  int ksize;      // 2 ceil(fs) + 1: the most taps an index can have
};

static PilAxis make_axis(int in, int out) {
  PilAxis a;
  a.in = in;
  a.out = out;
  a.scale = (double)in / out;
  a.fs = a.scale < 1.0 ? 1.0 : a.scale;
  a.ss = 1.0 / a.fs;
  a.ksize = (int)ceil(a.fs) * 2 + 1;
  return a;
}

// precompute_coeffs + normalize_coeffs_8bpc for output index xx: writes the taps' fixed-point weights to k[0 .. n) and
// returns n; *first = the first source index. The weights are evaluated twice (for the sum, then for the division) rather
// than stored: the same operations give the same doubles.
__device__ __forceinline__ int pil_coeffs(int xx, const PilAxis& a, int* k, int* first) {
  const double center = __dmul_rn((double)xx + 0.5, a.scale);
  const int lo = max(__double2int_rz(__dadd_rn(__dsub_rn(center, a.fs), 0.5)), 0);
  const int n = min(__double2int_rz(__dadd_rn(__dadd_rn(center, a.fs), 0.5)), a.in) - lo;
  double ww = 0.0;
  for (int x = 0; x < n; ++x) {
    const double t = fabs(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + lo), center), 0.5), a.ss));
    ww = __dadd_rn(ww, t < 1.0 ? __dsub_rn(1.0, t) : 0.0);
  }
  for (int x = 0; x < n; ++x) {
    const double t = fabs(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + lo), center), 0.5), a.ss));
    double w = t < 1.0 ? __dsub_rn(1.0, t) : 0.0;
    if (ww != 0.0) w = __ddiv_rn(w, ww);
    k[x] = __double2int_rz(__dadd_rn(0.5, __dmul_rn(w, (double)(1 << kPilBits))));   // w >= 0 for this filter
  }
  *first = lo;
  return n;
}

// clip8 of Resample.c: sums start at 2^21, so the shift rounds to nearest
__device__ __forceinline__ uint8_t clip8(int v) { return (uint8_t)min(max(v >> kPilBits, 0), 255); }

__global__ void __launch_bounds__(kPilThreads)
resize_pil_u8_kernel(const uint8_t* __restrict__ src, PilAxis ax, PilAxis ay, int need_h, int need_v, int col_tiles,
                     int bands, uint8_t* __restrict__ dst) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  extern __shared__ int4 pil_smem[];
  int* kx = reinterpret_cast<int*>(pil_smem);   // [kPilCols][ax.ksize]
  int* ky = kx + kPilCols * ax.ksize;           // [kPilRows][ay.ksize]
  int* bx = ky + kPilRows * ay.ksize;           // [kPilCols][2]: first source column, taps
  int* by = bx + 2 * kPilCols;                  // [kPilRows][2]: first source row, taps
  uint8_t* mid = reinterpret_cast<uint8_t*>(by + 2 * kPilRows);   // [rows][kPilCols * 3]

  const int tile = blockIdx.x % col_tiles;
  const int band = blockIdx.x / col_tiles % bands;
  const long long f = blockIdx.x / (col_tiles * bands);
  const int x0 = tile * kPilCols, y0 = band * kPilRows;
  const int ncols = min(kPilCols, ax.out - x0), nrows = min(kPilRows, ay.out - y0);
  const int tid = threadIdx.x;
  if (need_h && tid < ncols) bx[2 * tid + 1] = pil_coeffs(x0 + tid, ax, kx + tid * ax.ksize, bx + 2 * tid);
  if (need_v && tid >= kPilCols && tid < kPilCols + nrows) {
    const int r = tid - kPilCols;
    by[2 * r + 1] = pil_coeffs(y0 + r, ay, ky + r * ay.ksize, by + 2 * r);
  }
  __syncthreads();
  // the source rows the band reads: [row0, row0 + rows)
  const int row0 = need_v ? by[0] : y0;
  const int rows = need_v ? by[2 * (nrows - 1)] + by[2 * (nrows - 1) + 1] - row0 : nrows;
  griddep_wait();

  const uint8_t* img = src + f * ay.in * ax.in * 3;
  for (int i = tid; i < rows * ncols; i += kPilThreads) {
    const int r = i / ncols, c = i % ncols;
    const uint8_t* s = img + (long long)(row0 + r) * ax.in * 3;
    uint8_t* m = mid + (r * kPilCols + c) * 3;
    if (need_h) {
      const int* k = kx + c * ax.ksize;
      const uint8_t* p = s + bx[2 * c] * 3;
      const int n = bx[2 * c + 1];
      int s0 = 1 << (kPilBits - 1), s1 = s0, s2 = s0;
      for (int x = 0; x < n; ++x) {
        const int w = k[x];
        s0 += __ldg(p + 3 * x) * w;
        s1 += __ldg(p + 3 * x + 1) * w;
        s2 += __ldg(p + 3 * x + 2) * w;
      }
      m[0] = clip8(s0);
      m[1] = clip8(s1);
      m[2] = clip8(s2);
    } else {
      const uint8_t* p = s + (x0 + c) * 3;
      m[0] = __ldg(p);
      m[1] = __ldg(p + 1);
      m[2] = __ldg(p + 2);
    }
  }
  __syncthreads();

  uint8_t* out = dst + (f * ay.out + y0) * ax.out * 3;
  for (int i = tid; i < nrows * ncols; i += kPilThreads) {
    const int r = i / ncols, c = i % ncols;
    uint8_t* o = out + ((long long)r * ax.out + x0 + c) * 3;
    if (need_v) {
      const int* k = ky + r * ay.ksize;
      const uint8_t* m = mid + ((by[2 * r] - row0) * kPilCols + c) * 3;
      const int n = by[2 * r + 1];
      int s0 = 1 << (kPilBits - 1), s1 = s0, s2 = s0;
      for (int y = 0; y < n; ++y) {
        const int w = k[y];
        s0 += m[y * kPilCols * 3] * w;
        s1 += m[y * kPilCols * 3 + 1] * w;
        s2 += m[y * kPilCols * 3 + 2] * w;
      }
      o[0] = clip8(s0);
      o[1] = clip8(s1);
      o[2] = clip8(s2);
    } else {
      const uint8_t* m = mid + (r * kPilCols + c) * 3;
      o[0] = m[0];
      o[1] = m[1];
      o[2] = m[2];
    }
  }
}

// Source rows a band of kPilRows output rows reads, at most: the span (last first row + its taps) - first row is below
// (kPilRows - 1) scale + 2 support + 1 (see the bounds in pil_coeffs); one row of margin on top.
static int pil_band_rows(const PilAxis& a) {
  const int bound = (int)ceil((kPilRows - 1) * a.scale + 2.0 * a.fs + 2.0);
  return bound < a.in ? bound : a.in;
}

static bool pil_side_ok(int v) { return v >= 1 && v <= AP_RESIZE_MAX_SIDE; }

}  // namespace ap

extern "C" int ap_resize_pil_bilinear_u8(const void* src, int L, int src_w, int src_h, int dst_w, int dst_h, void* dst,
                                         void* stream) {
  AP_REQUIRE(src && dst && L > 0, "resize_pil_bilinear_u8: bad arguments");
  AP_REQUIRE(ap::pil_side_ok(src_w) && ap::pil_side_ok(src_h) && ap::pil_side_ok(dst_w) && ap::pil_side_ok(dst_h),
             "resize_pil_bilinear_u8: %dx%d -> %dx%d: every side must lie in [1, %d]", src_w, src_h, dst_w, dst_h,
             AP_RESIZE_MAX_SIDE);
  AP_REQUIRE((long long)src_w <= (long long)AP_RESIZE_PIL_MAX_SCALE * dst_w &&
                 (long long)src_h <= (long long)AP_RESIZE_PIL_MAX_SCALE * dst_h,
             "resize_pil_bilinear_u8: %dx%d -> %dx%d shrinks an axis by more than %dx", src_w, src_h, dst_w, dst_h,
             AP_RESIZE_PIL_MAX_SCALE);
  const int col_tiles = (dst_w + ap::kPilCols - 1) / ap::kPilCols;
  const int bands = (dst_h + ap::kPilRows - 1) / ap::kPilRows;
  const long long ctas = (long long)L * col_tiles * bands;
  AP_REQUIRE(ctas <= INT_MAX, "resize_pil_bilinear_u8: %d frames of %dx%d exceed one launch", L, dst_w, dst_h);
  const bool need_h = src_w != dst_w, need_v = src_h != dst_h;
  if (!need_h && !need_v) {   // Pillow returns a copy
    AP_CHECK_CUDA(cudaMemcpyAsync(dst, src, (size_t)L * src_h * src_w * 3, cudaMemcpyDeviceToDevice,
                                  (cudaStream_t)stream));
    return AP_OK;
  }
  const ap::PilAxis ax = ap::make_axis(src_w, dst_w), ay = ap::make_axis(src_h, dst_h);
  const int rows = need_v ? ap::pil_band_rows(ay) : ap::kPilRows;
  const size_t smem = sizeof(int) * ((size_t)ap::kPilCols * ax.ksize + (size_t)ap::kPilRows * ay.ksize +
                                     2 * ap::kPilCols + 2 * ap::kPilRows) +
                      (size_t)rows * ap::kPilCols * 3;
  if (smem > 48 * 1024)
    AP_CHECK_CUDA(cudaFuncSetAttribute(ap::resize_pil_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  AP_LAUNCH(ap::resize_pil_u8_kernel, (unsigned)ctas, ap::kPilThreads, smem, (cudaStream_t)stream, (const uint8_t*)src,
            ax, ay, need_h ? 1 : 0, need_v ? 1 : 0, col_tiles, bands, (uint8_t*)dst);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}
