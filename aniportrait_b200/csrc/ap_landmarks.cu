// Face-mesh projection and landmark pose-frame drawing: the stage of the reference's audio2vid / vid2vid scripts that
// turns the predicted mesh into pose images (src/utils/pose_util.py:30-59 + src/utils/draw_util.py:124-148, which is
// mediapipe's drawing_utils.draw_landmarks on cv2.line(..., thickness 2)).
#include <float.h>
#include <stdint.h>

#include "ap_host.h"
#include "ap_ptx.cuh"

namespace ap {

// ---------------------------------------------------------------------------------------------------------
// Projection: one thread per (frame, point). Evaluated in the reference's order with every operation rounded on its own
// (no fused multiply-add): base + offset in fp64, t = X_h . M^T, u = t . P with each dot product summed k = 0..3,
// then ((u / w) + 1) * 0.5 * size.
// ---------------------------------------------------------------------------------------------------------
struct ProjMatrix {
  double p[16];   // P row-major, u_j = sum_k t_k p[k * 4 + j]
};

__device__ __forceinline__ double dot4(double a0, double a1, double a2, double a3, double b0, double b1, double b2,
                                       double b3) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2)), __dmul_rn(a3, b3));
}

__global__ void __launch_bounds__(256)
project_points_kernel(const float* __restrict__ offsets, const double* __restrict__ base, long long base_frame_stride,
                      const double* __restrict__ matrices, ProjMatrix P, int L, int N, double width, double height,
                      double* __restrict__ out) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)L * N) return;
  const int f = (int)(t / N), n = (int)(t % N);
  const double* b = base + f * base_frame_stride + (long long)n * 3;
  double x = b[0], y = b[1], z = b[2];
  if (offsets) {
    x = __dadd_rn((double)offsets[t * 3 + 0], x);
    y = __dadd_rn((double)offsets[t * 3 + 1], y);
    z = __dadd_rn((double)offsets[t * 3 + 2], z);
  }
  const double* m = matrices + (long long)f * 16;
  double tr[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) tr[j] = dot4(x, y, z, 1.0, m[j * 4 + 0], m[j * 4 + 1], m[j * 4 + 2], m[j * 4 + 3]);
  double u[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) u[j] = dot4(tr[0], tr[1], tr[2], tr[3], P.p[j], P.p[4 + j], P.p[8 + j], P.p[12 + j]);
  out[t * 2 + 0] = __dmul_rn(__dmul_rn(__dadd_rn(__ddiv_rn(u[0], u[3]), 1.0), 0.5), width);
  out[t * 2 + 1] = __dmul_rn(__dmul_rn(__dadd_rn(__ddiv_rn(u[1], u[3]), 1.0), 0.5), height);
}

// ---------------------------------------------------------------------------------------------------------
// Landmark drawing. One CTA per (frame, band of kBand canvas rows), frame-major on a 1-D grid. Each CTA
//   A. converts the two endpoints of every edge to pixels as draw_landmarks does and builds, once per edge, the 16.16
//      polygon cv2's ThickLine fills (the only floating point of the rasteriser: the fp64 sqrt and cvRound of `dp`);
//   B. splits (edge, band row) pairs over its threads; each thread evaluates, in closed integer form, that row's pixels of
//      the polygon's scanline fill (FillConvexPoly), of its four outline segments (Line2, clipped to the canvas as cv2
//      clips them), and of the two radius-1 end caps, and raises the row's canvas entries to edge index + 1 with a shared
//      atomicMax. The largest index wins, which is cv2's painter's order (later edges overwrite earlier ones), so the result
//      does not depend on thread timing;
//   C. resolves index -> colour and writes the band's bytes with 16-byte stores.
// ---------------------------------------------------------------------------------------------------------
constexpr int kCanvas = AP_LMK_CANVAS;
constexpr int kBand = 16;
constexpr int kThreads = 256;
constexpr long long kOne = 1LL << 16, kHalf = kOne >> 1;

struct EdgeTable {
  int2 ends[AP_LMK_MAX_EDGES];
  uchar4 color[AP_LMK_MAX_EDGES];
};

struct EdgeGeom {
  int x0, y0, x1, y1;   // endpoint pixels; x0 < 0: the edge is not drawn
  int poly;             // 1: the polygon below exists (the endpoints differ)
  int vx[4], vy[4];     // ThickLine's polygon p0 + dp, p0 - dp, p1 - dp, p1 + dp in 16.16
};

__host__ __device__ __forceinline__ long long floor_div(long long a, long long b) {   // b > 0
  return a >= 0 ? a / b : -((-a + b - 1) / b);
}
__host__ __device__ __forceinline__ long long ceil_div(long long a, long long b) { return -floor_div(-a, b); }

// The row helpers below also compile for the host (single-threaded there), so that a CPU build can step through one edge
// against tests/landmark_reference.py.
__host__ __device__ __forceinline__ void mark(unsigned* row, int xa, int xb, unsigned v) {
  xa = xa < 0 ? 0 : xa;
  xb = xb > kCanvas - 1 ? kCanvas - 1 : xb;
  for (int x = xa; x <= xb; ++x) {
#ifdef __CUDA_ARCH__
    atomicMax(row + x, v);
#else
    row[x] = row[x] > v ? row[x] : v;
#endif
  }
}

// cv::clipLine on the (kCanvas << 16)^2 rectangle; the intercepts are double quotients truncated toward zero.
__host__ __device__ bool clip_line(long long& x1, long long& y1, long long& x2, long long& y2) {
  const long long right = ((long long)kCanvas << 16) - 1, bottom = right;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += (long long)((double)(a - y1) * (double)(x2 - x1) / (double)(y2 - y1));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += (long long)((double)(a - y2) * (double)(x2 - x1) / (double)(y2 - y1));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += (long long)((double)(a - x1) * (double)(y2 - y1) / (double)(x2 - x1));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += (long long)((double)(a - x2) * (double)(y2 - y1) / (double)(x2 - x1));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// Row y of cv::Line2 from (x1, y1) to (x2, y2) (16.16): the walk's pixels are (x0 + k, (yy + k * step) >> 16) for
// k = 0..ecount when x-major, ((xx + k * step) >> 16, y0 + k) when y-major, plus the rounded end point.
__host__ __device__ void line2_row(unsigned* row, int y, long long x1, long long y1, long long x2, long long y2, unsigned v) {
  if (!clip_line(x1, y1, x2, y2)) return;
  long long dx = x2 - x1, dy = y2 - y1;
  const long long ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  long long t;
  if (ax > ay) {
    if (dx < 0) {
      dy = -dy;
      t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    const long long step = (dy * kOne) / (ax | 1);
    const long long ecount = (x2 - x1) >> 16;
    const long long x0 = (x1 + kHalf) >> 16, yy = y1 + kHalf;
    const long long lo = (long long)y * kOne - yy, hi = lo + kOne - 1;   // lo <= k * step <= hi
    long long ka, kb;
    if (step > 0) {
      ka = ceil_div(lo, step);
      kb = floor_div(hi, step);
    } else if (step < 0) {
      ka = ceil_div(-hi, -step);
      kb = floor_div(-lo, -step);
    } else {
      ka = 0;
      kb = (lo <= 0 && 0 <= hi) ? ecount : -1;
    }
    ka = max(ka, 0LL);
    kb = min(kb, ecount);
    if (ka <= kb) mark(row, (int)(x0 + ka), (int)(x0 + kb), v);
  } else {
    if (dy < 0) {
      dx = -dx;
      t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    const long long step = (dx * kOne) / (ay | 1);
    const long long ecount = (y2 - y1) >> 16;
    const long long k = y - ((y1 + kHalf) >> 16);
    if (k >= 0 && k <= ecount) {
      const int x = (int)((x1 + kHalf + k * step) >> 16);
      mark(row, x, x, v);
    }
  }
  if (((y2 + kHalf) >> 16) == y) {
    const int x = (int)((x2 + kHalf) >> 16);
    mark(row, x, x, v);
  }
}

// Row y of cv::FillConvexPoly's scanline walk over the 4-point polygon, jumping from one edge pick-up row to the next:
// an edge picked up at row ys with start x xs is at xs + (y - ys) * dx on row y.
__host__ __device__ void fill_row(unsigned* row, int y, const int* vx, const int* vy, unsigned v) {
  long long ymin = vy[0], ymax = vy[0], xmin = vx[0], xmax = vx[0];
  int imin = 0;
  for (int k = 1; k < 4; ++k) {
    if (vy[k] < ymin) { ymin = vy[k]; imin = k; }
    ymax = max(ymax, (long long)vy[k]);
    xmax = max(xmax, (long long)vx[k]);
    xmin = min(xmin, (long long)vx[k]);
  }
  xmin = (xmin + kHalf) >> 16;
  xmax = (xmax + kHalf) >> 16;
  ymin = (ymin + kHalf) >> 16;
  ymax = (ymax + kHalf) >> 16;
  if (xmax < 0 || ymax < 0 || xmin >= kCanvas || ymin >= kCanvas) return;
  ymax = min(ymax, (long long)kCanvas - 1);
  if (y < ymin || y > ymax) return;
  int idx[2] = {imin, imin};
  const int di[2] = {1, 3};
  long long ye[2] = {ymin, ymin}, ys[2] = {ymin, ymin}, x[2] = {-kOne, -kOne}, dx[2] = {0, 0};
  int edges = 4;
  long long cy = ymin;
  for (;;) {
    for (int i = 0; i < 2; ++i) {
      if (cy < ye[i]) continue;
      int idx0 = idx[i], id = idx0 + di[i];
      if (id >= 4) id -= 4;
      while (edges-- > 0) {
        const long long ty = ((long long)vy[id] + kHalf) >> 16;
        if (ty > cy) {
          const long long xs = vx[idx0], xe = vx[id];
          ye[i] = ty;
          dx[i] = ((xe - xs) * 2 + (ty - cy)) / (2 * (ty - cy));
          x[i] = xs;
          ys[i] = cy;
          idx[i] = id;
          break;
        }
        idx0 = id;
        id += di[i];
        if (id >= 4) id -= 4;
      }
    }
    if (edges < 0) return;
    const long long next = min(ye[0], ye[1]);
    if (y < next) break;
    cy = next;
  }
  const long long xa = x[0] + (y - ys[0]) * dx[0], xb = x[1] + (y - ys[1]) * dx[1];
  const long long x1 = (min(xa, xb) + kHalf) >> 16, x2 = (max(xa, xb) + kHalf) >> 16;
  if (x2 >= 0 && x1 < kCanvas) mark(row, (int)x1, (int)x2, v);
}

__global__ void __launch_bounds__(kThreads)
draw_landmarks_kernel(const double* __restrict__ keypoints, int N, double size_x, double size_y, int normed,
                      const EdgeTable table, int E, uint8_t* __restrict__ out) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  __shared__ unsigned canvas[kBand][kCanvas];
  __shared__ EdgeGeom geom[AP_LMK_MAX_EDGES];
  __shared__ uchar4 palette[AP_LMK_MAX_EDGES + 1];
  constexpr int kBands = kCanvas / kBand;
  const int f = blockIdx.x / kBands;
  const int band0 = blockIdx.x % kBands * kBand;
  for (int i = threadIdx.x; i < kBand * kCanvas; i += kThreads) (&canvas[0][0])[i] = 0u;
  for (int i = threadIdx.x; i <= E; i += kThreads) palette[i] = i == 0 ? make_uchar4(0, 0, 0, 0) : table.color[i - 1];
  griddep_wait();

  // A. endpoints -> pixels (protobuf float32 x / y, kept iff in [0, 1], pixel min(floor(v * 512), 511)); polygon per edge
  const double* kp = keypoints + (long long)f * N * 2;
  for (int e = threadIdx.x; e < E; e += kThreads) {
    EdgeGeom g;
    int px[2][2];
    bool kept = true;
    const int ends[2] = {table.ends[e].x, table.ends[e].y};
#pragma unroll
    for (int s = 0; s < 2; ++s) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const double k = kp[(long long)ends[s] * 2 + c];
        const float v = __double2float_rn(normed ? k : __ddiv_rn(k, c == 0 ? size_x : size_y));
        kept = kept && v >= 0.f && v <= 1.f;   // NaN fails both
        px[s][c] = min((int)floor((double)v * kCanvas), kCanvas - 1);
      }
    }
    g.x0 = kept ? px[0][0] : -1;
    g.y0 = px[0][1];
    g.x1 = px[1][0];
    g.y1 = px[1][1];
    g.poly = 0;
    if (kept) {
      const double ddx = (double)(px[0][0] - px[1][0]), ddy = (double)(px[1][1] - px[0][1]);
      double r = __dadd_rn(__dmul_rn(ddx, ddx), __dmul_rn(ddy, ddy));
      if (r > DBL_EPSILON) {
        r = __ddiv_rn((double)kOne, __dsqrt_rn(r));   // (thickness 2) << (XY_SHIFT - 1)
        const int dpx = __double2int_rn(__dmul_rn(ddy, r)), dpy = __double2int_rn(__dmul_rn(ddx, r));   // cvRound
        const int x0 = px[0][0] << 16, y0 = px[0][1] << 16, x1 = px[1][0] << 16, y1 = px[1][1] << 16;
        g.poly = 1;
        g.vx[0] = x0 + dpx; g.vy[0] = y0 + dpy;
        g.vx[1] = x0 - dpx; g.vy[1] = y0 - dpy;
        g.vx[2] = x1 - dpx; g.vy[2] = y1 - dpy;
        g.vx[3] = x1 + dpx; g.vy[3] = y1 + dpy;
      }
    }
    geom[e] = g;
  }
  __syncthreads();

  // B. (edge, band row) pairs; every pixel of an edge lies within one row of its endpoints' rows
  for (int i = threadIdx.x; i < E * kBand; i += kThreads) {
    const int e = i / kBand, y = band0 + i % kBand;
    const EdgeGeom& g = geom[e];
    if (g.x0 < 0 || y < min(g.y0, g.y1) - 1 || y > max(g.y0, g.y1) + 1) continue;
    unsigned* row = canvas[y - band0];
    const unsigned v = (unsigned)e + 1;
    if (g.poly) {
      for (int k = 0; k < 4; ++k) {
        const int p = (k + 3) & 3;
        line2_row(row, y, g.vx[p], g.vy[p], g.vx[k], g.vy[k], v);
      }
      fill_row(row, y, g.vx, g.vy, v);
    }
    // radius-1 filled caps: a plus around each endpoint
    if (y == g.y0) mark(row, g.x0 - 1, g.x0 + 1, v);
    else if (y == g.y0 - 1 || y == g.y0 + 1) mark(row, g.x0, g.x0, v);
    if (y == g.y1) mark(row, g.x1 - 1, g.x1 + 1, v);
    else if (y == g.y1 - 1 || y == g.y1 + 1) mark(row, g.x1, g.x1, v);
  }
  __syncthreads();

  // C. index -> colour bytes (channel c of pixel x = colour byte c), 16 bytes per store
  constexpr int kBytes = kBand * kCanvas * 3;
  uint4* dst = reinterpret_cast<uint4*>(out + ((long long)f * kCanvas + band0) * kCanvas * 3);
  const unsigned* flat = &canvas[0][0];
  for (int q = threadIdx.x; q < kBytes / 16; q += kThreads) {
    unsigned w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      unsigned word = 0;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int byte = q * 16 + j * 4 + b;
        const uchar4 c = palette[flat[byte / 3]];
        const int ch = byte % 3;
        const unsigned val = ch == 0 ? c.x : (ch == 1 ? c.y : c.z);
        word |= val << (8 * b);
      }
      w[j] = word;
    }
    dst[q] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

}  // namespace ap

extern "C" int ap_project_points_f64(const float* offsets, const double* base, int base_per_frame,
                                     const double* matrices, const double* proj, int L, int N, double width,
                                     double height, double* out, void* stream) {
  AP_REQUIRE(base && matrices && proj && out && L > 0 && N > 0, "project_points: bad arguments");
  ap::ProjMatrix P;
  for (int i = 0; i < 16; ++i) P.p[i] = proj[i];
  const long long total = (long long)L * N;
  AP_LAUNCH((ap::project_points_kernel), (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, offsets, base,
            base_per_frame ? (long long)N * 3 : 0LL, matrices, P, L, N, width, height, out);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_draw_landmarks_u8(const double* keypoints, int L, int N, double size_x, double size_y, int normed,
                                    const int* edges, const unsigned char* colors, int E, int thickness, void* out,
                                    void* stream) {
  AP_REQUIRE(keypoints && out && L > 0 && N > 0, "draw_landmarks: bad arguments");
  AP_REQUIRE(L <= AP_LMK_MAX_FRAMES, "draw_landmarks: %d frames (at most %d per call)", L, AP_LMK_MAX_FRAMES);
  AP_REQUIRE(thickness == 2, "draw_landmarks: only thickness 2 is implemented (got %d)", thickness);
  AP_REQUIRE(E >= 0 && E <= AP_LMK_MAX_EDGES, "draw_landmarks: %d edges (at most %d)", E, AP_LMK_MAX_EDGES);
  AP_REQUIRE(E == 0 || (edges && colors), "draw_landmarks: null edge table");
  AP_REQUIRE(((uintptr_t)out & 15) == 0, "draw_landmarks: out must be 16-byte aligned");
  ap::EdgeTable table;
  for (int e = 0; e < E; ++e) {
    AP_REQUIRE(edges[2 * e] >= 0 && edges[2 * e] < N && edges[2 * e + 1] >= 0 && edges[2 * e + 1] < N,
               "draw_landmarks: edge %d (%d, %d) is outside [0, %d)", e, edges[2 * e], edges[2 * e + 1], N);
    table.ends[e] = make_int2(edges[2 * e], edges[2 * e + 1]);
    table.color[e] = make_uchar4(colors[3 * e], colors[3 * e + 1], colors[3 * e + 2], 0);
  }
  AP_LAUNCH((ap::draw_landmarks_kernel), (unsigned)(ap::kCanvas / ap::kBand) * (unsigned)L, ap::kThreads, 0, (cudaStream_t)stream,
            keypoints, N, size_x, size_y, normed, table, E, (uint8_t*)out);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}
