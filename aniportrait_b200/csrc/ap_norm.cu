// GroupNorm (two-phase, channels-last) and LayerNorm kernels. These are HBM-bound streaming kernels: 16-byte
// vectorised, coalesced accesses, fp32 statistics.
//
// Replaces InflatedGroupNorm / nn.GroupNorm (+SiLU) (reference src/models/resnet.py:21-29,221-222,232-238;
// src/models/transformer_3d.py:58-60,124; src/models/motion_module.py:119-121,156; src/models/unet_3d.py:238-249,573-574)
// and nn.LayerNorm (+ temporal positional-encoding add) (src/models/attention.py:331-362;
// src/models/motion_module.py:228-241,262-277,365-366).
#include <stdlib.h>

#include "ap_host.h"
#include "ap_ptx.cuh"

namespace ap {

// ---------------------------------------------------------------------------------------------------------
// GroupNorm statistics, deterministic two-stage reduction (no atomics: results are bit-reproducible run to run).
// Stage 1: grid (row_chunks, Nf); block = (C/8) * k threads; a thread owns 8 consecutive channels and strides over the
// block's rows; per-thread sums go through shared memory and are combined per group in a fixed order;
// partials[frame][chunk][group] = {sum, sumsq} (only the groups this source intersects are written).
// Stage 2 (gn_finalize_kernel): per frame, 8 lanes per group add the chunks' partials of both sources in double and
// write stats[frame][group] = {mean, rstd}.
// ---------------------------------------------------------------------------------------------------------
__global__ void gn_stats_kernel(const __half* __restrict__ x, int HW, int C, int c_off, int cpg, int rows_per_block,
                                float2* __restrict__ partials, int G) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int vecs = C >> 3;
  const int k = blockDim.x / vecs;
  const int cv = threadIdx.x % vecs;
  const int rl = threadIdx.x / vecs;
  const int frame = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(r0 + rows_per_block, HW);
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  if (rl < k) {
    const __half* base = x + ((long long)frame * HW) * C + cv * 8;
#pragma unroll 4
    for (int r = r0 + rl; r < r1; r += k) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(base + (long long)r * C));
      const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h2[j]);
        s[2 * j] += f.x; q[2 * j] += f.x * f.x;
        s[2 * j + 1] += f.y; q[2 * j + 1] += f.y * f.y;
      }
    }
  }
  extern __shared__ float2 sh[];  // [k][C] per-thread channel sums, then [C] channel totals
  if (rl < k) {
#pragma unroll
    for (int j = 0; j < 8; ++j) sh[rl * C + cv * 8 + j] = make_float2(s[j], q[j]);
  }
  __syncthreads();
  // fixed-order tree: rows -> channel totals (all threads), channels -> groups (one thread per group)
  float2* tot = sh + k * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float as = 0.f, aq = 0.f;
    for (int r = 0; r < k; ++r) {
      const float2 v = sh[r * C + c];
      as += v.x;
      aq += v.y;
    }
    tot[c] = make_float2(as, aq);
  }
  __syncthreads();
  const int g_lo = c_off / cpg, g_hi = (c_off + C - 1) / cpg;
  for (int g = g_lo + threadIdx.x; g <= g_hi; g += blockDim.x) {
    const int c0 = max(g * cpg, c_off) - c_off;
    const int c1 = min((g + 1) * cpg, c_off + C) - c_off;
    float as = 0.f, aq = 0.f;
    for (int c = c0; c < c1; ++c) {
      as += tot[c].x;
      aq += tot[c].y;
    }
    partials[((long long)frame * gridDim.x + blockIdx.x) * G + g] = make_float2(as, aq);
  }
}

// grid Nf, block 8 * G threads. Source i covers groups [glo_i, ghi_i] with chunks_i partials per frame (chunks1 = 0: none).
__global__ void gn_finalize_kernel(const float2* __restrict__ p0, int chunks0, int glo0, int ghi0,
                                   const float2* __restrict__ p1, int chunks1, int glo1, int ghi1, int G,
                                   double inv_count, float eps, float2* __restrict__ stats) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int frame = blockIdx.x;
  const int g = threadIdx.x >> 3, sub = threadIdx.x & 7;
  double s = 0.0, q = 0.0;
  if (g >= glo0 && g <= ghi0)
    for (int c = sub; c < chunks0; c += 8) {
      const float2 v = p0[((long long)frame * chunks0 + c) * G + g];
      s += v.x;
      q += v.y;
    }
  if (chunks1 > 0 && g >= glo1 && g <= ghi1)
    for (int c = sub; c < chunks1; c += 8) {
      const float2 v = p1[((long long)frame * chunks1 + c) * G + g];
      s += v.x;
      q += v.y;
    }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (sub == 0) {
    const double mean = s * inv_count;
    const double var = fmax(q * inv_count - mean * mean, 0.0);
    stats[(long long)frame * G + g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
  }
}

// Finalize from PER-COLUMN partials written by the producing GEMM / conv epilogue (ap_gemm.cu: col_stat_out): entry e holds
// {sum, sumsq} of every output channel over rows [32 e, 32 e + 32) of the producer's output, i.e. frame e / (HW / 32).
// Grid (Nf, ceil(G / 8)), block 1024 = 8 groups x 4 warps: each warp adds a quarter of the frame's entries for the channels
// of its group (double accumulation, fixed order), xor-shuffle tree, then the four quarter sums are combined through shared
// memory in a fixed order -> stats[frame][group] = {mean, rstd}. The group may straddle the two concatenated sources.
__global__ void __launch_bounds__(1024)
gn_finalize_cols_kernel(const float2* __restrict__ p0, long long ld0, int C1, const float2* __restrict__ p1, long long ld1,
                        int epf, int cpg, int G, double inv_count, float eps, float2* __restrict__ stats) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  __shared__ double sh[8][4][2];
  const int frame = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gl = warp >> 2, sub = warp & 3;
  const int g = blockIdx.y * 8 + gl;
  double s = 0.0, q = 0.0;
  if (g < G) {
    const int e0 = (epf * sub) / 4, e1 = (epf * (sub + 1)) / 4;
    const int total = (e1 - e0) * cpg;
    for (int idx = lane; idx < total; idx += 32) {
      const int e = e0 + idx / cpg;
      const int c = g * cpg + idx % cpg;
      const long long row = (long long)frame * epf + e;
      const float2 v = c < C1 ? __ldg(p0 + row * ld0 + c) : __ldg(p1 + row * ld1 + (c - C1));
      s += v.x;
      q += v.y;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (lane == 0) {
    sh[gl][sub][0] = s;
    sh[gl][sub][1] = q;
  }
  __syncthreads();
  if (g < G && sub == 0 && lane == 0) {
    const double S = ((sh[gl][0][0] + sh[gl][1][0]) + sh[gl][2][0]) + sh[gl][3][0];
    const double Q = ((sh[gl][0][1] + sh[gl][1][1]) + sh[gl][2][1]) + sh[gl][3][1];
    const double mean = S * inv_count;
    const double var = fmax(Q * inv_count - mean * mean, 0.0);
    stats[(long long)frame * G + g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
  }
}

// x * sigmoid(x) with two MUFU ops (ex2, rcp) and no IEEE-division sequence: the SiLU variant of gn_apply was ALU-bound
// (47 us against 25 us without SiLU at 32 x 4096 x 320), not HBM-bound. Relative error ~2^-22, far below fp16 resolution.
__device__ __forceinline__ float silu_fast(float v) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.f + e));
  return v * r;
}

// Apply: y = (x - mean) * rstd * gamma + beta  (optionally SiLU), written at channel offset c_off of an
// [rows, C_total] output (this is also how the skip-concat gets materialised, in normalised form, for free).
template <bool SILU>
__global__ void gn_apply_kernel(const __half* __restrict__ x, int HW, int C, int c_off, int C_total, int cpg,
                                int rows_per_block, const float2* __restrict__ stats, int G,
                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                __half* __restrict__ y) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int vecs = C >> 3;
  const int k = blockDim.x / vecs;
  const int cv = threadIdx.x % vecs;
  const int rl = threadIdx.x / vecs;
  if (rl >= k) return;
  const int frame = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(r0 + rows_per_block, HW);
  float a[8], b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c_off + cv * 8 + j;
    const int g = c / cpg;
    const float2 mr = stats[(long long)frame * G + g];   // {mean, rstd}
    a[j] = mr.y * gamma[c];
    b[j] = beta[c] - mr.x * a[j];
  }
  const __half* src = x + ((long long)frame * HW) * C + cv * 8;
  __half* dst = y + ((long long)frame * HW) * C_total + c_off + cv * 8;
#pragma unroll 4
  for (int r = r0 + rl; r < r1; r += k) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(src + (long long)r * C));
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
    uint4 o;
    __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h2[j]);
      float v0 = f.x * a[2 * j] + b[2 * j];
      float v1 = f.y * a[2 * j + 1] + b[2 * j + 1];
      if (SILU) {
        v0 = silu_fast(v0);
        v1 = silu_fast(v1);
      }
      o2[j] = __floats2half2_rn(v0, v1);
    }
    *reinterpret_cast<uint4*>(dst + (long long)r * C_total) = o;
  }
}

// ---------------------------------------------------------------------------------------------------------
// LayerNorm over the channel dim, one warp per row, values kept in registers (exact two-pass statistics).
// Optional additive table pe[(row / rows_per_pe) % pe_period][C] (the temporal positional encoding, which the
// reference adds to the LayerNorm output before the q/k/v projections).
// ---------------------------------------------------------------------------------------------------------
template <int MAXV>  // MAXV = max half2 per lane  (C <= 64 * MAXV)
__global__ void layernorm_kernel(const __half* __restrict__ x, long long rows, int C, float eps,
                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ pe, int rows_per_pe, int pe_period,
                                 __half* __restrict__ y) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int warps_per_block = blockDim.x >> 5;
  const long long row = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nv = C >> 1;  // half2 per row
  const __half2* src = reinterpret_cast<const __half2*>(x + row * C);
  float2 v[MAXV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nv) {
      v[i] = __half22float2(src[idx]);
      sum += v[i].x + v[i].y;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nv) {
      const float dx = v[i].x - mean, dy = v[i].y - mean;
      sq += dx * dx + dy * dy;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / C + eps);
  const float* pe_row = pe ? pe + (long long)((row / rows_per_pe) % pe_period) * C : nullptr;
  __half2* dst = reinterpret_cast<__half2*>(y + row * C);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nv) {
      const float2 g = *reinterpret_cast<const float2*>(gamma + 2 * idx);
      const float2 b = *reinterpret_cast<const float2*>(beta + 2 * idx);
      float o0 = (v[i].x - mean) * rstd * g.x + b.x;
      float o1 = (v[i].y - mean) * rstd * g.y + b.y;
      if (pe_row) {
        const float2 p = *reinterpret_cast<const float2*>(pe_row + 2 * idx);
        o0 += p.x;
        o1 += p.y;
      }
      dst[idx] = __floats2half2_rn(o0, o1);
    }
  }
}

// LayerNorm, wide-load variant for C % 8 == 0, C <= 1536: LPR lanes per row (32 / LPR rows per warp), each lane keeps up
// to 6 16-byte vectors of its row in registers (vector v of the row belongs to lane v % LPR), so every load / store
// instruction moves full 128-byte lines; LPR = 8 / 16 / 32 for C = 320 / 640 / 1280 keeps 5 vectors per lane at every
// level (the one-warp-per-row kernel above issues 4-byte accesses; a fixed 8 lanes per row left the 1280-wide levels with
// 20 vectors per lane, 128 registers and a quarter of the blocks). Same exact two-pass statistics.
template <int LPR>
__global__ void __launch_bounds__(256)
layernormv_kernel(const __half* __restrict__ x, long long rows, int C, float eps, const float* __restrict__ gamma,
                  const float* __restrict__ beta, const float* __restrict__ pe, int rows_per_pe, int pe_period,
                  __half* __restrict__ y) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  constexpr int MAXV = 6;
  constexpr int RPW = 32 / LPR;   // rows per warp
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPR;
  const long long row = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + lane / LPR;
  const bool ok = row < rows;
  const int nvec = C >> 3;   // 16-byte vectors per row
  const uint4* src = reinterpret_cast<const uint4*>(x + (ok ? row : 0) * C);
  uint4 v[MAXV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = sub + LPR * i;
    v[i] = (ok && vi < nvec) ? __ldg(src + vi) : make_uint4(0u, 0u, 0u, 0u);
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 f = __half22float2(h[t]);
      sum += f.x + f.y;           // vectors past the row end were zero-filled
    }
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (sub + LPR * i < nvec) {
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 f = __half22float2(h[t]);
        const float dx = f.x - mean, dy = f.y - mean;
        sq += dx * dx + dy * dy;
      }
    }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / C + eps);
  if (!ok) return;
  const float* pe_row = pe ? pe + (long long)((row / rows_per_pe) % pe_period) * C : nullptr;
  uint4* dst = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = sub + LPR * i;
    if (vi < nvec) {
      const int c0 = vi * 8;
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c0)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c0 + 4));
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float o[8];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 f = __half22float2(h[t]);
        o[2 * t] = (f.x - mean) * rstd * gg[2 * t] + bb[2 * t];
        o[2 * t + 1] = (f.y - mean) * rstd * gg[2 * t + 1] + bb[2 * t + 1];
      }
      if (pe_row) {
        const float4 p0 = __ldg(reinterpret_cast<const float4*>(pe_row + c0)), p1 = __ldg(reinterpret_cast<const float4*>(pe_row + c0 + 4));
        o[0] += p0.x; o[1] += p0.y; o[2] += p0.z; o[3] += p0.w;
        o[4] += p1.x; o[5] += p1.y; o[6] += p1.z; o[7] += p1.w;
      }
      uint4 u;
      __half2* oh = reinterpret_cast<__half2*>(&u);
#pragma unroll
      for (int t = 0; t < 4; ++t) oh[t] = __floats2half2_rn(o[2 * t], o[2 * t + 1]);
      dst[vi] = u;
    }
  }
}

// LayerNorm folding: row partials {sum, sumsq} of x (written by the producing GEMM's epilogue warps) -> the row's rstd and
// the 8-column fp16 operand (-mean_hi, -mean_lo, -mean_hi, 0...) that carries the mean term through the tensor core.
__global__ void ln_finalize_kernel(const float2* __restrict__ st, int parts, long long ld, long long M, float inv_k, float eps,
                                   uint4* __restrict__ a2, float* __restrict__ rstd) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float S = 0.f, Q = 0.f;
  for (int i = 0; i < parts; ++i) {
    const float2 t = __ldg(st + (long long)i * ld + m);
    S += t.x;
    Q += t.y;
  }
  const float mean = S * inv_k;
  rstd[m] = rsqrtf(fmaxf(Q * inv_k - mean * mean, 0.f) + eps);
  const __half hi = __float2half_rn(-mean);
  const __half lo = __float2half_rn(-mean - __half2float(hi));
  const __half2 a = __halves2half2(hi, lo), b = __halves2half2(hi, __float2half_rn(0.f));
  uint4 o;
  o.x = *reinterpret_cast<const uint32_t*>(&a);
  o.y = *reinterpret_cast<const uint32_t*>(&b);
  o.z = 0u;
  o.w = 0u;
  a2[m] = o;
}

// Row softmax (fp16 in/out, fp32 math) for the VAE's single-head 4096-token attention, which is evaluated as
// GEMM -> softmax -> GEMM (head dim 512 does not fit the fused attention kernel's register budget). One block per row.
__global__ void __launch_bounds__(256) softmax_rows_kernel(const __half* __restrict__ x, __half* __restrict__ y,
                                                           int cols, long long ld) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long row = blockIdx.x;
  const __half2* src = reinterpret_cast<const __half2*>(x + row * ld);
  __half2* dst = reinterpret_cast<__half2*>(y + row * ld);
  const int nv = cols >> 1;
  __shared__ float red[8];
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const float2 f = __half22float2(src[i]);
    mx = fmaxf(mx, fmaxf(f.x, f.y));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const float2 f = __half22float2(src[i]);
    sum += __expf(f.x - mx) + __expf(f.y - mx);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) sum += red[w];
  const float inv = 1.f / sum;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const float2 f = __half22float2(src[i]);
    dst[i] = __floats2half2_rn(__expf(f.x - mx) * inv, __expf(f.y - mx) * inv);
  }
}

static void gn_launch_geometry(int HW, int C, int Nf, int* threads, int* rows_per_block, int* chunks) {
  const int vecs = C / 8;
  int k = 256 / vecs;
  if (k < 1) k = 1;
  *threads = vecs * k;
  // aim for >= ~4 waves of the SMs when the tensor is large, but at least 8 rows per row-lane
  int rpb = 8 * k;
  while ((long long)((HW + rpb - 1) / rpb) * Nf > AP_GN_MAX_BLOCKS && rpb < HW) rpb *= 2;
  *rows_per_block = rpb;
  *chunks = (HW + rpb - 1) / rpb;
}

}  // namespace ap

using namespace ap;

// stats: fp32 workspace of 2*groups*(Nf + 2*AP_GN_MAX_BLOCKS) floats: [Nf, G] {mean, rstd} followed by the per-block
// partial sums of the (up to two) sources. x2/C2 optional second source (channel concat).
extern "C" int ap_groupnorm_nhwc_f16(const void* x, int C1, const void* x2, int C2, int Nf, int HW, int groups,
                                     float eps, const float* gamma, const float* beta, int silu, float* stats,
                                     void* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const int C = C1 + (x2 ? C2 : 0);
  AP_REQUIRE(x && out && stats && gamma && beta, "groupnorm: null pointer");
  AP_REQUIRE(C % groups == 0, "groupnorm: C=%d not divisible by groups=%d", C, groups);
  AP_REQUIRE(C1 % 8 == 0 && (!x2 || C2 % 8 == 0), "groupnorm: channel counts must be multiples of 8");
  AP_REQUIRE(C1 / 8 <= 1024 && (!x2 || C2 / 8 <= 1024), "groupnorm: too many channels");
  AP_REQUIRE(groups * 8 <= 1024, "groupnorm: at most 128 groups");
  AP_REQUIRE(aligned16(x) && aligned16(x2) && aligned16(out), "groupnorm: x, x2 and out must be 16-byte aligned");
  const int cpg = C / groups;
  const int nsrc = x2 ? 2 : 1;
  const void* srcs[2] = {x, x2};
  const int cs[2] = {C1, C2};
  const int offs[2] = {0, C1};
  int threads[2], rpb[2], chunks[2] = {0, 0};
  float2* stat2 = reinterpret_cast<float2*>(stats);
  float2* part[2] = {stat2 + (long long)Nf * groups, nullptr};
  for (int s = 0; s < nsrc; ++s) {
    gn_launch_geometry(HW, cs[s], Nf, &threads[s], &rpb[s], &chunks[s]);
    AP_REQUIRE((long long)chunks[s] * Nf <= AP_GN_MAX_BLOCKS, "groupnorm: %d frames exceed the partial-sum workspace", Nf);
    const int k = threads[s] / (cs[s] / 8);
    AP_REQUIRE((size_t)(k + 1) * cs[s] * sizeof(float2) <= 48 * 1024, "groupnorm: C=%d too wide for the reduction buffer", cs[s]);
    if (s == 0) part[1] = part[0] + (long long)Nf * chunks[0] * groups;
    AP_LAUNCH((gn_stats_kernel), dim3(chunks[s], Nf), threads[s], sizeof(float2) * (k + 1) * cs[s], stream, 
        (const __half*)srcs[s], HW, cs[s], offs[s], cpg, rpb[s], part[s], groups);
  }
  AP_CHECK_CUDA(cudaGetLastError());
  const double inv_count = 1.0 / ((double)HW * (double)cpg);
  AP_LAUNCH((gn_finalize_kernel), Nf, 8 * groups, 0, stream, part[0], chunks[0], 0, (C1 - 1) / cpg, part[1], nsrc == 2 ? chunks[1] : 0,
                                                   C1 / cpg, (C - 1) / cpg, groups, inv_count, eps, stat2);
  AP_CHECK_CUDA(cudaGetLastError());
  for (int s = 0; s < nsrc; ++s) {
    if (silu)
      AP_LAUNCH((gn_apply_kernel<true>), dim3(chunks[s], Nf), threads[s], 0, stream, (const __half*)srcs[s], HW, cs[s], offs[s], C,
                                                                            cpg, rpb[s], stat2, groups, gamma, beta,
                                                                            (__half*)out);
    else
      AP_LAUNCH((gn_apply_kernel<false>), dim3(chunks[s], Nf), threads[s], 0, stream, (const __half*)srcs[s], HW, cs[s], offs[s], C,
                                                                             cpg, rpb[s], stat2, groups, gamma, beta,
                                                                             (__half*)out);
  }
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

// GroupNorm whose statistics come from the producers' epilogues: finalize (column partials -> {mean, rstd}) + apply.
extern "C" int ap_groupnorm_apply_nhwc_f16(const void* x, int C1, const void* colstat1, long long ld1, const void* x2,
                                           int C2, const void* colstat2, long long ld2, int Nf, int HW, int groups,
                                           float eps, const float* gamma, const float* beta, int silu, float* stats,
                                           void* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const int C = C1 + (x2 ? C2 : 0);
  AP_REQUIRE(x && out && stats && gamma && beta && colstat1 && (!x2 || colstat2), "groupnorm_apply: null pointer");
  AP_REQUIRE(C % groups == 0, "groupnorm_apply: C=%d not divisible by groups=%d", C, groups);
  AP_REQUIRE(C1 % 8 == 0 && (!x2 || C2 % 8 == 0), "groupnorm_apply: channel counts must be multiples of 8");
  AP_REQUIRE(HW % 32 == 0, "groupnorm_apply: HW=%d must be a multiple of 32 (32-row statistics entries)", HW);
  AP_REQUIRE(ld1 >= C1 && (!x2 || ld2 >= C2), "groupnorm_apply: partial row stride smaller than the channel count");
  AP_REQUIRE(aligned16(x) && aligned16(x2) && aligned16(out), "groupnorm_apply: x, x2 and out must be 16-byte aligned");
  const int cpg = C / groups;
  float2* stat2 = reinterpret_cast<float2*>(stats);
  AP_LAUNCH((gn_finalize_cols_kernel), dim3(Nf, (groups + 7) / 8), 1024, 0, stream, 
      (const float2*)colstat1, ld1, C1, (const float2*)colstat2, ld2, HW / 32, cpg, groups,
      1.0 / ((double)HW * (double)cpg), eps, stat2);
  AP_CHECK_CUDA(cudaGetLastError());
  const void* srcs[2] = {x, x2};
  const int cs[2] = {C1, C2};
  const int offs[2] = {0, C1};
  for (int s = 0; s < (x2 ? 2 : 1); ++s) {
    int threads, rpb, chunks;
    gn_launch_geometry(HW, cs[s], Nf, &threads, &rpb, &chunks);
    if (silu)
      AP_LAUNCH((gn_apply_kernel<true>), dim3(chunks, Nf), threads, 0, stream, (const __half*)srcs[s], HW, cs[s], offs[s], C, cpg, rpb,
                                                                      stat2, groups, gamma, beta, (__half*)out);
    else
      AP_LAUNCH((gn_apply_kernel<false>), dim3(chunks, Nf), threads, 0, stream, (const __half*)srcs[s], HW, cs[s], offs[s], C, cpg, rpb,
                                                                       stat2, groups, gamma, beta, (__half*)out);
  }
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_layernorm_finalize_f16(const void* row_stat, int parts, long long ld, long long M, int K, float eps,
                                         void* a2_out, float* rstd_out, void* stream) {
  AP_REQUIRE(row_stat && a2_out && rstd_out && parts > 0 && M > 0 && K > 0 && ld >= M, "layernorm_finalize: bad arguments");
  AP_REQUIRE((reinterpret_cast<uintptr_t>(a2_out) & 15) == 0, "layernorm_finalize: a2_out must be 16-byte aligned");
  AP_LAUNCH((ln_finalize_kernel), (unsigned)((M + 255) / 256), 256, 0, (cudaStream_t)stream, 
      (const float2*)row_stat, parts, ld, M, 1.f / (float)K, eps, (uint4*)a2_out, rstd_out);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_softmax_rows_f16(const void* x, void* out, long long rows, int cols, long long ld, void* stream) {
  AP_REQUIRE(x && out && cols % 2 == 0 && ld % 2 == 0, "softmax_rows: cols/ld must be even");
  AP_REQUIRE((reinterpret_cast<uintptr_t>(x) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0,
             "softmax_rows: x and out must be 4-byte aligned (__half2 accesses)");
  AP_LAUNCH((softmax_rows_kernel), (unsigned)rows, 256, 0, (cudaStream_t)stream, (const __half*)x, (__half*)out, cols, ld);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_layernorm_f16(const void* x, long long rows, int C, float eps, const float* gamma,
                                const float* beta, const float* pe, int rows_per_pe, int pe_period, void* out,
                                void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  AP_REQUIRE(x && out && gamma && beta, "layernorm: null pointer");
  AP_REQUIRE(C % 2 == 0 && C <= 64 * 32, "layernorm: C=%d unsupported (even, <= 2048)", C);
  AP_REQUIRE(pe == nullptr || (rows_per_pe > 0 && pe_period > 0), "layernorm: bad pe geometry");
  AP_REQUIRE(aligned16(x) && aligned16(out) && aligned16(gamma) && aligned16(beta) && aligned16(pe),
             "layernorm: x, out, gamma, beta and pe must be 16-byte aligned");
  const int wpb = 8;
  if (C % 8 == 0 && C / 8 <= 6 * 32 && getenv("AP_LAYERNORM_NARROW") == nullptr) {
    const int nvec = C / 8;
    const int lpr = nvec <= 6 * 8 ? 8 : (nvec <= 6 * 16 ? 16 : 32);
    const unsigned gridv = (unsigned)((rows + (32 / lpr) * wpb - 1) / ((32 / lpr) * wpb));
#define AP_LNV(L)                                                                                                        \
  AP_LAUNCH((layernormv_kernel<L>), gridv, wpb * 32, 0, stream, (const __half*)x, rows, C, eps, gamma, beta, pe,                   \
                                                       rows_per_pe > 0 ? rows_per_pe : 1, pe_period > 0 ? pe_period : 1, \
                                                       (__half*)out)
    if (lpr == 8) AP_LNV(8);
    else if (lpr == 16) AP_LNV(16);
    else AP_LNV(32);
#undef AP_LNV
    AP_CHECK_CUDA(cudaGetLastError());
    return AP_OK;
  }
  const unsigned grid = (unsigned)((rows + wpb - 1) / wpb);
  const int maxv = (C / 2 + 31) / 32;
#define AP_LN(MV)                                                                                              \
  AP_LAUNCH((layernorm_kernel<MV>), grid, wpb * 32, 0, stream, (const __half*)x, rows, C, eps, gamma, beta, pe,          \
                                                      rows_per_pe > 0 ? rows_per_pe : 1, pe_period > 0 ? pe_period : 1, \
                                                      (__half*)out)
  if (maxv <= 5) AP_LN(5);
  else if (maxv <= 10) AP_LN(10);
  else if (maxv <= 20) AP_LN(20);
  else AP_LN(32);
#undef AP_LN
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}
