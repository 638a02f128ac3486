// Temporal (frame-axis) attention core and small HBM-bound elementwise / layout kernels of the hot path.
#include <stdlib.h>

#include "ap_host.h"
#include "ap_ptx.cuh"
#include "ap_u8.cuh"

namespace ap {

// ---------------------------------------------------------------------------------------------------------
// Temporal self-attention core of the motion module: for every (batch b, spatial position p, head h) a softmax
// over the F frames of the window (F <= 32). Reads q/k/v straight out of the fused projection buffer
// [B*F*N, 3C] (token row = (b*F + f)*N + p) and writes [B*F*N, C] in the same token order, i.e. the two
// "(b f) d c <-> (b d) f c" rearranges of the reference (src/models/motion_module.py:359-386) are pure index math.
// Block = 8 warps = 8 heads of a group of positions (so whole 3C-wide token rows are consumed by one block);
// lane = (position sub-index, query frame i). K then V are staged through shared memory in channel chunks.
// ---------------------------------------------------------------------------------------------------------
template <int FP, int VEC>  // FP: frames padded to a power of two (4, 8, 16, 32); VEC: uint4 (8 halves) per channel chunk
__global__ void __launch_bounds__(256)
temporal_attn_kernel(const __half* __restrict__ qkv, long long ld, __half* __restrict__ out, long long ldo, int B,
                     int F, int N, int C, int heads, float scale) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  constexpr int PW = 32 / FP;  // positions per warp
  constexpr int CH = 8 * VEC;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int d = C / heads;
  const int head = warp % heads;
  const int sub = lane / FP;
  const int i = lane % FP;
  const long long pos_group = blockIdx.x;              // over B * ceil(N / PW)
  const int groups_per_b = (N + PW - 1) / PW;
  const int b = (int)(pos_group / groups_per_b);
  const int p = (int)(pos_group % groups_per_b) * PW + sub;
  const bool active = (i < F) && (p < N) && (warp < heads);
  extern __shared__ __align__(16) uint8_t tsm[];
  // per warp: K and V staging, PW * FP rows x CH halves each
  __half* kst = reinterpret_cast<__half*>(tsm) + (size_t)warp * 2 * PW * FP * CH;
  __half* vst = kst + PW * FP * CH;
  const long long row = ((long long)(b * F + (i < F ? i : 0))) * N + (p < N ? p : 0);
  const __half* qrow = qkv + row * ld + head * d;
  const __half* krow = qrow + C;
  const __half* vrow = qrow + 2 * C;
  __half* orow = out + row * ldo + head * d;
  const int chunks = d / CH;

  // Pass 1: S = Q.K^T accumulated over channel chunks. All global loads of a chunk are issued before any is consumed.
  float s[FP];
#pragma unroll
  for (int j = 0; j < FP; ++j) s[j] = 0.f;
  for (int c = 0; c < chunks; ++c) {
    uint4 qv[VEC], kv[VEC];
    if (active) {
#pragma unroll
      for (int u = 0; u < VEC; ++u) {
        qv[u] = __ldg(reinterpret_cast<const uint4*>(qrow + c * CH + u * 8));
        kv[u] = __ldg(reinterpret_cast<const uint4*>(krow + c * CH + u * 8));
      }
#pragma unroll
      for (int u = 0; u < VEC; ++u) *reinterpret_cast<uint4*>(kst + (sub * FP + i) * CH + u * 8) = kv[u];
    }
    __syncwarp();
    if (active) {
#pragma unroll
      for (int u = 0; u < VEC; ++u) {
        const __half2* q2 = reinterpret_cast<const __half2*>(&qv[u]);
        float2 qf[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) qf[t] = __half22float2(q2[t]);
#pragma unroll
        for (int j = 0; j < FP; ++j) {
          if (j < F) {
            const uint4 ku = *reinterpret_cast<const uint4*>(kst + (sub * FP + j) * CH + u * 8);
            const __half2* k2 = reinterpret_cast<const __half2*>(&ku);
#pragma unroll
            for (int t = 0; t < 4; ++t) {
              const float2 kf = __half22float2(k2[t]);
              s[j] = fmaf(qf[t].x, kf.x, s[j]);
              s[j] = fmaf(qf[t].y, kf.y, s[j]);
            }
          }
        }
      }
    }
    __syncwarp();
  }
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < FP; ++j)
    if (j < F) mx = fmaxf(mx, s[j] * scale);
  float l = 0.f;
#pragma unroll
  for (int j = 0; j < FP; ++j) {
    s[j] = (j < F) ? __expf(s[j] * scale - mx) : 0.f;
    l += s[j];
  }
  const float inv_l = 1.f / l;
#pragma unroll
  for (int j = 0; j < FP; ++j) s[j] *= inv_l;

  // Pass 2: O = P.V per channel chunk (next chunk's V is in flight while this one is consumed).
  uint4 vv[VEC];
  if (active) {
#pragma unroll
    for (int u = 0; u < VEC; ++u) vv[u] = __ldg(reinterpret_cast<const uint4*>(vrow + u * 8));
  }
  for (int c = 0; c < chunks; ++c) {
    if (active) {
#pragma unroll
      for (int u = 0; u < VEC; ++u) *reinterpret_cast<uint4*>(vst + (sub * FP + i) * CH + u * 8) = vv[u];
      if (c + 1 < chunks) {
#pragma unroll
        for (int u = 0; u < VEC; ++u) vv[u] = __ldg(reinterpret_cast<const uint4*>(vrow + (c + 1) * CH + u * 8));
      }
    }
    __syncwarp();
    if (active) {
#pragma unroll
      for (int u = 0; u < VEC; ++u) {
        float acc[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) acc[t] = 0.f;
#pragma unroll
        for (int j = 0; j < FP; ++j) {
          if (j < F) {
            const uint4 vu = *reinterpret_cast<const uint4*>(vst + (sub * FP + j) * CH + u * 8);
            const __half2* v2 = reinterpret_cast<const __half2*>(&vu);
#pragma unroll
            for (int t = 0; t < 4; ++t) {
              const float2 vf = __half22float2(v2[t]);
              acc[2 * t] = fmaf(s[j], vf.x, acc[2 * t]);
              acc[2 * t + 1] = fmaf(s[j], vf.y, acc[2 * t + 1]);
            }
          }
        }
        __half2 o[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) o[t] = __floats2half2_rn(acc[2 * t], acc[2 * t + 1]);
        *reinterpret_cast<uint4*>(orow + c * CH + u * 8) = *reinterpret_cast<uint4*>(o);
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------------------
// Temporal attention, F <= 16, head_dim D in {40, 80, 160}: the path every UNet call takes (F = 16 window).
// A block owns one (batch, position) and a group of HG = 320 / D heads, i.e. 320 channels of q, k and v of the F token
// rows (b*F + f)*N + p. The rows are fetched with fully coalesced 16-byte cp.async (each row contributes three contiguous
// 640-byte segments) into a padded shared tile (row stride 1936 B: conflict-free ldmatrix); one warp per head then does
// S = Q.K^T and O = P.V with mma.sync m16n8k16 (the 16 frames are exactly one MMA tile), the softmax lives in the
// accumulator registers, O goes back through shared memory (over the head's dead Q columns) and leaves as coalesced
// 640-byte row segments. The previous kernel (kept below for F > 16 / other head sizes) let every lane walk its own token
// row: 32 cache lines per load instruction and ~1.3 G scalar FMAs made it 3x slower than the HBM time of its operands.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2_t(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                          uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_1688(float* c, uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(b0));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

constexpr int TA_GC = 320;            // channels of q (and of k, v) per block
constexpr int TA_RS = 3 * TA_GC + 8;  // padded shared row stride in halves (1936 B)

template <int D>
__global__ void __launch_bounds__(32 * (TA_GC / D))
temporal_attn_mma_kernel(const __half* __restrict__ qkv, long long ld, __half* __restrict__ out, long long ldo, int F,
                         int N, int C, float scale_log2) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  constexpr int HG = TA_GC / D;        // heads (= warps) per block
  constexpr int NT = 32 * HG;
  constexpr int SEG_V = TA_GC / 8;     // uint4 per 640-byte segment
  __shared__ __align__(16) __half tile[16 * TA_RS];
  const int groups = C / TA_GC;
  const int hg = blockIdx.x % groups;
  const long long bp = blockIdx.x / groups;      // b * N + p
  const int b = (int)(bp / N), p = (int)(bp % N);
  const long long row0 = (long long)b * F * N + p;   // token row of frame f: row0 + f * N
  const uint32_t tile_s = (uint32_t)__cvta_generic_to_shared(tile);

  // ---- coalesced fetch: F rows x 3 segments (q | k | v) x 40 x 16 B
  for (int idx = threadIdx.x; idx < F * 3 * SEG_V; idx += NT) {
    const int f = idx / (3 * SEG_V), c = idx % (3 * SEG_V);
    const int seg = c / SEG_V, within = c % SEG_V;
    const __half* src = qkv + (row0 + (long long)f * N) * ld + seg * C + hg * TA_GC + within * 8;
    const uint32_t dst = tile_s + (uint32_t)(f * TA_RS + c * 8) * 2;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
  }
  if (F < 16) {   // unused frame rows must read as zeros (they enter the MMAs as K / V rows)
    for (int idx = threadIdx.x; idx < (16 - F) * 3 * SEG_V; idx += NT) {
      const int f = F + idx / (3 * SEG_V), c = idx % (3 * SEG_V);
      *reinterpret_cast<uint4*>(tile + f * TA_RS + c * 8) = make_uint4(0u, 0u, 0u, 0u);
    }
  }
  asm volatile("cp.async.commit_group;\n cp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const int g = l >> 2, q4 = l & 3;
  const int j8 = l >> 3, r8 = l & 7;
  const uint32_t q_s = tile_s + (uint32_t)(w * D) * 2;
  const uint32_t k_s = q_s + TA_GC * 2;
  const uint32_t v_s = k_s + TA_GC * 2;

  // ---- S = Q K^T   (16 x 16 per head): two n-tiles of 8 key frames
  float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int ks = 0; ks < D / 16; ++ks) {
    uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
    ldsm_x4(q_s + (uint32_t)((((j8 & 1) * 8 + r8) * TA_RS) + ks * 16 + (j8 >> 1) * 8) * 2, a0, a1, a2, a3);
    ldsm_x4(k_s + (uint32_t)((((j8 >> 1) * 8 + r8) * TA_RS) + ks * 16 + (j8 & 1) * 8) * 2, b0, b1, b2, b3);
    mma_16816(s0, a0, a1, a2, a3, b0, b1);
    mma_16816(s1, a0, a1, a2, a3, b2, b3);
  }
  if (D % 16 == 8) {   // d = 40: 8-channel tail
    constexpr int c0 = (D / 16) * 16;
    uint32_t a0, a1, b0, b1;
    const int jj = j8 & 1;   // lanes 16-31 mirror 0-15 (their addresses are ignored by .x2)
    ldsm_x2(q_s + (uint32_t)((jj * 8 + r8) * TA_RS + c0) * 2, a0, a1);
    ldsm_x2(k_s + (uint32_t)((jj * 8 + r8) * TA_RS + c0) * 2, b0, b1);
    mma_1688(s0, a0, a1, b0);
    mma_1688(s1, a0, a1, b1);
  }
  // ---- softmax over the key frames: rows g (c0,c1) and g+8 (c2,c3); columns nt*8 + 2*q4 + {0,1}
  const int col = 2 * q4;
  float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (col + e >= F) { s0[e] = -INFINITY; s0[2 + e] = -INFINITY; }
    if (8 + col + e >= F) { s1[e] = -INFINITY; s1[2 + e] = -INFINITY; }
    mx_lo = fmaxf(mx_lo, fmaxf(s0[e], s1[e]));
    mx_hi = fmaxf(mx_hi, fmaxf(s0[2 + e], s1[2 + e]));
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, o));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, o));
  }
  float l_lo = 0.f, l_hi = 0.f;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    s0[e] = exp2f((s0[e] - mx_lo) * scale_log2);
    s1[e] = exp2f((s1[e] - mx_lo) * scale_log2);
    s0[2 + e] = exp2f((s0[2 + e] - mx_hi) * scale_log2);
    s1[2 + e] = exp2f((s1[2 + e] - mx_hi) * scale_log2);
    l_lo += s0[e] + s1[e];
    l_hi += s0[2 + e] + s1[2 + e];
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, o);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, o);
  }
  const float il = 1.f / l_lo, ih = 1.f / l_hi;
  const uint32_t pa0 = pack_h2(s0[0] * il, s0[1] * il), pa1 = pack_h2(s0[2] * ih, s0[3] * ih);
  const uint32_t pa2 = pack_h2(s1[0] * il, s1[1] * il), pa3 = pack_h2(s1[2] * ih, s1[3] * ih);

  // ---- O = P V   (16 x D per head), channel n-tiles of 8, two per ldmatrix.x4.trans
  __half* o_row_lo = tile + g * TA_RS + w * D + col;          // O overwrites this head's (dead) Q columns
  __half* o_row_hi = o_row_lo + 8 * TA_RS;
#pragma unroll
  for (int np = 0; np < D / 16; ++np) {
    uint32_t b0, b1, b2, b3;
    ldsm_x4_t(v_s + (uint32_t)((((j8 & 1) * 8 + r8) * TA_RS) + (np * 2 + (j8 >> 1)) * 8) * 2, b0, b1, b2, b3);
    float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
    mma_16816(o0, pa0, pa1, pa2, pa3, b0, b1);
    mma_16816(o1, pa0, pa1, pa2, pa3, b2, b3);
    *reinterpret_cast<uint32_t*>(o_row_lo + np * 16) = pack_h2(o0[0], o0[1]);
    *reinterpret_cast<uint32_t*>(o_row_hi + np * 16) = pack_h2(o0[2], o0[3]);
    *reinterpret_cast<uint32_t*>(o_row_lo + np * 16 + 8) = pack_h2(o1[0], o1[1]);
    *reinterpret_cast<uint32_t*>(o_row_hi + np * 16 + 8) = pack_h2(o1[2], o1[3]);
  }
  if (D % 16 == 8) {
    constexpr int c0 = (D / 16) * 16;
    uint32_t b0, b1;
    ldsm_x2_t(v_s + (uint32_t)((((j8 & 1) * 8 + r8) * TA_RS) + c0) * 2, b0, b1);
    float o0[4] = {0.f, 0.f, 0.f, 0.f};
    mma_16816(o0, pa0, pa1, pa2, pa3, b0, b1);
    *reinterpret_cast<uint32_t*>(o_row_lo + c0) = pack_h2(o0[0], o0[1]);
    *reinterpret_cast<uint32_t*>(o_row_hi + c0) = pack_h2(o0[2], o0[3]);
  }
  __syncthreads();
  // ---- coalesced store: F rows x 640 B
  for (int idx = threadIdx.x; idx < F * SEG_V; idx += NT) {
    const int f = idx / SEG_V, c = idx % SEG_V;
    *reinterpret_cast<uint4*>(out + (row0 + (long long)f * N) * ldo + hg * TA_GC + c * 8) =
        *reinterpret_cast<const uint4*>(tile + f * TA_RS + c * 8);
  }
}

// ---------------------------------------------------------------------------------------------------------
// elementwise / layout helpers (16-byte vectorised)
// ---------------------------------------------------------------------------------------------------------
__global__ void add_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ o,
                           long long nvec) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; idx < nvec; idx += stride) {
    const uint4 x = __ldg(a + idx), y = __ldg(b + idx);
    uint4 r;
    const __half2* x2 = reinterpret_cast<const __half2*>(&x);
    const __half2* y2 = reinterpret_cast<const __half2*>(&y);
    __half2* r2 = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 fx = __half22float2(x2[t]), fy = __half22float2(y2[t]);
      r2[t] = __floats2half2_rn(fx.x + fy.x, fx.y + fy.y);
    }
    o[idx] = r;
  }
}

__global__ void add_bcast_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ o,
                                 long long nvec, long long nbvec) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; idx < nvec; idx += stride) {
    const uint4 x = __ldg(a + idx), y = __ldg(b + idx % nbvec);
    uint4 r;
    const __half2* x2 = reinterpret_cast<const __half2*>(&x);
    const __half2* y2 = reinterpret_cast<const __half2*>(&y);
    __half2* r2 = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 fx = __half22float2(x2[t]), fy = __half22float2(y2[t]);
      r2[t] = __floats2half2_rn(fx.x + fy.x, fx.y + fy.y);
    }
    o[idx] = r;
  }
}

__global__ void timestep_embedding_kernel(const float* __restrict__ t, int B, int dim, __half* __restrict__ out) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (idx >= B * half) return;
  const int b = idx / half, i = idx % half;
  const float freq = expf(-9.210340371976184f * (float)i / (float)half);  // ln(10000)
  const float arg = t[b] * freq;
  out[b * dim + i] = __float2half_rn(cosf(arg));
  out[b * dim + half + i] = __float2half_rn(sinf(arg));
}

__global__ void silu_kernel(const __half* __restrict__ x, __half* __restrict__ y, long long n) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n) {
    const float v = __half2float(x[idx]);
    y[idx] = __float2half_rn(v / (1.f + __expf(-v)));
  }
}

// nearest-neighbour 2x upsample, channels-last: out[n, y, x, :] = in[n, y/2, x/2, :]
__global__ void upsample2x_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int Nf, int H, int W,
                                  int cvec) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long total = (long long)Nf * 2 * H * 2 * W * cvec;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; idx < total; idx += stride) {
    const int c = (int)(idx % cvec);
    long long r = idx / cvec;
    const int x = (int)(r % (2 * W));
    r /= 2 * W;
    const int y = (int)(r % (2 * H));
    const int n = (int)(r / (2 * H));
    out[idx] = __ldg(in + (((long long)n * H + (y >> 1)) * W + (x >> 1)) * cvec + c);
  }
}

// [B, C, F, H, W] (reference layout) -> [(b f), H, W, Cpad] channels-last, zero padded channels
__global__ void ncfhw_to_nhwc_kernel(const __half* __restrict__ in, __half* __restrict__ out, int B, int C, int F,
                                     int HW, int Cpad) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long total = (long long)B * F * HW * Cpad;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; idx < total; idx += stride) {
    const int c = (int)(idx % Cpad);
    long long r = idx / Cpad;
    const int px = (int)(r % HW);
    r /= HW;
    const int f = (int)(r % F);
    const int b = (int)(r / F);
    out[idx] = c < C ? in[(((long long)b * C + c) * F + f) * HW + px] : __float2half(0.f);
  }
}

// [(b f), HW, ld] channels-last (first C channels) -> [B, C, F, H, W]
__global__ void nhwc_to_ncfhw_kernel(const __half* __restrict__ in, __half* __restrict__ out, int B, int C, int F,
                                     int HW, int ld) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long total = (long long)B * C * F * HW;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; idx < total; idx += stride) {
    const int px = (int)(idx % HW);
    long long r = idx / HW;
    const int f = (int)(r % F);
    r /= F;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    out[idx] = in[(((long long)b * F + f) * HW + px) * ld + c];
  }
}

// ---------------------------------------------------------------------------------------------------------
// Denoising-loop elementwise ops (reference src/pipelines/pipeline_pose2vid_long.py:521-559)
// latents: fp16 [L, HW, 4] channels-last master copy.
// ---------------------------------------------------------------------------------------------------------
// UNet input for one window: out[(b, f), px, 0..Cpad) = latents[idx[f], px, 0..4) duplicated over `dup` CFG branches
__global__ void gather_window_kernel(const __half* __restrict__ lat, const int* __restrict__ idx, __half* __restrict__ out,
                                     int dup, int F, int HW, int Cpad) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long total = (long long)dup * F * HW;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int px = (int)(t % HW);
  const int f = (int)((t / HW) % F);
  const uint2 v = *reinterpret_cast<const uint2*>(lat + ((long long)idx[f] * HW + px) * 4);
  uint4* o = reinterpret_cast<uint4*>(out + t * Cpad);
  o[0] = make_uint4(v.x, v.y, 0u, 0u);
  for (int u = 1; u < Cpad / 8; ++u) o[u] = make_uint4(0u, 0u, 0u, 0u);
}

// gather_window with the UNet input scaled: out = fp16_rn(fp32(lat) * scale[0]), one rounding. The scale is read from
// device memory so that a captured graph sees each step's value (EulerDiscreteScheduler.scale_model_input).
__global__ void gather_window_scaled_kernel(const __half* __restrict__ lat, const int* __restrict__ idx,
                                            const float* __restrict__ scale, __half* __restrict__ out, int dup, int F,
                                            int HW, int Cpad) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long total = (long long)dup * F * HW;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int px = (int)(t % HW);
  const int f = (int)((t / HW) % F);
  const float s = scale[0];
  const uint2 v = *reinterpret_cast<const uint2*>(lat + ((long long)idx[f] * HW + px) * 4);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
  const __half2 lo = __floats2half2_rn(a.x * s, a.y * s), hi = __floats2half2_rn(b.x * s, b.y * s);
  uint4* o = reinterpret_cast<uint4*>(out + t * Cpad);
  o[0] = make_uint4(*reinterpret_cast<const unsigned*>(&lo), *reinterpret_cast<const unsigned*>(&hi), 0u, 0u);
  for (int u = 1; u < Cpad / 8; ++u) o[u] = make_uint4(0u, 0u, 0u, 0u);
}

// acc[b, idx[f], px, :] += pred[(b, f), px, 0..4)   (fp32 accumulation of overlapping windows)
// A window that holds the same frame twice (dilated windows wrapping around a short clip) contributes that frame ONCE, from
// its last occurrence — the semantics of the reference's index assignment noise_pred[:, :, c] = noise_pred[:, :, c] + pred
// (pipeline_pose2vid_long.py:546-547), and race-free.
__global__ void scatter_accumulate_kernel(const __half* __restrict__ pred, int ld, const int* __restrict__ idx,
                                          float* __restrict__ acc, int B, int F, int L, int HW) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long total = (long long)B * F * HW;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int px = (int)(t % HW);
  const int f = (int)((t / HW) % F);
  const int b = (int)(t / ((long long)HW * F));
  const int frame = idx[f];
  for (int g = f + 1; g < F; ++g)
    if (idx[g] == frame) return;
  const __half* s = pred + t * ld;
  float4* d = reinterpret_cast<float4*>(acc + (((long long)b * L + frame) * HW + px) * 4);
  float4 a = *d;
  a.x += __half2float(s[0]); a.y += __half2float(s[1]); a.z += __half2float(s[2]); a.w += __half2float(s[3]);
  *d = a;
}

// noise = acc * inv_count ; CFG: u + g (c - u) ; DDIM step (eta = 0) ; latents updated in place; acc zeroed.
// inv_count is the caller's per-frame weight: 1 / count under CFG (the overlap average), 1 without CFG, where the reference
// steps on the sum of the overlapping windows' predictions (pipeline_pose2vid_long.py:551-559; sharding.step_weights).
// x0 = c_xx x + c_xv v, eps = c_ex x + c_ev v (the three diffusers prediction types differ only in these coefficients),
// optional clamp of x0 (clip_sample; eps is NOT recomputed: use_clipped_model_output = False), then the eta = 0 update.
__global__ void cfg_ddim_step_kernel(float* __restrict__ acc, const float* __restrict__ inv_count, int cfg, float guidance,
                                     float c_xx, float c_xv, float c_ex, float c_ev, float clip, float sqrt_ap,
                                     float sqrt_bp, __half* __restrict__ lat, int L, int HW) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long total = (long long)L * HW * 4;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int f = (int)(t / ((long long)HW * 4));
  const float ic = inv_count[f];
  float v;
  if (cfg) {
    const float u = acc[t] * ic;
    const float c = acc[total + t] * ic;
    v = u + guidance * (c - u);
    acc[total + t] = 0.f;
  } else {
    v = acc[t] * ic;
  }
  acc[t] = 0.f;
  const float x = __half2float(lat[t]);
  float x0 = c_xx * x + c_xv * v;
  const float eps = c_ex * x + c_ev * v;
  if (clip > 0.f) x0 = fminf(fmaxf(x0, -clip), clip);
  lat[t] = __float2half_rn(sqrt_ap * x0 + sqrt_bp * eps);
}

// noise = acc * inv_count ; CFG as above ; then one step of a multistep sampler (DPM-Solver(++) order 1 / 2, Euler):
//   m = c_xx x + c_xv v   (x0, or eps for dpmsolver)      x_next = k_x x + k_0 m + k_1 m_prev
// m_prev is the previous step's m, kept in fp32 in `hist`. hist is read only when k_1 != 0 (at the first step it holds
// whatever the buffer held, and 0 * NaN = NaN), and overwritten with m when the next step reads it (store).
__global__ void cfg_multistep_step_kernel(float* __restrict__ acc, const float* __restrict__ inv_count, int cfg,
                                          float guidance, float c_xx, float c_xv, float k_x, float k_0, float k_1,
                                          int store, float* __restrict__ hist, __half* __restrict__ lat, int L, int HW) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const long long total = (long long)L * HW * 4;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int f = (int)(t / ((long long)HW * 4));
  const float ic = inv_count[f];
  float v;
  if (cfg) {
    const float u = acc[t] * ic;
    const float c = acc[total + t] * ic;
    v = u + guidance * (c - u);
    acc[total + t] = 0.f;
  } else {
    v = acc[t] * ic;
  }
  acc[t] = 0.f;
  const float x = __half2float(lat[t]);
  const float m = c_xx * x + c_xv * v;
  float y = k_x * x + k_0 * m;
  if (k_1 != 0.f) y += k_1 * hist[t];
  if (store) hist[t] = m;
  lat[t] = __float2half_rn(y);
}

// ---------------------------------------------------------------------------------------------------------
// Video frames -> packed 8-bit RGB (what the reference does on the host: src/utils/util.py:87-104 save_videos_grid,
// `(x * 255).numpy().astype(np.uint8)` after an optional `(x + 1) / 2`, on the fp32 copy of the fp16 video). in: fp16
// [B, 3, F, H, W] addressed through element strides (the decoder's frames live as [F, 3, H, W]); out: [B, F, H, W, 3]
// bytes. The per-sample arithmetic is ap_u8.cuh::to_u8.
// ---------------------------------------------------------------------------------------------------------

// VEC = 4: one thread packs four neighbouring pixels of a row (three 8-byte loads, three 4-byte stores); VEC = 1: any strides
template <int VEC>
__global__ void __launch_bounds__(256)
pack_frames_u8_kernel(const __half* __restrict__ in, long long sb, long long sc, long long sf, long long sh, long long sw,
                      int B, int F, int H, int W, int rescale, uint8_t* __restrict__ out) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int Wv = W / VEC;
  const long long total = (long long)B * F * H * Wv;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; t < total; t += stride) {
    const int xv = (int)(t % Wv);
    long long r = t / Wv;
    const int y = (int)(r % H);
    r /= H;
    const int f = (int)(r % F);
    const int b = (int)(r / F);
    const __half* src = in + b * sb + f * sf + y * sh;
    if (VEC == 4) {
      unsigned px[3][4];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const uint2 v = *reinterpret_cast<const uint2*>(src + c * sc + xv * 4);
        const __half2 lo = *reinterpret_cast<const __half2*>(&v.x), hi = *reinterpret_cast<const __half2*>(&v.y);
        px[c][0] = to_u8(__low2half(lo), rescale);
        px[c][1] = to_u8(__high2half(lo), rescale);
        px[c][2] = to_u8(__low2half(hi), rescale);
        px[c][3] = to_u8(__high2half(hi), rescale);
      }
      // 12 bytes r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3 (little endian)
      uint32_t* o = reinterpret_cast<uint32_t*>(out + t * 12);
      o[0] = px[0][0] | (px[1][0] << 8) | (px[2][0] << 16) | (px[0][1] << 24);
      o[1] = px[1][1] | (px[2][1] << 8) | (px[0][2] << 16) | (px[1][2] << 24);
      o[2] = px[2][2] | (px[0][3] << 8) | (px[1][3] << 16) | (px[2][3] << 24);
    } else {
      uint8_t* o = out + t * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = (uint8_t)to_u8(src[c * sc + xv * sw], rescale);
    }
  }
}

static inline unsigned grid_for(long long n, int threads, int cap = 0) {
  if (cap <= 0) cap = num_sms() * 16;
  long long g = (n + threads - 1) / threads;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (unsigned)g;
}

}  // namespace ap

using namespace ap;

extern "C" int ap_temporal_attention_f16(const void* qkv, long long ld, void* out, long long ldo, int B, int F, int N,
                                         int C, int heads, float scale, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  AP_REQUIRE(qkv && out, "temporal_attention: null pointer");
  AP_REQUIRE(F >= 1 && F <= 32, "temporal_attention: window length %d not in [1,32]", F);
  AP_REQUIRE(heads >= 1 && heads <= 8 && C % heads == 0, "temporal_attention: heads=%d unsupported", heads);
  const int d = C / heads;
  AP_REQUIRE(d % 8 == 0 && ld % 8 == 0 && ldo % 8 == 0, "temporal_attention: head_dim/ld must be multiples of 8");
  // both kernels move q/k/v and out in 16-byte pieces (cp.async / uint4)
  AP_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "temporal_attention: qkv and out must be 16-byte aligned");
  static const bool force_scalar = getenv("AP_TEMPORAL_SCALAR") != nullptr;   // A/B switch: the pre-MMA kernel
  if (!force_scalar && F <= 16 && C % TA_GC == 0 && heads * d == C && (d == 40 || d == 80 || d == 160)) {
    const unsigned grid = (unsigned)((long long)B * N * (C / TA_GC));
    const float sl2 = scale * 1.4426950408889634f;
    if (d == 40) AP_LAUNCH((temporal_attn_mma_kernel<40>), grid, 256, 0, stream, (const __half*)qkv, ld, (__half*)out, ldo, F, N, C, sl2);
    else if (d == 80) AP_LAUNCH((temporal_attn_mma_kernel<80>), grid, 128, 0, stream, (const __half*)qkv, ld, (__half*)out, ldo, F, N, C, sl2);
    else AP_LAUNCH((temporal_attn_mma_kernel<160>), grid, 64, 0, stream, (const __half*)qkv, ld, (__half*)out, ldo, F, N, C, sl2);
    AP_CHECK_CUDA(cudaGetLastError());
    return AP_OK;
  }
  int VEC = 1;
  for (int v : {5, 4, 2, 1})
    if (d % (8 * v) == 0) { VEC = v; break; }
  const int FP = F <= 4 ? 4 : (F <= 8 ? 8 : (F <= 16 ? 16 : 32));
  const int PW = 32 / FP;
  const long long groups = (long long)B * ((N + PW - 1) / PW);
  const size_t smem = (size_t)8 * 2 * PW * FP * (8 * VEC) * sizeof(__half);
#define AP_T(FP_, V_)                                                                                             \
  AP_LAUNCH((temporal_attn_kernel<FP_, V_>), (unsigned)groups, 256, smem, stream, (const __half*)qkv, ld, (__half*)out, ldo, B, \
                                                                         F, N, C, heads, scale)
#define AP_TV(FP_)                      \
  do {                                  \
    if (VEC == 5) AP_T(FP_, 5);         \
    else if (VEC == 4) AP_T(FP_, 4);    \
    else if (VEC == 2) AP_T(FP_, 2);    \
    else AP_T(FP_, 1);                  \
  } while (0)
  if (FP == 4) AP_TV(4);
  else if (FP == 8) AP_TV(8);
  else if (FP == 16) AP_TV(16);
  else AP_TV(32);
#undef AP_TV
#undef AP_T
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_add_f16(const void* a, const void* b, void* out, long long n, void* stream) {
  AP_REQUIRE(a && b && out && n % 8 == 0, "add: n must be a multiple of 8");
  AP_REQUIRE(aligned16(a) && aligned16(b) && aligned16(out), "add: a, b and out must be 16-byte aligned");
  AP_LAUNCH((add_kernel), grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream, (const uint4*)a, (const uint4*)b, (uint4*)out, n / 8);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_add_bcast_f16(const void* a, const void* b, void* out, long long n, long long nb, void* stream) {
  AP_REQUIRE(a && b && out && n % 8 == 0 && nb % 8 == 0 && nb > 0 && n % nb == 0, "add_bcast: bad sizes");
  AP_REQUIRE(aligned16(a) && aligned16(b) && aligned16(out), "add_bcast: a, b and out must be 16-byte aligned");
  AP_LAUNCH((add_bcast_kernel), grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream, (const uint4*)a, (const uint4*)b, (uint4*)out,
                                                                         n / 8, nb / 8);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_timestep_embedding_f16(const float* t, int B, int dim, void* out, void* stream) {
  AP_REQUIRE(t && out && dim % 2 == 0, "timestep_embedding: bad arguments");
  const int n = B * dim / 2;
  AP_LAUNCH((timestep_embedding_kernel), (n + 127) / 128, 128, 0, (cudaStream_t)stream, t, B, dim, (__half*)out);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_silu_f16(const void* x, void* out, long long n, void* stream) {
  AP_REQUIRE(x && out, "silu: null pointer");
  AP_LAUNCH((silu_kernel), (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, (const __half*)x, (__half*)out, n);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_upsample2x_nhwc_f16(const void* x, void* out, int Nf, int H, int W, int C, void* stream) {
  AP_REQUIRE(x && out && C % 8 == 0, "upsample2x: C must be a multiple of 8");
  AP_REQUIRE(aligned16(x) && aligned16(out), "upsample2x: x and out must be 16-byte aligned");
  const long long total = (long long)Nf * 4 * H * W * (C / 8);
  AP_LAUNCH((upsample2x_kernel), grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const uint4*)x, (uint4*)out, Nf, H, W, C / 8);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_ncfhw_to_nhwc_f16(const void* x, void* out, int B, int C, int F, int HW, int Cpad, void* stream) {
  AP_REQUIRE(x && out && Cpad >= C, "ncfhw_to_nhwc: bad arguments");
  const long long total = (long long)B * F * HW * Cpad;
  AP_LAUNCH((ncfhw_to_nhwc_kernel), grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const __half*)x, (__half*)out, B, C, F, HW, Cpad);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_nhwc_to_ncfhw_f16(const void* x, void* out, int B, int C, int F, int HW, int ld, void* stream) {
  AP_REQUIRE(x && out && ld >= C, "nhwc_to_ncfhw: bad arguments");
  const long long total = (long long)B * C * F * HW;
  AP_LAUNCH((nhwc_to_ncfhw_kernel), grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const __half*)x, (__half*)out, B, C, F, HW, ld);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_gather_window_f16(const void* latents, const int* frame_idx, void* out, int dup, int F, int HW,
                                    int Cpad, void* stream) {
  AP_REQUIRE(latents && frame_idx && out && Cpad % 8 == 0 && Cpad >= 8, "gather_window: bad arguments");
  AP_REQUIRE(dup >= 1 && F >= 1 && HW >= 1, "gather_window: dup=%d F=%d HW=%d must be positive", dup, F, HW);
  // the kernel loads a pixel's 4 latent channels as one uint2 and stores Cpad-channel rows as uint4
  AP_REQUIRE((reinterpret_cast<uintptr_t>(latents) & 7) == 0 && aligned16(out),
             "gather_window: latents must be 8-byte and out 16-byte aligned");
  const long long total = (long long)dup * F * HW;
  AP_LAUNCH((gather_window_kernel), (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, 
      (const __half*)latents, frame_idx, (__half*)out, dup, F, HW, Cpad);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_gather_window_scaled_f16(const void* latents, const int* frame_idx, const float* scale, void* out,
                                           int dup, int F, int HW, int Cpad, void* stream) {
  AP_REQUIRE(latents && frame_idx && scale && out && Cpad % 8 == 0 && Cpad >= 8, "gather_window_scaled: bad arguments");
  AP_REQUIRE(dup >= 1 && F >= 1 && HW >= 1, "gather_window_scaled: dup=%d F=%d HW=%d must be positive", dup, F, HW);
  AP_REQUIRE((reinterpret_cast<uintptr_t>(latents) & 7) == 0 && aligned16(out),
             "gather_window_scaled: latents must be 8-byte and out 16-byte aligned");
  const long long total = (long long)dup * F * HW;
  AP_LAUNCH((gather_window_scaled_kernel), (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream,
      (const __half*)latents, frame_idx, scale, (__half*)out, dup, F, HW, Cpad);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_scatter_accumulate_f16(const void* pred, int ld, const int* frame_idx, float* acc, int B, int F,
                                         int L, int HW, void* stream) {
  AP_REQUIRE(pred && frame_idx && acc, "scatter_accumulate: null pointer");
  AP_REQUIRE(B >= 1 && F >= 1 && L >= 1 && HW >= 1 && ld >= 4,
             "scatter_accumulate: B=%d F=%d L=%d HW=%d must be positive and ld=%d >= 4", B, F, L, HW, ld);
  // one float4 read-modify-write per (b, frame, pixel)
  AP_REQUIRE(aligned16(acc), "scatter_accumulate: acc must be 16-byte aligned");
  const long long total = (long long)B * F * HW;
  AP_LAUNCH((scatter_accumulate_kernel), (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, 
      (const __half*)pred, ld, frame_idx, acc, B, F, L, HW);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_cfg_ddim_step_f16(float* acc, const float* inv_count, int cfg, float guidance, float alpha_t,
                                    float alpha_prev, int prediction_type, float clip_range, void* latents, int L, int HW,
                                    void* stream) {
  AP_REQUIRE(acc && inv_count && latents, "cfg_ddim_step: null pointer");
  AP_REQUIRE(L >= 1 && HW >= 1, "cfg_ddim_step: L=%d HW=%d must be positive", L, HW);
  const float sa = sqrtf(alpha_t), sb = sqrtf(1.f - alpha_t);
  float c_xx, c_xv, c_ex, c_ev;
  if (prediction_type == AP_PRED_V) {
    c_xx = sa; c_xv = -sb; c_ex = sb; c_ev = sa;
  } else if (prediction_type == AP_PRED_EPSILON) {
    AP_REQUIRE(alpha_t > 0.f, "cfg_ddim_step: epsilon prediction needs alpha_t > 0");
    c_xx = 1.f / sa; c_xv = -sb / sa; c_ex = 0.f; c_ev = 1.f;
  } else if (prediction_type == AP_PRED_SAMPLE) {
    AP_REQUIRE(alpha_t < 1.f, "cfg_ddim_step: sample prediction needs alpha_t < 1");
    c_xx = 0.f; c_xv = 1.f; c_ex = 1.f / sb; c_ev = -sa / sb;
  } else {
    return ap::fail(AP_ERR_INVALID, "cfg_ddim_step: unknown prediction_type %d", prediction_type);
  }
  const long long total = (long long)L * HW * 4;
  AP_LAUNCH((cfg_ddim_step_kernel), (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, 
      acc, inv_count, cfg, guidance, c_xx, c_xv, c_ex, c_ev, clip_range, sqrtf(alpha_prev), sqrtf(1.f - alpha_prev),
      (__half*)latents, L, HW);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_cfg_multistep_step_f16(float* acc, const float* inv_count, int cfg, float guidance, float c_xx,
                                         float c_xv, float k_x, float k_0, float k_1, int store, float* hist,
                                         void* latents, int L, int HW, void* stream) {
  AP_REQUIRE(acc && inv_count && latents, "cfg_multistep_step: null pointer");
  AP_REQUIRE(L >= 1 && HW >= 1, "cfg_multistep_step: L=%d HW=%d must be positive", L, HW);
  AP_REQUIRE(hist || (k_1 == 0.f && !store), "cfg_multistep_step: k_1 != 0 or store needs the history buffer");
  AP_REQUIRE(isfinite(guidance) && isfinite(c_xx) && isfinite(c_xv) && isfinite(k_x) && isfinite(k_0) && isfinite(k_1),
             "cfg_multistep_step: non-finite coefficient");
  const long long total = (long long)L * HW * 4;
  AP_LAUNCH((cfg_multistep_step_kernel), (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream,
      acc, inv_count, cfg, guidance, c_xx, c_xv, k_x, k_0, k_1, store ? 1 : 0, hist, (__half*)latents, L, HW);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_pack_frames_u8(const void* video, const long long* strides, int B, int F, int H, int W, int rescale,
                                 void* out, void* stream) {
  AP_REQUIRE(video && strides && out && B > 0 && F > 0 && H > 0 && W > 0, "pack_frames_u8: bad arguments");
  const long long sb = strides[0], sc = strides[1], sf = strides[2], sh = strides[3], sw = strides[4];
  const bool vec = sw == 1 && W % 4 == 0 && sb % 4 == 0 && sc % 4 == 0 && sf % 4 == 0 && sh % 4 == 0 &&
                   ((uintptr_t)video & 7) == 0 && ((uintptr_t)out & 3) == 0;
  if (vec) {
    const long long total = (long long)B * F * H * (W / 4);
    AP_LAUNCH((pack_frames_u8_kernel<4>), grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const __half*)video, sb, sc,
              sf, sh, sw, B, F, H, W, rescale, (uint8_t*)out);
  } else {
    const long long total = (long long)B * F * H * W;
    AP_LAUNCH((pack_frames_u8_kernel<1>), grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const __half*)video, sb, sc,
              sf, sh, sw, B, F, H, W, rescale, (uint8_t*)out);
  }
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}
