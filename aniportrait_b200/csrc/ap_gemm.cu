// wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
//   out[M, N] = epilogue( A[M, K] * W[N, K]^T )           fp16 operands, fp32 accumulation in registers
//
// One persistent CTA per SM, warp-specialised, 128 x BN output tiles:
//   warpgroup 0     TMA producer  (warp 0: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier full/empty)
//   warpgroups 1-2  consumers     (wgmma m64nBNk16: warpgroup g computes tile rows [64 g, +64) and then runs the epilogue
//                                  of those rows: accumulators -> fp32 shared staging -> +bias, +residual | GEGLU -> fp16 ->
//                                  swizzled smem box -> TMA store); the producer runs ahead into the next tile meanwhile
//
// The A operand is fetched by TMA in one of three addressing modes, so that linear layers, 1x1 convs, 3x3 convs
// (stride 1 and 2, zero padding via TMA out-of-bounds fill) and channel-concatenated inputs (two K sources) share
// one mainloop and no im2col / concat buffer is ever materialised:
//   A_GEMM      2-D map [M, K]            (optionally a second map: K = K1 ++ K2)
//   A_CONV_S1   4-D map (C, W, H, Nf)     box {64, bw, bh, bn}, tap (ky,kx) -> coordinate shift (kx-1, ky-1)
//   A_CONV_S2   5-D map (2C, W/2, 2, H/2, Nf) (even/odd pixel phases split out), box {64, bw, 1, bh, bn}
//
// Replaces, for the hot path: cuDNN/cuBLAS calls behind InflatedConv3d (reference src/models/resnet.py:10-18),
// nn.Linear / 1x1 nn.Conv2d in Transformer3DModel (src/models/transformer_3d.py:64-66,93-95), diffusers Attention
// to_q/k/v/out and FeedForward(GEGLU) (src/models/attention.py:323-361, src/models/motion_module.py:122,144,233).
#include <stdio.h>
#include <stdlib.h>

#include "ap_host.h"
#include "ap_ptx.cuh"
#include "ap_wgmma.cuh"

namespace ap {

enum { A_GEMM = 0, A_CONV_S1 = 1, A_CONV_S2 = 2 };
enum { EPI_LINEAR = 0, EPI_GEGLU = 1 };

struct GemmParams {
  int M, N;                // output rows; weight rows (N % BN == 0)
  int num_m_tiles, num_n_tiles, num_kb;
  int a_mode;
  int kb_src1, kb_src2;    // 64-wide k-blocks per tap taken from source 1 / source 2
  // conv geometry (output grid) and tile box
  int Nf, Ho, Wo;
  int bw, bh, bn;
  int tiles_x, tiles_y;
  int C1, C2;              // channels of source 1 / 2 (A_CONV_S2: each source's merged (phase, channel) coordinate)
  // epilogue
  const float* bias;       // [groups, Nout] fp32 or null
  int bias_group_rows;     // rows sharing one bias row (>= M -> single row)
  long long bias_ld;       // floats between bias rows (N unless several ops share one table)
  const __half* residual;  // [M, ldr] or null
  int ldr;
  __half* out;             // [M, ldo]
  int ldo;
  int out_al16, res_al16;  // out / residual base 16-byte aligned: the direct epilogue may use 16-byte vector accesses
  int n_valid;             // columns >= n_valid are not stored
  int out_f32;             // store fp32 instead of fp16 (small bias-table GEMMs)
  int gelu;                // AP_GEMM_GELU: out = gelu_erf(acc + bias) (never with a residual)
  int quick_gelu;          // AP_GEMM_QUICK_GELU: out = quick_gelu(acc + bias) (same restrictions; never with gelu)
  // TMA epilogue (per-warp 32-row x 32-column boxes staged in 64B-swizzled shared memory)
  int tma_epi;             // 1: outputs leave through TMA stores, the residual arrives through TMA loads
  int sub_w, sub_h, sub_n; // conv modes: geometry of a warp's 32-row sub-box
  int epi_double;          // double-buffered output staging when there is no residual (AP_GEMM_EPI_DOUBLE=0 disables: A/B)
  int debug;               // AP_GEMM_DEBUG: 1 = skip TMA loads (MMA pace), 2 = skip MMAs (TMA pace), 3 / 4 = skip every other
                           // B / A load (traffic sensitivity); results are garbage
  // ---- statistics fused into the epilogue (TMA epilogue only) --------------------------------------------------------
  // Producer side. Both are computed from the fp16-ROUNDED outputs (what the consumer will read) and written as per-warp
  // partials in a fixed layout: no atomics, the consumer adds them in a fixed order (bit-reproducible).
  float2* row_stat_out;    // LayerNorm of the NEXT op: {sum, sum of squares} of output row m over the columns this epilogue
                           // warp handled: [part][row_stat_ld], part = 2 * (n-group of the work item) + (warp's column half)
  long long row_stat_ld;
  float2* col_stat_out;    // GroupNorm of the NEXT op: {sum, sumsq} per output column over the 32 rows of the warp's 32-row
                           // quarter: [4 * m_tile + quarter][col_stat_ld]
  long long col_stat_ld;
  // Consumer side (LayerNorm folded into this GEMM): A = [x | -mean (hi, lo, hi)], W = [W diag(gamma) | colsum (hi, hi, lo)],
  // so the accumulator already holds x.W'^T - mean colsum(W') (the mean term rides on one extra k-block of the tensor
  // core; the two-source A path existed for the skip concat); the epilogue only scales by the row's rstd:
  //   out = rstd * acc + (beta.W^T + b)   [the last term arrives as `bias`]: one FMA where the bias add used to be.
  const float* ln_rstd;    // [M] fp32, written by ln_finalize_kernel from the producer's row partials
};


// The epilogue reads the accumulators row-per-thread (a thread owns one output row and 32 consecutive columns), while
// wgmma leaves each row spread over a quad of threads. Every consumer warpgroup therefore passes its accumulators through
// an fp32 shared staging area, ACC_PW columns (two epilogue chunks) at a time.
template <int BN, int EPI>
struct GemmCfg {
  static constexpr int BM = 128;
  static constexpr int BK = 64;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int EPI_STAGING = 8 * 4096;  // 8 epilogue warps x (2 KB output box + 2 KB residual box)
  static constexpr int ACC_PW = EPI == EPI_GEGLU ? 128 : 64;
  static constexpr int ACC_LD = ACC_PW + 8;     // +8 floats: conflict-free float2 writes of the wgmma fragments
  static constexpr int ACC_STAGING = 2 * 64 * ACC_LD * 4;
  static constexpr int MAX_SMEM = 227 * 1024 - 1024 /*align slack*/ - 256 /*barriers*/ - EPI_STAGING - ACC_STAGING;
  static constexpr int STAGES_RAW = MAX_SMEM / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_STAGING + ACC_STAGING + 1024 + 256;
  static_assert(STAGES >= 2, "need at least a double-buffered operand ring");
  static_assert(B_BYTES % 1024 == 0, "B stage must keep 1024B alignment");
};


template <int BN, int EPI>
__global__ void __launch_bounds__(384, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmA2,
            const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
            const __grid_constant__ CUtensorMap tmRes, const GemmParams p) {
  using Cfg = GemmCfg<BN, EPI>;
  constexpr int STAGES = Cfg::STAGES;
  griddep_launch_dependents();   // PDL: the next kernel may be scheduled; it waits for this one in ITS griddep_wait()
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * Cfg::A_BYTES;
  uint8_t* smem_epi = smem + STAGES * Cfg::STAGE_BYTES;   // 1024-aligned: per epilogue warp [2 KB out | 2 KB residual]
  float* smem_acc = reinterpret_cast<float*>(smem_epi + Cfg::EPI_STAGING);   // per consumer warpgroup [64][ACC_LD]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_acc + 2 * 64 * Cfg::ACC_LD);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* res_bar = empty_bar + STAGES;   // [8] one per epilogue warp

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_groups = p.num_n_tiles;
  const int num_tiles = p.num_m_tiles * n_groups;
  const int first_tile = blockIdx.x;
  const int tile_stride = gridDim.x;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA1);
    tma_prefetch_desc(&tmB);
    if (p.kb_src2 > 0) tma_prefetch_desc(&tmA2);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);   // one arrival per consumer warp
    }
    for (int s = 0; s < 8; ++s) mbar_init(&res_bar[s], 1);
    if (p.tma_epi) {
      tma_prefetch_desc(&tmOut);
      if (p.residual != nullptr) tma_prefetch_desc(&tmRes);
    }
    fence_mbar_init();
  }
  __syncthreads();
  // everything above (barriers, descriptor prefetch) is independent of the previous kernel's data; from here on the
  // TMA loads / epilogue reads touch it: wait until the previous kernel of the stream has completed (PDL)
  griddep_wait();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp != 0) return;
    // ------------------------------------------------------------------ TMA producer (warp-uniform loop, elected lane
    // issues; tap / channel-block indices advance incrementally instead of by per-k-block integer division)
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = first_tile; tile < num_tiles; tile += tile_stride) {
      const int m_tile = tile / n_groups;
      const int n_tile = tile % n_groups;
      int n0 = 0, y0 = 0, x0 = 0;
      if (p.a_mode != A_GEMM) {
        const int per_frame = p.tiles_x * p.tiles_y;
        const int tn = m_tile / per_frame;
        const int rem = m_tile % per_frame;
        n0 = tn * p.bn;
        y0 = (rem / p.tiles_x) * p.bh;
        x0 = (rem % p.tiles_x) * p.bw;
      }
      int within = 0, kx = 0, ky = 0;   // channel block inside the tap; tap = (ky, kx)
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait_quiet(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          if (p.debug == 1) {   // timing experiment: no loads at all, the MMA consumes stale shared memory
            mbar_arrive(&full_bar[stage]);
          } else {
            // debug 3 / 4 (timing experiments, garbage results): odd k-blocks skip the B / the A load
            const bool load_a = !(p.debug == 4 && (kb & 1)), load_b = !(p.debug == 3 && (kb & 1));
            mbar_arrive_expect_tx(&full_bar[stage], (load_a ? Cfg::A_BYTES : 0) + (load_b ? Cfg::B_BYTES : 0));
            void* a_dst = smem_a + stage * Cfg::A_BYTES;
            void* b_dst = smem_b + stage * Cfg::B_BYTES;
            const bool second = within >= p.kb_src1;
            const CUtensorMap* am = second ? &tmA2 : &tmA1;
            const int c0 = (second ? within - p.kb_src1 : within) * Cfg::BK;
            if (!load_a) {
            } else if (p.a_mode == A_GEMM) {
              tma_load_2d(am, &full_bar[stage], a_dst, c0, m_tile * Cfg::BM);
            } else if (p.a_mode == A_CONV_S1) {
              tma_load_4d(am, &full_bar[stage], a_dst, c0, x0 + kx - 1, y0 + ky - 1, n0);
            } else {
              // input pixel = 2*o + k - 1  ->  k=0: (o-1, phase 1), k=1: (o, phase 0), k=2: (o, phase 1)
              const int px = (kx == 1) ? 0 : 1, dx = (kx == 0) ? -1 : 0;
              const int py = (ky == 1) ? 0 : 1, dy = (ky == 0) ? -1 : 0;
              tma_load_5d(am, &full_bar[stage], a_dst, px * (second ? p.C2 : p.C1) + c0, x0 + dx, py, y0 + dy, n0);
            }
            if (load_b) tma_load_2d(&tmB, &full_bar[stage], b_dst, kb * Cfg::BK, n_tile * BN);
          }
        }
        __syncwarp();
        if (++within == p.kb_src1 + p.kb_src2) {
          within = 0;
          if (++kx == 3) { kx = 0; ++ky; }
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: mainloop + epilogue
  setmaxnreg_inc<232>();
  const int wg = (warp >> 2) - 1;        // tile rows [64 wg, +64)
  const int wq = warp & 3;
  // epilogue roles: 32-row quarter of the tile, and which of every two 32-column chunks this warp takes
  const int lane_group = 2 * wg + (wq & 1);
  const int col_half = wq >> 1;
  const int row = lane_group * 32 + lane;
  const int r0 = lane_group * 32;
  float* acc_stage = smem_acc + wg * 64 * Cfg::ACC_LD;
  const float* acc_row = acc_stage + ((wq & 1) * 32 + lane) * Cfg::ACC_LD;
  constexpr int ACC_PER_CHUNK = (EPI == EPI_GEGLU) ? 64 : 32;
  constexpr int NCHUNK = BN / ACC_PER_CHUNK;
  constexpr int NPASS = (BN + Cfg::ACC_PW - 1) / Cfg::ACC_PW;
  const uint32_t a_base = smem_u32(smem_a) + wg * (64 * 128), b_base = smem_u32(smem_b);
  int stage = 0;
  uint32_t phase = 0;

  const int ew = warp - 4;
  uint8_t* obuf0 = smem_epi + ew * 4096;
  uint8_t* rbuf = obuf0 + 2048;
  // Without a residual the second 2 KB box of this warp is free: the output staging is then DOUBLE-buffered, so a chunk's
  // fp16 tile can be written while the TMA store of the previous chunk is still reading the other box.
  uint32_t ochunk = 0;
  uint64_t* rbar = &res_bar[ew];
  uint32_t rphase = 0;
  const bool has_res = (EPI == EPI_LINEAR) && p.residual != nullptr;
  const int sw = (lane >> 1) & 3;                       // 64B-swizzle XOR term of this thread's row
  // LayerNorm-folding consumers: rstd of this thread's row in the NEXT tile
  float ln_next = 1.f;
  auto ln_prefetch = [&](int tile_) {
    if (tile_ >= num_tiles) return;
    const long long mm = (long long)(tile_ / n_groups) * Cfg::BM + r0 + lane;   // A_GEMM rows
    ln_next = mm < p.M ? __ldg(p.ln_rstd + mm) : 1.f;
  };
  if (p.tma_epi && p.ln_rstd != nullptr) ln_prefetch(first_tile);

  float acc[BN / 2];
  for (int tile = first_tile; tile < num_tiles; tile += tile_stride) {
    const int m_tile = tile / n_groups;
    const int n_tile = tile % n_groups;
    // ---------------------------------------------------------------- mainloop: one wgmma group per 64-wide k-block,
    // one group kept in flight; a stage is released once the group that read it has completed
    int prev_stage = -1;
    for (int kb = 0; kb < p.num_kb; ++kb) {
      mbar_wait_quiet(&full_bar[stage], phase);
      if (p.debug != 2) {
        wgmma_fence();
        const uint64_t da = wgmma_desc_k_sw128(a_base + stage * Cfg::A_BYTES);
        const uint64_t db = wgmma_desc_k_sw128(b_base + stage * Cfg::B_BYTES);
#pragma unroll
        for (int k = 0; k < Cfg::BK / 16; ++k) wgmma_ss<BN>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        wgmma_commit();
      }
      wgmma_wait<1>();
      if (prev_stage >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      }
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    reg_fence<BN / 2>(acc);
    __syncwarp();
    if (lane == 0 && prev_stage >= 0) mbar_arrive(&empty_bar[prev_stage]);

    // ---------------------------------------------------------------- epilogue
    // coordinates of this warp's 32-row box and of this thread's output row
    int cy = 0, cx = 0, cn = 0;
    long long m = 0;
    bool row_ok = true;
    if (p.a_mode == A_GEMM) {
      cy = m_tile * Cfg::BM + r0;
      m = (long long)cy + lane;
      row_ok = m < p.M;
    } else {
      const int per_frame = p.tiles_x * p.tiles_y;
      const int tn = m_tile / per_frame;
      const int rem = m_tile % per_frame;
      cn = tn * p.bn + r0 / (p.bh * p.bw);
      cy = (rem / p.tiles_x) * p.bh + (r0 / p.bw) % p.bh;
      cx = (rem % p.tiles_x) * p.bw + r0 % p.bw;
      const int n = tn * p.bn + row / (p.bh * p.bw);
      const int y = (rem / p.tiles_x) * p.bh + (row / p.bw) % p.bh;
      const int x = (rem % p.tiles_x) * p.bw + row % p.bw;
      row_ok = (n < p.Nf) && (y < p.Ho) && (x < p.Wo);
      m = ((long long)n * p.Ho + y) * p.Wo + x;
    }
    const float* bias_row = nullptr;
    if (p.bias != nullptr) bias_row = p.bias + (row_ok ? (m / p.bias_group_rows) : 0) * p.bias_ld;
    // LayerNorm folding (consumer): the row's rstd, requested one tile ago
    float ln_a = 1.f;
    if (p.tma_epi && p.ln_rstd != nullptr) {
      ln_a = ln_next;
      ln_prefetch(tile + tile_stride);
    }
    float rs_s = 0.f, rs_q = 0.f;   // producer: this warp's share of the row's {sum, sumsq}
    const bool want_stats = (EPI == EPI_LINEAR) && (p.row_stat_out != nullptr || p.col_stat_out != nullptr);
    auto load_res = [&](int chunk) {
      if (lane == 0) {
        mbar_arrive_expect_tx(rbar, 2048);
        const int col = n_tile * BN + chunk * 32;
        if (p.a_mode == A_GEMM) tma_load_2d(&tmRes, rbar, rbuf, col, cy);
        else tma_load_4d(&tmRes, rbar, rbuf, col, cx, cy, cn);
      }
    };
    if (p.tma_epi && has_res && col_half < NCHUNK) load_res(col_half);

    // TMA epilogue. Each warp owns rows [32*lane_group, +32) of the tile and every other 32-output-column chunk. A chunk
    // travels staging -> registers -> (bias / residual / GEGLU) -> fp16 -> this warp's 2 KB shared box (64B swizzle:
    // bank-conflict free row-per-thread writes) -> one TMA store; the residual chunk arrives the same way through a TMA
    // load that is issued one chunk ahead. `src` is this thread's row of the chunk in the accumulator staging.
    auto chunk_tma = [&](int c, const float* src) {
      const int acol = n_tile * BN + c * ACC_PER_CHUNK;       // first accumulator (weight-row) column
      float v[32];
      if (EPI == EPI_GEGLU) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float bv[16], bg[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) { bv[j] = 0.f; bg[j] = 0.f; }
          if (bias_row != nullptr) {
            const float4* b4 = reinterpret_cast<const float4*>(bias_row + acol + h * 32);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float4 a = __ldg(b4 + j), g = __ldg(b4 + 4 + j);
              bv[4 * j] = a.x; bv[4 * j + 1] = a.y; bv[4 * j + 2] = a.z; bv[4 * j + 3] = a.w;
              bg[4 * j] = g.x; bg[4 * j + 1] = g.y; bg[4 * j + 2] = g.z; bg[4 * j + 3] = g.w;
            }
          }
#pragma unroll
          for (int j = 0; j < 16; ++j)
            v[h * 16 + j] = fmaf(src[h * 32 + j], ln_a, bv[j]) * gelu_erf(fmaf(src[h * 32 + 16 + j], ln_a, bg[j]));
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 a = reinterpret_cast<const float4*>(src)[j];
          v[4 * j] = a.x; v[4 * j + 1] = a.y; v[4 * j + 2] = a.z; v[4 * j + 3] = a.w;
        }
        if (p.ln_rstd != nullptr) {   // v = rstd * acc + bias (the folded beta.W^T + b: always present)
          const float4* b4 = reinterpret_cast<const float4*>(bias_row + acol);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 b = __ldg(b4 + j);
            v[4 * j + 0] = fmaf(v[4 * j + 0], ln_a, b.x);
            v[4 * j + 1] = fmaf(v[4 * j + 1], ln_a, b.y);
            v[4 * j + 2] = fmaf(v[4 * j + 2], ln_a, b.z);
            v[4 * j + 3] = fmaf(v[4 * j + 3], ln_a, b.w);
          }
        } else if (bias_row != nullptr) {
          const float4* b4 = reinterpret_cast<const float4*>(bias_row + acol);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 b = __ldg(b4 + j);
            v[4 * j + 0] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.z; v[4 * j + 3] += b.w;
          }
        }
        if (p.gelu) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
        } else if (p.quick_gelu) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = quick_gelu(v[j]);
        }
        if (has_res) {
          mbar_wait_quiet(rbar, rphase);
          rphase ^= 1;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const uint4 u = *reinterpret_cast<const uint4*>(rbuf + lane * 64 + ((q ^ sw) << 4));
            const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 f = __half22float2(h2[j]);
              v[q * 8 + 2 * j] += f.x;
              v[q * 8 + 2 * j + 1] += f.y;
            }
          }
        }
      }
      // the TMA store that last read the staging box we are about to overwrite must have finished reading it
      const bool dbl = !has_res && p.epi_double;
      uint8_t* obuf = (dbl && (ochunk & 1)) ? rbuf : obuf0;
      ++ochunk;
      if (lane == 0) {
        if (dbl) tma_store_wait_read<1>();
        else tma_store_wait_read<0>();
      }
      __syncwarp();
      if (want_stats && !row_ok) {   // rows past the end of the tensor are clipped by the store; keep them out of the sums
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = 0.f;
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        __half2 o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = __floats2half2_rn(v[q * 8 + 2 * j], v[q * 8 + 2 * j + 1]);
        if (EPI == EPI_LINEAR && p.row_stat_out != nullptr) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(o[j]);
            rs_s += f.x + f.y;
            rs_q = fmaf(f.x, f.x, fmaf(f.y, f.y, rs_q));
          }
        }
        *reinterpret_cast<uint4*>(obuf + lane * 64 + ((q ^ sw) << 4)) = *reinterpret_cast<uint4*>(o);
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (EPI == EPI_LINEAR && p.col_stat_out != nullptr) {
        // column sums over the 32 rows of this warp's box, read back from the staged fp16 tile: lane = (row parity,
        // half2 column), 16 conflict-free 4-byte loads per lane, then the two row parities are added
        const int hc = lane & 15, rp = lane >> 4;
        float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll
        for (int rr = 0; rr < 16; ++rr) {
          const int rw = 2 * rr + rp;
          const uint32_t u = *reinterpret_cast<const uint32_t*>(
              obuf + rw * 64 + ((((hc >> 2) ^ ((rw >> 1) & 3))) << 4) + ((hc & 3) << 2));
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u));
          s0 += f.x; q0 = fmaf(f.x, f.x, q0);
          s1 += f.y; q1 = fmaf(f.y, f.y, q1);
        }
        s0 += __shfl_xor_sync(0xffffffffu, s0, 16);
        q0 += __shfl_xor_sync(0xffffffffu, q0, 16);
        s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
        q1 += __shfl_xor_sync(0xffffffffu, q1, 16);
        if (lane < 16) {
          float4* dst = reinterpret_cast<float4*>(p.col_stat_out + (long long)(m_tile * 4 + lane_group) * p.col_stat_ld +
                                                  n_tile * BN + c * 32 + 2 * hc);
          *dst = make_float4(s0, q0, s1, q1);
        }
      }
      if (has_res && c + 2 < NCHUNK) load_res(c + 2);      // rbuf fully consumed by every lane (syncwarp above)
      if (lane == 0) {
        const int ocol = n_tile * (BN / (EPI == EPI_GEGLU ? 2 : 1)) + c * 32;
        if (p.a_mode == A_GEMM) tma_store_2d(&tmOut, obuf, ocol, cy);
        else tma_store_4d(&tmOut, obuf, ocol, cx, cy, cn);
        tma_store_commit();
      }
    };

    // direct-store epilogue (outputs or residual that TMA cannot address, fp32 outputs)
    auto chunk_direct = [&](int c, const float* src) {
      if (EPI == EPI_GEGLU) {
        // interleaved weights: columns [0,16) = value half, [16,32) = gate half of the same 16 outputs
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ncol = n_tile * BN + c * 64 + h * 32;
          const float* s = src + h * 32;
          float v[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = s[j] + (bias_row != nullptr ? __ldg(bias_row + ncol + j) : 0.f);
          const int ocol = ncol >> 1;
          if (row_ok) {
            __half2 o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float a0 = v[2 * j] * gelu_erf(v[16 + 2 * j]);
              const float a1 = v[2 * j + 1] * gelu_erf(v[16 + 2 * j + 1]);
              o[j] = __floats2half2_rn(a0, a1);
            }
            __half* dst = p.out + m * p.ldo + ocol;
            if (ocol + 16 <= p.n_valid && (p.ldo & 7) == 0 && p.out_al16) {
              uint4* d4 = reinterpret_cast<uint4*>(dst);
              d4[0] = *reinterpret_cast<uint4*>(&o[0]);
              d4[1] = *reinterpret_cast<uint4*>(&o[4]);
            } else {
              const __half* oh = reinterpret_cast<const __half*>(o);
              for (int j = 0; j < 16; ++j)
                if (ocol + j < p.n_valid) dst[j] = oh[j];
            }
          }
        }
        return;
      }
      const int ncol = n_tile * BN + c * 32;  // column in weight-row space
      float v[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = src[j];
      if (bias_row != nullptr) {
        const float4* b4 = reinterpret_cast<const float4*>(bias_row + ncol);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 b = __ldg(b4 + j);
          v[4 * j + 0] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.z; v[4 * j + 3] += b.w;
        }
      }
      if (p.gelu) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
      } else if (p.quick_gelu) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = quick_gelu(v[j]);
      }
      if (!row_ok) return;
      const bool vec_ok = (ncol + 32 <= p.n_valid) && ((p.ldo & 7) == 0) && p.out_al16;
      if (p.residual != nullptr) {
        if (ncol + 32 <= p.n_valid && (p.ldr & 7) == 0 && p.res_al16) {
          const uint4* r4 = reinterpret_cast<const uint4*>(p.residual + m * p.ldr + ncol);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const uint4 u = __ldg(r4 + q);
            const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 f = __half22float2(h2[j]);
              v[q * 8 + 2 * j] += f.x;
              v[q * 8 + 2 * j + 1] += f.y;
            }
          }
        } else {
          const __half* rs = p.residual + m * p.ldr + ncol;
          for (int j = 0; j < 32; ++j)
            if (ncol + j < p.n_valid) v[j] += __half2float(rs[j]);
        }
      }
      __half* dst = p.out + m * p.ldo + ncol;
      if (p.out_f32) {
        float* dstf = reinterpret_cast<float*>(p.out) + m * p.ldo + ncol;
        for (int j = 0; j < 32; ++j)
          if (ncol + j < p.n_valid) dstf[j] = v[j];
      } else if (vec_ok) {
        uint4* d4 = reinterpret_cast<uint4*>(dst);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          __half2 o[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) o[j] = __floats2half2_rn(v[q * 8 + 2 * j], v[q * 8 + 2 * j + 1]);
          d4[q] = *reinterpret_cast<uint4*>(o);
        }
      } else {
        for (int j = 0; j < 32; ++j)
          if (ncol + j < p.n_valid) dst[j] = __float2half_rn(v[j]);
      }
    };

#pragma unroll
    for (int ps = 0; ps < NPASS; ++ps) {
      // fragments of accumulator columns [ps * ACC_PW, +ACC_PW) -> staging (rows wq*16 + lane/4 and +8 of this warpgroup)
#pragma unroll
      for (int jl = 0; jl < Cfg::ACC_PW / 8; ++jl) {
        const int jn = ps * (Cfg::ACC_PW / 8) + jl;
        if (jn < BN / 8) {
          float* d0 = acc_stage + (wq * 16 + (lane >> 2)) * Cfg::ACC_LD + jl * 8 + 2 * (lane & 3);
          *reinterpret_cast<float2*>(d0) = make_float2(acc[4 * jn], acc[4 * jn + 1]);
          *reinterpret_cast<float2*>(d0 + 8 * Cfg::ACC_LD) = make_float2(acc[4 * jn + 2], acc[4 * jn + 3]);
        }
      }
      named_bar_sync(1 + wg, 128);
      const int c = ps * 2 + col_half;
      if (c < NCHUNK) {
        const float* src = acc_row + col_half * ACC_PER_CHUNK;
        if (p.tma_epi) chunk_tma(c, src);
        else chunk_direct(c, src);
      }
      named_bar_sync(1 + wg, 128);   // staging fully read before the next pass overwrites it
    }
    if (p.tma_epi && EPI == EPI_LINEAR && p.row_stat_out != nullptr && row_ok)
      p.row_stat_out[(long long)(2 * n_tile + col_half) * p.row_stat_ld + m] = make_float2(rs_s, rs_q);
  }
  if (p.tma_epi && lane == 0) tma_store_wait_all<0>();   // stores must complete before the CTA (and its smem) goes away
}

// ------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------
template <int BN, int EPI>
static int launch_gemm(const CUtensorMap& a1, const CUtensorMap& a2, const CUtensorMap& b, const CUtensorMap& to,
                       const CUtensorMap& tr, const GemmParams& p, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, EPI>;
  static bool attr_set = false;
  if (!attr_set) {
    AP_CHECK_CUDA(cudaFuncSetAttribute(gemm_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       Cfg::SMEM_BYTES));
    attr_set = true;
  }
  const int items = p.num_m_tiles * p.num_n_tiles;
  const int grid = items < num_sms() ? items : num_sms();
  {
    cudaError_t le = launch_pdl(gemm_kernel<BN, EPI>, dim3(grid), dim3(384), (size_t)Cfg::SMEM_BYTES, stream, 1, a1, a2,
                                b, to, tr, p);
    if (le != cudaSuccess) return fail(AP_ERR_CUDA, "gemm launch: %s", cudaGetErrorString(le));
  }
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

// Tile-width choice: wider tiles re-use the A operand more (less L2 traffic per FLOP) but give fewer tiles; small-M
// problems (16x16 / 8x8 levels) prefer narrower tiles to fill the SMs and reduce wave-quantisation loss. 256-wide tiles
// are only built on request (block_n): their 128 accumulator registers per thread spill in the epilogue.
static int pick_bn(int N, int forced, long long m_tiles, bool geglu = false) {
  if (forced > 0) return forced;
  const int cand[4] = {160, 128, 64, 32};
  const double quality[4] = {0.95, 0.90, 0.70, 0.45};
  int best = -1;
  double best_score = -1.0;
  const int sms = num_sms();
  for (int i = 0; i < 4; ++i) {
    if (N % cand[i] != 0) continue;
    if (geglu && cand[i] % 64 != 0) continue;   // a GEGLU output chunk needs 64 accumulator columns
    const long long tiles = m_tiles * (N / cand[i]);
    const long long waves = (tiles + sms - 1) / sms;
    const double fill = (double)tiles / (double)(waves * sms);
    const double score = fill * quality[i];
    if (score > best_score + 1e-9) { best_score = score; best = cand[i]; }
  }
  return best;
}

static int dispatch(int bn, int epi, const CUtensorMap& a1, const CUtensorMap& a2, const CUtensorMap& b,
                    const CUtensorMap& to, const CUtensorMap& tr, const GemmParams& p, cudaStream_t stream) {
  if (epi == EPI_GEGLU) {
    switch (bn) {
      case 128: return launch_gemm<128, EPI_GEGLU>(a1, a2, b, to, tr, p, stream);
      case 64: return launch_gemm<64, EPI_GEGLU>(a1, a2, b, to, tr, p, stream);
      default: return fail(AP_ERR_INVALID, "gemm: unsupported GEGLU BLOCK_N %d", bn);
    }
  }
  switch (bn) {
    case 256: return launch_gemm<256, EPI_LINEAR>(a1, a2, b, to, tr, p, stream);
    case 160: return launch_gemm<160, EPI_LINEAR>(a1, a2, b, to, tr, p, stream);
    case 128: return launch_gemm<128, EPI_LINEAR>(a1, a2, b, to, tr, p, stream);
    case 64: return launch_gemm<64, EPI_LINEAR>(a1, a2, b, to, tr, p, stream);
    case 32: return launch_gemm<32, EPI_LINEAR>(a1, a2, b, to, tr, p, stream);
    default: return fail(AP_ERR_INVALID, "gemm: unsupported BLOCK_N %d", bn);
  }
}

static int make_weight_map(CUtensorMap* tm, const void* w, int N, long long K, int bn_box) {
  const uint64_t dims[2] = {(uint64_t)K, (uint64_t)N};
  const uint64_t strides[1] = {(uint64_t)K * 2};
  const uint32_t box[2] = {64, (uint32_t)bn_box};
  return encode_tmap(tm, w, 2, dims, strides, box, true);
}

// Validates and copies the optional epilogue extensions into the kernel parameters (after tma_epi / tile counts are known).
static int apply_ext(GemmParams& p, const ap_epilogue_ext* ext, int epi, long long m_pad, int k_ln) {
  p.bias_ld = p.N;
  static const int epi_double = getenv("AP_GEMM_EPI_DOUBLE") ? atoi(getenv("AP_GEMM_EPI_DOUBLE")) : 1;
  p.epi_double = epi_double;
  if (ext != nullptr && ext->bias_ld > 0) p.bias_ld = ext->bias_ld;
  // both epilogues read the bias as float4: every bias row must start on a 16-byte boundary
  if (p.bias != nullptr && ((reinterpret_cast<uintptr_t>(p.bias) & 15) != 0 || (p.bias_ld & 3) != 0))
    return fail(AP_ERR_INVALID, "gemm: bias must be 16-byte aligned with bias_ld %% 4 == 0 (bias_ld %lld)", p.bias_ld);
  if (ext == nullptr) return AP_OK;
  const bool any = ext->row_stat_out || ext->col_stat_out || ext->ln_rstd;
  if (!any) return AP_OK;
  if (!p.tma_epi) return fail(AP_ERR_INVALID, "gemm: epilogue statistics / LayerNorm folding need the TMA epilogue (aligned fp16 out)");
  // the partials sum what the epilogue computed, not what the clipped TMA store kept: only whole-width outputs
  if ((ext->row_stat_out || ext->col_stat_out) && p.n_valid < (epi == EPI_GEGLU ? p.N / 2 : p.N))
    return fail(AP_ERR_INVALID, "gemm: row / column statistics need n_valid (%d) == the output width", p.n_valid);
  if (ext->row_stat_out) {
    if (epi != EPI_LINEAR) return fail(AP_ERR_INVALID, "gemm: row statistics are not available with GEGLU");
    if (ext->row_stat_ld < m_pad) return fail(AP_ERR_INVALID, "gemm: row_stat_ld %lld < padded M %lld", ext->row_stat_ld, m_pad);
    if (p.a_mode != A_GEMM) return fail(AP_ERR_INVALID, "gemm: row statistics only for plain GEMMs");
    p.row_stat_out = (float2*)ext->row_stat_out;
    p.row_stat_ld = ext->row_stat_ld;
  }
  if (ext->col_stat_out) {
    if (epi != EPI_LINEAR) return fail(AP_ERR_INVALID, "gemm: column statistics are not available with GEGLU");
    if (ext->col_stat_ld < p.N || (ext->col_stat_ld & 1)) return fail(AP_ERR_INVALID, "gemm: bad col_stat_ld %lld", ext->col_stat_ld);
    if ((reinterpret_cast<uintptr_t>(ext->col_stat_out) & 15) != 0) return fail(AP_ERR_INVALID, "gemm: col_stat_out must be 16-byte aligned");
    if (p.a_mode != A_GEMM && p.sub_n != 1)
      return fail(AP_ERR_INVALID, "conv3x3: column statistics need Ho*Wo %% 32 == 0 with 32-row sub-boxes inside one frame");
    p.col_stat_out = (float2*)ext->col_stat_out;
    p.col_stat_ld = ext->col_stat_ld;
  }
  if (ext->ln_rstd) {
    if (p.a_mode != A_GEMM) return fail(AP_ERR_INVALID, "gemm: LayerNorm folding only for plain GEMMs");
    if (p.bias == nullptr) return fail(AP_ERR_INVALID, "gemm: LayerNorm folding needs the folded bias (beta.W^T + b)");
    p.ln_rstd = ext->ln_rstd;
  }
  return AP_OK;
}

}  // namespace ap

using namespace ap;

extern "C" int ap_gemm_row_stat_parts(long long M, int N, int K, int flags, int block_n) {
  const int epi = (flags & AP_GEMM_GEGLU) ? EPI_GEGLU : EPI_LINEAR;
  const int bn = pick_bn(N, block_n, (M + 127) / 128, epi == EPI_GEGLU);
  if (bn <= 0 || N % bn != 0) return fail(AP_ERR_INVALID, "gemm: N=%d not tileable (block_n=%d)", N, block_n);
  GemmParams p{};
  p.num_m_tiles = (int)((M + 127) / 128);
  p.num_n_tiles = N / bn;
  p.num_kb = (K + 63) / 64;
  p.tma_epi = 1;
  return p.num_n_tiles;
}

extern "C" int ap_gemm_f16(const void* a, long long lda, int K1, const void* a2, long long lda2, int K2,
                           const void* w, long long M, int N, const float* bias, long long bias_group_rows,
                           const void* residual, long long ldr, void* out, long long ldo, int n_valid, int flags,
                           int block_n, void* stream, const ap_epilogue_ext* ext) {
  AP_REQUIRE(a && w && out, "gemm: null pointer");
  AP_REQUIRE(M > 0 && N > 0 && K1 > 0, "gemm: bad shape M=%lld N=%d K1=%d", M, N, K1);
  AP_REQUIRE(K1 % 64 == 0 || (a2 == nullptr), "gemm: K1 must be a multiple of 64 when a second source follows");
  AP_REQUIRE((lda % 8) == 0 && (a2 == nullptr || (lda2 % 8) == 0), "gemm: lda must be a multiple of 8 elements");
  const int epi = (flags & AP_GEMM_GEGLU) ? EPI_GEGLU : EPI_LINEAR;
  const int bn = pick_bn(N, block_n, (M + 127) / 128, epi == EPI_GEGLU);
  AP_REQUIRE(epi != EPI_GEGLU || (bn > 0 && bn % 64 == 0), "gemm: GEGLU needs a BLOCK_N multiple of 64");
  AP_REQUIRE(bn > 0 && N % bn == 0, "gemm: N=%d not tileable (block_n=%d)", N, block_n);
  const long long K = (long long)K1 + (a2 ? K2 : 0);
  AP_REQUIRE((K * 2) % 16 == 0, "gemm: K*2 bytes must be a multiple of 16");

  GemmParams p{};
  p.M = (int)M;
  p.N = N;
  p.num_m_tiles = (int)((M + 127) / 128);
  p.num_n_tiles = N / bn;
  p.a_mode = A_GEMM;
  p.kb_src1 = (K1 + 63) / 64;
  p.kb_src2 = a2 ? (K2 + 63) / 64 : 0;
  p.num_kb = p.kb_src1 + p.kb_src2;
  p.bias = bias;
  p.bias_group_rows = (int)(bias_group_rows > 0 ? (bias_group_rows > 0x7fffffff ? 0x7fffffff : bias_group_rows)
                                                : 0x7fffffff);
  p.residual = (const __half*)residual;
  p.ldr = (int)ldr;
  p.out = (__half*)out;
  p.ldo = (int)ldo;
  const int nout = epi == EPI_GEGLU ? N / 2 : N;
  p.n_valid = n_valid > 0 ? n_valid : nout;
  p.out_f32 = (flags & AP_GEMM_OUT_F32) ? 1 : 0;
  AP_REQUIRE(!(p.out_f32 && epi == EPI_GEGLU), "gemm: fp32 output is not available with GEGLU");
  p.gelu = (flags & AP_GEMM_GELU) ? 1 : 0;
  AP_REQUIRE(!p.gelu || (epi == EPI_LINEAR && residual == nullptr && !(ext && ext->ln_rstd)),
             "gemm: GELU epilogue is not available with GEGLU, a residual or LayerNorm folding");
  p.quick_gelu = (flags & AP_GEMM_QUICK_GELU) ? 1 : 0;
  AP_REQUIRE(!(p.gelu && p.quick_gelu), "gemm: AP_GEMM_GELU and AP_GEMM_QUICK_GELU are mutually exclusive");
  AP_REQUIRE(!p.quick_gelu || (epi == EPI_LINEAR && residual == nullptr && !(ext && ext->ln_rstd)),
             "gemm: quick-GELU epilogue is not available with GEGLU, a residual or LayerNorm folding");

  CUtensorMap tmA1, tmA2, tmB;
  {
    const uint64_t dims[2] = {(uint64_t)K1, (uint64_t)M};
    const uint64_t strides[1] = {(uint64_t)lda * 2};
    const uint32_t box[2] = {64, 128};
    int rc = encode_tmap(&tmA1, a, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  if (a2) {
    const uint64_t dims[2] = {(uint64_t)K2, (uint64_t)M};
    const uint64_t strides[1] = {(uint64_t)lda2 * 2};
    const uint32_t box[2] = {64, 128};
    int rc = encode_tmap(&tmA2, a2, 2, dims, strides, box, true);
    if (rc) return rc;
  } else {
    tmA2 = tmA1;
  }
  int rc = make_weight_map(&tmB, w, N, K, bn);
  if (rc) return rc;
  // TMA epilogue whenever the output (and residual) satisfy TMA's 16-byte rules
  CUtensorMap tmOut = tmB, tmRes = tmB;
  p.out_al16 = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  p.res_al16 = (reinterpret_cast<uintptr_t>(residual) & 15) == 0;
  const bool aligned_out = p.out_al16 && (ldo % 8) == 0 && (p.n_valid % 8) == 0;
  const bool aligned_res = residual == nullptr || (p.res_al16 && (ldr % 8) == 0);
  static const bool no_tma_epi = getenv("AP_GEMM_NO_TMA_EPI") != nullptr;
  if (!p.out_f32 && aligned_out && aligned_res && !no_tma_epi) {
    const uint64_t dims[2] = {(uint64_t)p.n_valid, (uint64_t)M};
    const uint32_t box[2] = {32, 32};
    const uint64_t so[1] = {(uint64_t)ldo * 2};
    if ((rc = encode_tmap(&tmOut, out, 2, dims, so, box, false, 2, 64))) return rc;
    if (residual) {
      const uint64_t sr[1] = {(uint64_t)ldr * 2};
      if ((rc = encode_tmap(&tmRes, residual, 2, dims, sr, box, false, 2, 64))) return rc;
    }
    p.tma_epi = 1;
  }
  if ((rc = apply_ext(p, ext, epi, (long long)p.num_m_tiles * 128, K1))) return rc;
  return dispatch(bn, epi, tmA1, tmA2, tmB, tmOut, tmRes, p, (cudaStream_t)stream);
}

// 3x3 convolution, padding 1, stride 1 or 2, NHWC fp16, optional channel-concatenated second input.
extern "C" int ap_conv3x3_nhwc_f16(const void* x, int C1, const void* x2, int C2, int Nf, int H, int W, int stride,
                                   const void* w, int Cout, const float* bias, long long bias_group_rows,
                                   const void* residual, void* out, long long ldo, int n_valid, int block_n,
                                   void* stream, const ap_epilogue_ext* ext) {
  AP_REQUIRE(x && w && out, "conv3x3: null pointer");
  AP_REQUIRE(stride == 1 || stride == 2, "conv3x3: stride must be 1 or 2");
  AP_REQUIRE(C1 % 64 == 0 && (x2 == nullptr || C2 % 64 == 0), "conv3x3: channels must be multiples of 64 (pad)");
  AP_REQUIRE(stride == 1 || (H % 2 == 0 && W % 2 == 0), "conv3x3: stride 2 needs even H, W");
  const int Ho = H / stride, Wo = W / stride;
  const int bn_ = pick_bn(Cout, block_n, ((long long)Nf * Ho * Wo + 127) / 128);
  AP_REQUIRE(bn_ > 0 && Cout % bn_ == 0, "conv3x3: Cout=%d not tileable", Cout);

  // tile box: bw x bh x bn output pixels = 128 rows, bw | Wo, bh | Ho (powers of two)
  auto pow2_div = [](int v, int cap) { int d = 1; while (d * 2 <= cap && v % (d * 2) == 0) d *= 2; return d; };
  const int bw = pow2_div(Wo, 128);
  const int bh = pow2_div(Ho, 128 / bw);
  const int bnf = 128 / (bw * bh);

  GemmParams p{};
  p.Nf = Nf; p.Ho = Ho; p.Wo = Wo;
  p.bw = bw; p.bh = bh; p.bn = bnf;
  p.tiles_x = Wo / bw;
  p.tiles_y = Ho / bh;
  p.M = Nf * Ho * Wo;
  p.N = Cout;
  p.num_m_tiles = ((Nf + bnf - 1) / bnf) * p.tiles_x * p.tiles_y;
  p.num_n_tiles = Cout / bn_;
  p.a_mode = stride == 1 ? A_CONV_S1 : A_CONV_S2;
  p.kb_src1 = C1 / 64;
  p.kb_src2 = x2 ? C2 / 64 : 0;
  p.num_kb = 9 * (p.kb_src1 + p.kb_src2);
  p.C1 = C1;
  p.C2 = x2 ? C2 : 0;
  p.bias = bias;
  p.bias_group_rows = (int)(bias_group_rows > 0 ? (bias_group_rows > 0x7fffffff ? 0x7fffffff : bias_group_rows)
                                                : 0x7fffffff);
  p.residual = (const __half*)residual;
  p.ldr = (int)ldo;
  p.out = (__half*)out;
  p.ldo = (int)ldo;
  p.n_valid = n_valid > 0 ? n_valid : Cout;
  p.debug = getenv("AP_GEMM_DEBUG") ? atoi(getenv("AP_GEMM_DEBUG")) : 0;

  auto make_act_map = [&](CUtensorMap* tm, const void* base, int C) -> int {
    if (stride == 1) {
      const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)Nf};
      const uint64_t strides[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
      const uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bnf};
      return encode_tmap(tm, base, 4, dims, strides, box, true);
    }
    // (phase_x * C + c, W/2, phase_y, H/2, Nf)
    const uint64_t dims[5] = {(uint64_t)2 * C, (uint64_t)W / 2, 2, (uint64_t)H / 2, (uint64_t)Nf};
    const uint64_t strides[4] = {(uint64_t)2 * C * 2, (uint64_t)W * C * 2, (uint64_t)2 * W * C * 2,
                                 (uint64_t)H * W * C * 2};
    const uint32_t box[5] = {64, (uint32_t)bw, 1, (uint32_t)bh, (uint32_t)bnf};
    return encode_tmap(tm, base, 5, dims, strides, box, true);
  };
  CUtensorMap tmA1, tmA2, tmB;
  int rc = make_act_map(&tmA1, x, C1);
  if (rc) return rc;
  if (x2) {
    rc = make_act_map(&tmA2, x2, C2);
    if (rc) return rc;
  } else {
    tmA2 = tmA1;
  }
  rc = make_weight_map(&tmB, w, Cout, 9ll * (C1 + (x2 ? C2 : 0)), bn_);
  if (rc) return rc;
  CUtensorMap tmOut = tmB, tmRes = tmB;
  p.out_al16 = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  p.res_al16 = (reinterpret_cast<uintptr_t>(residual) & 15) == 0;
  const bool aligned_out = p.out_al16 && (ldo % 8) == 0 && (p.n_valid % 8) == 0;
  const bool aligned_res = residual == nullptr || p.res_al16;
  static const bool no_tma_epi = getenv("AP_GEMM_NO_TMA_EPI") != nullptr;
  if (aligned_out && aligned_res && !no_tma_epi) {
    p.sub_w = bw < 32 ? bw : 32;
    p.sub_h = bh < 32 / p.sub_w ? bh : 32 / p.sub_w;
    p.sub_n = 32 / (p.sub_w * p.sub_h);
    const uint64_t dims[4] = {(uint64_t)p.n_valid, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)Nf};
    const uint64_t so[3] = {(uint64_t)ldo * 2, (uint64_t)Wo * ldo * 2, (uint64_t)Ho * Wo * ldo * 2};
    const uint32_t box[4] = {32, (uint32_t)p.sub_w, (uint32_t)p.sub_h, (uint32_t)p.sub_n};
    if ((rc = encode_tmap(&tmOut, out, 4, dims, so, box, false, 2, 64))) return rc;
    if (residual && (rc = encode_tmap(&tmRes, residual, 4, dims, so, box, false, 2, 64))) return rc;
    p.tma_epi = 1;
  }
  if ((rc = apply_ext(p, ext, EPI_LINEAR, (long long)p.num_m_tiles * 128, 0))) return rc;
  // entry e of the partials must belong to frame e / (Ho*Wo/32): tiles inside one frame, or whole frames per tile
  if (p.col_stat_out)
    AP_REQUIRE((Ho * Wo) % 32 == 0 && (p.bn == 1 || p.tiles_x * p.tiles_y == 1),
               "conv3x3: column statistics need Ho*Wo %% 32 == 0 and frame-major 32-row sub-boxes (Ho=%d Wo=%d)", Ho, Wo);
  return dispatch(bn_, EPI_LINEAR, tmA1, tmA2, tmB, tmOut, tmRes, p, (cudaStream_t)stream);
}
