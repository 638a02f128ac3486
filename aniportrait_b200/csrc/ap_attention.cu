// Fused spatial self / reference attention for sm_90a (flash-style, wgmma + TMA).
//
//   O[f, h] = softmax( Q[f,h] . [K_own[f,h] ; K_bank[h]]^T * scale ) . [V_own[f,h] ; V_bank[h]]
//
// One launch covers every frame of a UNet call: frames before `first_bank_frame` (the unconditional CFG branch)
// attend to their own N tokens only, the others to 2N keys (own tokens followed by the ReferenceNet bank, whose K/V
// were projected once per video and are read in place: no `bank.repeat(F)` / `torch.cat` copy, no discarded
// reference-attention for the unconditional half, no CPU-mask scatter).
//
// Replaces diffusers Attention/AttnProcessor2_0 -> F.scaled_dot_product_attention as driven by the patched block
// forward of ReferenceAttentionControl (reference src/models/mutual_self_attention.py:147-186; plain blocks
// src/models/attention.py:323-330, write mode :137-146; PoseGuider's self-attention src/models/pose_guider.py:86-89).
//
// Persistent CTAs over (frame, head, 128-query tile) work units; three warpgroups:
//   warpgroup 0     TMA producer: Q tile once per unit, K/V tiles through an mbarrier ring (own rows, then bank rows)
//   warpgroups 1-2  64 query rows each: S = Q.K^T (wgmma, both operands in shared memory, S in registers), base-2
//                   online softmax in registers, O += P.V (wgmma with P as the register A operand, V MN-major in shared
//                   memory, O in registers), then O / l -> fp16 -> global
// Head dim d is zero-padded to DPAD in {64,128,192} by the QKV projection (padded weight rows), so every operand slab
// is a clean 64-column / 128-byte swizzle atom.
#include <stdio.h>
#include <stdlib.h>

#include "ap_host.h"
#include "ap_ptx.cuh"
#include "ap_wgmma.cuh"

namespace ap {

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct AttnParams {
  int n_frames, tokens, heads, head_dim;
  int bank_tokens;        // 0 = no bank
  int first_bank_frame;   // frames >= this attend to the bank as well
  int frames_per_bank;    // bank index = (frame - first_bank_frame) / frames_per_bank
  int m_tiles;            // ceil(tokens / 128)
  int num_units;          // n_frames * heads * m_tiles
  float scale_log2;       // softmax scale * log2(e)
  __half* out;
  long long ldo;
};

template <int DPAD, int BN>
struct AttnCfg {
  static constexpr int SLABS = DPAD / 64;
  static constexpr int Q_BYTES = 128 * DPAD * 2;
  static constexpr int K_BYTES = BN * DPAD * 2;
  static constexpr int KV_STAGE = 2 * K_BYTES;
  static constexpr int BUDGET = 227 * 1024 - 1024 - 256 - Q_BYTES;
  static constexpr int STAGES_RAW = BUDGET / KV_STAGE;
  static constexpr int STAGES = STAGES_RAW > 4 ? 4 : STAGES_RAW;
  static constexpr int SMEM_BYTES = Q_BYTES + STAGES * KV_STAGE + 1024 + 256;
  static_assert(STAGES >= 2, "need at least a double-buffered K/V ring");
  static_assert(DPAD % 64 == 0 && DPAD <= 192 && (BN == 64 || BN == 128), "tile config");
};

template <int DPAD, int BN>
__global__ void __launch_bounds__(384, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmBK,
                 const __grid_constant__ CUtensorMap tmBV, const AttnParams p) {
  using Cfg = AttnCfg<DPAD, BN>;
  constexpr int ST = Cfg::STAGES;
  griddep_launch_dependents();   // PDL (ap_host.h::launch_pdl)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_kv = smem_q + Cfg::Q_BYTES;  // stage s: K at s*KV_STAGE, V at s*KV_STAGE + K_BYTES
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_kv + ST * Cfg::KV_STAGE);
  uint64_t* q_full = bars + 0;
  uint64_t* q_empty = bars + 1;
  uint64_t* k_full = bars + 2;            // [ST]
  uint64_t* v_full = k_full + ST;         // [ST]
  uint64_t* kv_empty = v_full + ST;       // [ST]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 8);   // one arrival per consumer warp
    for (int s = 0; s < ST; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&kv_empty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  griddep_wait();   // PDL: Q/K/V come from the previous kernel

  const int own_tiles = (p.tokens + BN - 1) / BN;
  const int bank_tiles = (p.bank_tokens + BN - 1) / BN;
  const int units_per_frame = p.heads * p.m_tiles;

  // unit -> (frame, head, m_tile); frames with a bank (the heavy ones) are scheduled first
  auto decode = [&](int unit, int& frame, int& head, int& m_tile, int& T) {
    const int fk = unit / units_per_frame;
    const int rem = unit % units_per_frame;
    frame = (fk + p.first_bank_frame) % p.n_frames;
    head = rem / p.m_tiles;
    m_tile = rem % p.m_tiles;
    const bool has_bank = p.bank_tokens > 0 && frame >= p.first_bank_frame;
    T = own_tiles + (has_bank ? bank_tiles : 0);
  };

  if (warp < 4) {
    // ---------------------------------------------------------------------------- TMA producer
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      uint32_t g = 0;   // global K/V tile counter
      uint32_t uc = 0;  // unit counter
      for (int unit = blockIdx.x; unit < p.num_units; unit += gridDim.x, ++uc) {
        int frame, head, m_tile, T;
        decode(unit, frame, head, m_tile, T);
        mbar_wait_quiet(q_empty, (uc & 1) ^ 1);
        mbar_arrive_expect_tx(q_full, Cfg::Q_BYTES);
#pragma unroll
        for (int s = 0; s < Cfg::SLABS; ++s)
          tma_load_2d(&tmQ, q_full, smem_q + s * (128 * 128), head * DPAD + s * 64, frame * p.tokens + m_tile * 128);
        const int bank_idx = (frame - p.first_bank_frame) / p.frames_per_bank;
        for (int j = 0; j < T; ++j, ++g) {
          const int stage = g % ST;
          const uint32_t ph = (g / ST) & 1;
          mbar_wait_quiet(&kv_empty[stage], ph ^ 1);
          const bool own = j < own_tiles;
          const CUtensorMap* mk = own ? &tmK : &tmBK;
          const CUtensorMap* mv = own ? &tmV : &tmBV;
          const int row = own ? frame * p.tokens + j * BN : bank_idx * p.bank_tokens + (j - own_tiles) * BN;
          uint8_t* kd = smem_kv + stage * Cfg::KV_STAGE;
          uint8_t* vd = kd + Cfg::K_BYTES;
          mbar_arrive_expect_tx(&k_full[stage], Cfg::K_BYTES);
#pragma unroll
          for (int s = 0; s < Cfg::SLABS; ++s)
            tma_load_2d(mk, &k_full[stage], kd + s * (BN * 128), head * DPAD + s * 64, row);
          mbar_arrive_expect_tx(&v_full[stage], Cfg::K_BYTES);
#pragma unroll
          for (int s = 0; s < Cfg::SLABS; ++s)
            tma_load_2d(mv, &v_full[stage], vd + s * (BN * 128), head * DPAD + s * 64, row);
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------------------ consumers
  setmaxnreg_inc<232>();
  const int wg = (warp >> 2) - 1;   // query rows [64 wg, +64) of the unit's tile
  const int wq = warp & 3;          // this warp's accumulator rows: 16 wq + lane / 4 and + 8
  const int qd = lane & 3;          // accumulator columns 8 i + 2 qd, + 1
  const uint32_t q_base = smem_u32(smem_q) + wg * (64 * 128);
  uint32_t g = 0, uc = 0;
  for (int unit = blockIdx.x; unit < p.num_units; unit += gridDim.x, ++uc) {
    int frame, head, m_tile, T;
    decode(unit, frame, head, m_tile, T);
    float o[DPAD / 2];
#pragma unroll
    for (int i = 0; i < DPAD / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    mbar_wait_quiet(q_full, uc & 1);
    for (int j = 0; j < T; ++j, ++g) {
      const int stage = g % ST;
      const uint32_t ph = (g / ST) & 1;
      const uint32_t k_addr = smem_u32(smem_kv + stage * Cfg::KV_STAGE);
      const uint32_t v_addr = k_addr + Cfg::K_BYTES;
      // S = Q . K^T
      float s[BN / 2];
      mbar_wait_quiet(&k_full[stage], ph);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < DPAD / 16; ++kk)
        wgmma_ss<BN>(s, wgmma_desc_k_sw128(q_base + (kk / 4) * (128 * 128) + (kk % 4) * 32),
                     wgmma_desc_k_sw128(k_addr + (kk / 4) * (BN * 128) + (kk % 4) * 32), kk != 0);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence<BN / 2>(s);
      if (j == T - 1) {   // the last read of this unit's Q tile
        __syncwarp();
        if (lane == 0) mbar_arrive(q_empty);
      }

      // keys past the end of the own / bank sequence
      const bool own = j < own_tiles;
      const int jj = own ? j : j - own_tiles;
      const int ntok = own ? p.tokens : p.bank_tokens;
      const int valid = min(BN, ntok - jj * BN);
      if (valid != BN) {
#pragma unroll
        for (int i = 0; i < BN / 8; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (8 * i + 2 * qd + e >= valid) {
              s[4 * i + e] = -INFINITY;
              s[4 * i + 2 + e] = -INFINITY;
            }
      }
      // online softmax (base 2) over the two rows of this thread; a row is spread over the 4 threads of a quad
      float mx[2] = {s[0], s[2]};
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        mx[0] = fmaxf(mx[0], fmaxf(s[4 * i], s[4 * i + 1]));
        mx[1] = fmaxf(mx[1], fmaxf(s[4 * i + 2], s[4 * i + 3]));
      }
      float alpha[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float m_new = fmaxf(m_run[r], mx[r] * p.scale_log2);
        alpha[r] = fast_exp2(m_run[r] - m_new);
        m_run[r] = m_new;
        l_run[r] *= alpha[r];
      }
#pragma unroll
      for (int i = 0; i < DPAD / 8; ++i) {
        o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
        o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
      }
      // P = exp2(S*c - m) as fp16 pairs, laid out as the A fragments of the P.V wgmma (k16 step kk = columns 16kk..+16)
      uint32_t pk[BN / 4];
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const float p0 = fast_exp2(fmaf(s[4 * i], p.scale_log2, -m_run[0]));
        const float p1 = fast_exp2(fmaf(s[4 * i + 1], p.scale_log2, -m_run[0]));
        const float p2 = fast_exp2(fmaf(s[4 * i + 2], p.scale_log2, -m_run[1]));
        const float p3 = fast_exp2(fmaf(s[4 * i + 3], p.scale_log2, -m_run[1]));
        l_run[0] += p0 + p1;
        l_run[1] += p2 + p3;
        const __half2 h01 = __floats2half2_rn(p0, p1), h23 = __floats2half2_rn(p2, p3);
        pk[2 * i] = *reinterpret_cast<const uint32_t*>(&h01);
        pk[2 * i + 1] = *reinterpret_cast<const uint32_t*>(&h23);
      }
      // O += P . V
      mbar_wait_quiet(&v_full[stage], ph);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk)
        wgmma_rs_tb<DPAD>(o, pk + 4 * kk, wgmma_desc_mn_sw128(v_addr + kk * (16 * 128), BN * 128), 1);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence<DPAD / 2>(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[stage]);
    }
    // ------------------------------------------------------------------ epilogue: O / l -> fp16 -> global
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float inv_l = 1.f / l_run[r];
      const int q_idx = m_tile * 128 + wg * 64 + wq * 16 + (lane >> 2) + 8 * r;
      if (q_idx < p.tokens) {
        __half* dst = p.out + ((long long)frame * p.tokens + q_idx) * p.ldo + head * p.head_dim;
#pragma unroll
        for (int i = 0; i < DPAD / 8; ++i)
          if (8 * i + 2 * qd < p.head_dim)
            *reinterpret_cast<__half2*>(dst + 8 * i + 2 * qd) =
                __floats2half2_rn(o[4 * i + 2 * r] * inv_l, o[4 * i + 2 * r + 1] * inv_l);
      }
    }
  }
}

template <int DPAD, int BN>
static int launch_attention(const CUtensorMap* maps, const AttnParams& p, cudaStream_t stream) {
  using Cfg = AttnCfg<DPAD, BN>;
  static bool attr_set = false;
  if (!attr_set) {
    AP_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel<DPAD, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       Cfg::SMEM_BYTES));
    attr_set = true;
  }
  const int grid = p.num_units < num_sms() ? p.num_units : num_sms();
  AP_LAUNCH((attention_kernel<DPAD, BN>), grid, 384, Cfg::SMEM_BYTES, stream, maps[0], maps[1], maps[2], maps[3], maps[4], p);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

}  // namespace ap

using namespace ap;

extern "C" int ap_attention_f16(const void* q, const void* k, const void* v, long long ld_qkv, const void* bank_k,
                                const void* bank_v, long long ld_bank, int bank_tokens, int n_banks, int n_frames,
                                int tokens, int heads, int head_dim, int dpad, int first_bank_frame,
                                int frames_per_bank, float scale, void* out, long long ldo, void* stream) {
  AP_REQUIRE(q && k && v && out, "attention: null pointer");
  AP_REQUIRE(dpad == 64 || dpad == 128 || dpad == 192, "attention: dpad must be 64/128/192 (got %d)", dpad);
  AP_REQUIRE(head_dim % 8 == 0 && head_dim <= dpad, "attention: head_dim %d must be a multiple of 8 and <= dpad", head_dim);
  AP_REQUIRE(ld_qkv % 8 == 0 && ldo % 8 == 0, "attention: leading dims must be multiples of 8 elements");
  // the epilogue stores __half2 pairs; q/k/v and the bank are checked by encode_tmap (16 B)
  AP_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0, "attention: out must be 4-byte aligned");
  AP_REQUIRE(n_frames > 0 && tokens > 0 && heads > 0, "attention: bad shape");
  const bool has_bank = bank_k != nullptr && bank_tokens > 0;
  AP_REQUIRE(!has_bank || (bank_v && frames_per_bank > 0 && first_bank_frame >= 0 && n_banks > 0),
             "attention: bad bank arguments");
  // 128-key tiles; 64 for dpad = 192, where 128 would leave room for only one K/V stage
  const int bn = dpad == 192 ? 64 : 128;
  AttnParams p{};
  p.n_frames = n_frames;
  p.tokens = tokens;
  p.heads = heads;
  p.head_dim = head_dim;
  p.bank_tokens = has_bank ? bank_tokens : 0;
  p.first_bank_frame = has_bank ? first_bank_frame : 0;
  p.frames_per_bank = has_bank ? frames_per_bank : 1;
  p.m_tiles = (tokens + 127) / 128;
  p.num_units = n_frames * heads * p.m_tiles;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = (__half*)out;
  p.ldo = ldo;
  if (has_bank) {
    const int max_bank = (n_frames - 1 - first_bank_frame) / frames_per_bank;
    AP_REQUIRE(first_bank_frame >= n_frames || max_bank < n_banks, "attention: bank index out of range");
  }

  CUtensorMap maps[5];
  const uint64_t cols = (uint64_t)heads * dpad;
  auto mk = [&](CUtensorMap* tm, const void* base, uint64_t rows, long long ld, uint32_t box_rows) -> int {
    const uint64_t dims[2] = {cols, rows};
    const uint64_t strides[1] = {(uint64_t)ld * 2};
    const uint32_t box[2] = {64, box_rows};
    return encode_tmap(tm, base, 2, dims, strides, box, true);
  };
  int rc;
  const uint64_t rows = (uint64_t)n_frames * tokens;
  if ((rc = mk(&maps[0], q, rows, ld_qkv, 128))) return rc;
  if ((rc = mk(&maps[1], k, rows, ld_qkv, bn))) return rc;
  if ((rc = mk(&maps[2], v, rows, ld_qkv, bn))) return rc;
  if (has_bank) {
    const uint64_t brows = (uint64_t)n_banks * bank_tokens;
    if ((rc = mk(&maps[3], bank_k, brows, ld_bank, bn))) return rc;
    if ((rc = mk(&maps[4], bank_v, brows, ld_bank, bn))) return rc;
  } else {
    maps[3] = maps[1];
    maps[4] = maps[2];
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (dpad == 64) return launch_attention<64, 128>(maps, p, st);
  if (dpad == 128) return launch_attention<128, 128>(maps, p, st);
  return launch_attention<192, 64>(maps, p, st);
}
