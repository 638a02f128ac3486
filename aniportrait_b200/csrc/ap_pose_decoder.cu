// The autoregressive head-pose decoder of Audio2PoseModel.infer (reference src/audio_models/pose_model.py:97-124, in its
// incremental form aniportrait_b200/audio_models/pose_infer.py): all T steps of one chunk in ONE launch.
//
// One step is a chain of matrix-vector products (M = 1) through `layers` post-norm nn.TransformerDecoderLayers at E = 512,
// 8 heads of 64, FFN 1024, ReLU. 16.8 M fp16 weights for 8 layers (33.6 MB) stay in L2, so a step is bounded by how fast
// the SMs can pull them from L2 and by the dependency chain between the matrix-vector products, not by FLOPs.
//
// Grid = one thread-block cluster of NC CTAs (16, or 8 where 16 cannot be co-scheduled), 512 threads each. Every CTA owns
// a fixed slice of output rows of every matrix and keeps its own copy of the 512-vector x. Per layer:
//   A  its in_proj rows; each q/k/v value is stored into the shared memory of the CTA that owns its head (DSMEM)
//   B  CTA h < 8: appends k/v to the fp16 cache at row i, attention of one query over rows 0..i with mask[h, i, :]
//      (the module's own causal + ALiBi row), the 64 outputs broadcast to every CTA; the other CTAs idle
//   C  its out_proj rows + bias + residual, broadcast
//   D  every CTA redundantly: LN1, + cross[l, i], LN2 (a block reduction costs less than another cluster barrier);
//      then its linear1 rows + ReLU, broadcast
//   E  its linear2 rows + bias + residual, broadcast; LN3 runs redundantly at the start of the next layer
// Phases are separated by the cluster barrier (barrier.cluster.arrive.release / wait.acquire): 5 per layer. Every buffer a
// phase writes remotely is read in the next phase only and written again after at least one more barrier, so one barrier
// between phases covers both the read-after-write and the write-after-read order. The pose head (pose_map_r), the output
// row and the next token (pose_map) are computed redundantly by every CTA, with no extra barrier.
//
// Nothing a step reads from global memory on its critical path except the KV cache: the weights do not depend on
// activations and stream from L2 into a shared-memory ring with cp.async.bulk, ahead of the phase that uses them (see
// PoseStream); the per-layer biases, LayerNorm parameters and the cross row arrive the same way one layer ahead. A step
// then costs about the larger of the weight stream and the chain of barriers, LayerNorms and attention, not their sum.
//
// Numerics: fp16 weights and KV cache; everything else fp32 (activations, accumulation, LayerNorm statistics, softmax,
// biases, cross, pe, mask, pose head, output). Every reduction has a fixed order and there are no atomics: two calls give
// identical bytes.
#include <cstdlib>
#include <cstring>

#include "ap_host.h"
#include "ap_ptx.cuh"

namespace ap {

constexpr int PD_E = 512, PD_HEADS = 8, PD_D = 64, PD_FF = 1024, PD_QKV = 3 * PD_E;
constexpr int PD_THREADS = 512, PD_WARPS = PD_THREADS / 32;
constexpr int PD_MAX_T = 1024;     // score buffer of the attention phase
constexpr int PD_PV_GROUPS = PD_THREADS / 8;   // attention P.V: 8 threads per key (one uint4 of 8 dims each)
static_assert(PD_E == PD_THREADS, "one thread per element of the 512-vector");
static_assert(PD_MAX_T == 2 * PD_THREADS, "the score pass gives every thread at most two keys");

// ----------------------------------------------------------------------------------------------
// cluster primitives
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// shared::cluster address of `p` (a shared variable of this CTA) in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t dsmem_addr(const void* p, uint32_t rank) {
  uint32_t out;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(out) : "r"(smem_u32(p)), "r"(rank));
  return out;
}
__device__ __forceinline__ void dsmem_st(uint32_t addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ float dot8(uint4 w, const float* x) {   // x: 8 consecutive fp32 in shared memory
  const __half2* h = reinterpret_cast<const __half2*>(&w);
  const float4 x0 = *reinterpret_cast<const float4*>(x), x1 = *reinterpret_cast<const float4*>(x + 4);
  float2 a = __half22float2(h[0]), b = __half22float2(h[1]), c = __half22float2(h[2]), d = __half22float2(h[3]);
  float s = a.x * x0.x;
  s = fmaf(a.y, x0.y, s);
  s = fmaf(b.x, x0.z, s);
  s = fmaf(b.y, x0.w, s);
  s = fmaf(c.x, x1.x, s);
  s = fmaf(c.y, x1.y, s);
  s = fmaf(d.x, x1.z, s);
  s = fmaf(d.y, x1.w, s);
  return s;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Sum / max over the CTA; every thread gets the result. `red`: 2 x PD_WARPS floats of shared scratch, used alternately
// (the flip is CTA-uniform), so the barrier of one reduction also retires the previous reduction's reads and no second
// barrier is needed. The 16 warp partials are combined by a fixed butterfly and lane 0's value is broadcast: fixed order,
// the same bits in every thread.
struct BlockReduce {
  float* red;
  int flip = 0;
  template <bool kMax>
  __device__ __forceinline__ float run(float v) {
    v = kMax ? warp_max(v) : warp_sum(v);
    float* r = red + flip * PD_WARPS;
    flip ^= 1;
    if ((threadIdx.x & 31) == 0) r[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = r[threadIdx.x & (PD_WARPS - 1)];
#pragma unroll
    for (int o = PD_WARPS / 2; o > 0; o >>= 1) {
      const float t = __shfl_xor_sync(0xffffffffu, s, o);
      s = kMax ? fmaxf(s, t) : s + t;
    }
    return __shfl_sync(0xffffffffu, s, 0);
  }
  __device__ __forceinline__ float sum(float v) { return run<false>(v); }
  __device__ __forceinline__ float max(float v) { return run<true>(v); }
};
static_assert(PD_WARPS == 16, "BlockReduce's butterfly spans 16 warp partials");

// LayerNorm of one element per thread over the 512-vector (biased variance, two passes). g, b: shared memory.
__device__ __forceinline__ float layer_norm(float v, const float* g, const float* b, float eps, BlockReduce& br) {
  const float mean = br.sum(v) * (1.f / PD_E);
  const float c = v - mean;
  const float var = br.sum(c * c) * (1.f / PD_E);
  return c * rsqrtf(var + eps) * g[threadIdx.x] + b[threadIdx.x];
}

// ----------------------------------------------------------------------------------------------
// Weight stream. A CTA's slice of each matrix is a contiguous run of rows in global memory (96 | 32 | 64 | 32 KB of
// in_proj | out_proj | linear1 | linear2 per layer with 16 CTAs, twice that with 8), cut into 32 KB chunks. Thread 0 keeps
// PD_SLOTS chunks in flight into a shared-memory ring with cp.async.bulk, each completing on its slot's mbarrier; the chunk
// sequence runs through layers and steps without regard to phases, so the copies for the next phase and layer proceed
// while the CTA waits at cluster barriers. After the CTA has consumed a chunk (a __syncthreads), thread 0 issues the chunk
// PD_SLOTS further on into the freed slot. Bulk copies go through the copy engine rather than the load path of the SM,
// which is what lets one SM keep enough bytes in flight to stream from L2 at a useful rate.
// ----------------------------------------------------------------------------------------------
constexpr int PD_CHUNK = 32768;   // bytes per chunk = the transaction count of a slot's mbarrier
constexpr int PD_SLOTS = 5;
static_assert(PD_CHUNK % 16 == 0, "cp.async.bulk sizes are multiples of 16 bytes");

__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

template <int NC>
struct PoseShape {
  // chunks per layer of each matrix slice, in consumption order A (in_proj), C (out_proj), D (linear1), E (linear2)
  static constexpr int NA = PD_QKV / NC * PD_E * 2 / PD_CHUNK, NCo = PD_E / NC * PD_E * 2 / PD_CHUNK;
  static constexpr int ND = PD_FF / NC * PD_E * 2 / PD_CHUNK, NE = PD_E / NC * PD_FF * 2 / PD_CHUNK;
  static constexpr int CPL = NA + NCo + ND + NE;
  static_assert(NA * PD_CHUNK == PD_QKV / NC * PD_E * 2 && NCo * PD_CHUNK == PD_E / NC * PD_E * 2 &&
                    ND * PD_CHUNK == PD_FF / NC * PD_E * 2 && NE * PD_CHUNK == PD_E / NC * PD_FF * 2,
                "every slice is a whole number of chunks");
  // per-layer parameter block (floats): LayerNorm 1..3 weight and bias [6][512] | this CTA's bias slices of in_proj,
  // out_proj, linear1, linear2 | the cross row of (step, layer)
  static constexpr int BQ = PD_QKV / NC, BO = PD_E / NC, B1 = PD_FF / NC, B2 = PD_E / NC;
  static constexpr int P_LN = 0, P_BQ = 6 * PD_E, P_BO = P_BQ + BQ, P_B1 = P_BO + BO, P_B2 = P_B1 + B1, P_CR = P_B2 + B2;
  static constexpr int PFLOATS = P_CR + PD_E;
  static constexpr uint32_t PBYTES = PFLOATS * 4;   // the transaction count of a parameter block's mbarrier
  static_assert(BQ % 4 == 0 && BO % 4 == 0 && B1 % 4 == 0 && B2 % 4 == 0, "16-byte bulk copies");
  static_assert(AP_POSE_LN1_G + 6 * PD_E == AP_POSE_VEC && AP_POSE_LN1_B == AP_POSE_LN1_G + PD_E &&
                    AP_POSE_LN2_G == AP_POSE_LN1_G + 2 * PD_E && AP_POSE_LN3_B == AP_POSE_LN1_G + 5 * PD_E,
                "the three LayerNorms are one contiguous run at the end of the per-layer vector");
  static constexpr size_t SMEM = (size_t)PD_SLOTS * PD_CHUNK + 2 * (size_t)PBYTES;
};

template <int NC>
struct PoseStream {
  using S = PoseShape<NC>;
  const ap_pose_decoder_params* p;
  int rank;
  long long total;   // chunks in the whole call: T * layers * CPL

  // source of chunk q: layer (q / CPL) % layers, piece q % CPL
  __device__ __forceinline__ const void* chunk_src(long long q) const {
    const int l = (int)((q / S::CPL) % p->layers);
    int k = (int)(q % S::CPL);
    const __half* base;
    size_t slice;   // byte offset of this CTA's slice in the matrix of layer l
    if (k < S::NA) {
      base = reinterpret_cast<const __half*>(p->w_qkv);
      slice = ((size_t)l * PD_QKV + (size_t)rank * (PD_QKV / NC)) * PD_E * 2;
    } else if ((k -= S::NA) < S::NCo) {
      base = reinterpret_cast<const __half*>(p->w_out);
      slice = ((size_t)l * PD_E + (size_t)rank * (PD_E / NC)) * PD_E * 2;
    } else if ((k -= S::NCo) < S::ND) {
      base = reinterpret_cast<const __half*>(p->w_ff1);
      slice = ((size_t)l * PD_FF + (size_t)rank * (PD_FF / NC)) * PD_E * 2;
    } else {
      k -= S::ND;
      base = reinterpret_cast<const __half*>(p->w_ff2);
      slice = ((size_t)l * PD_E + (size_t)rank * (PD_E / NC)) * PD_FF * 2;
    }
    return reinterpret_cast<const char*>(base) + slice + (size_t)k * PD_CHUNK;
  }
  __device__ __forceinline__ void issue(long long q, char* ring, uint64_t* full) const {
    if (q >= total) return;
    const int slot = (int)(q % PD_SLOTS);
    mbar_arrive_expect_tx(&full[slot], PD_CHUNK);
    bulk_g2s(ring + (size_t)slot * PD_CHUNK, chunk_src(q), PD_CHUNK, &full[slot]);
  }
  // parameter block of global layer index g = step * layers + layer into buffer g & 1
  __device__ __forceinline__ void issue_params(long long g, float* pbuf, uint64_t* pbar, int T) const {
    if (g >= (long long)T * p->layers) return;
    const int l = (int)(g % p->layers);
    float* dst = pbuf + (g & 1) * S::PFLOATS;
    uint64_t* bar = &pbar[g & 1];
    const float* v = p->vec + (size_t)l * AP_POSE_VEC;
    mbar_arrive_expect_tx(bar, S::PBYTES);
    bulk_g2s(dst + S::P_LN, v + AP_POSE_LN1_G, 6 * PD_E * 4, bar);
    bulk_g2s(dst + S::P_BQ, v + AP_POSE_B_QKV + rank * S::BQ, S::BQ * 4, bar);
    bulk_g2s(dst + S::P_BO, v + AP_POSE_B_OUT + rank * S::BO, S::BO * 4, bar);
    bulk_g2s(dst + S::P_B1, v + AP_POSE_B_FF1 + rank * S::B1, S::B1 * 4, bar);
    bulk_g2s(dst + S::P_B2, v + AP_POSE_B_FF2 + rank * S::B2, S::B2 * 4, bar);
    bulk_g2s(dst + S::P_CR, p->cross + (size_t)g * PD_E, PD_E * 4, bar);   // cross [T, layers, 512]: row g
  }
};

// ----------------------------------------------------------------------------------------------
// Matrix-vector products over the chunks of one phase: a chunk holds RCH rows of K fp16; warp w takes RPW consecutive
// rows, lane l reads uint4 (8 weights) number l + 32 u, u < K / 256, of each (conflict-free 512-byte runs).
// emit(local row of the CTA's slice, row . x); every lane holds the sum. x: fp32 [K] in shared memory.
// ----------------------------------------------------------------------------------------------
template <int K, int NCHUNK, int NC, typename Emit>
__device__ __forceinline__ void gemv_phase(const float* x, char* ring, uint64_t* full, long long& q,
                                           const PoseStream<NC>& st, Emit emit) {
  constexpr int RCH = PD_CHUNK / (K * 2), RPW = RCH / PD_WARPS, U = K / 256;
  static_assert(RPW * PD_WARPS == RCH && K % 256 == 0, "chunk rows split evenly over the warps");
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float xr[U * 8];
#pragma unroll
  for (int u = 0; u < U; ++u)
#pragma unroll
    for (int e = 0; e < 8; ++e) xr[u * 8 + e] = x[(lane + 32 * u) * 8 + e];
#pragma unroll 1
  for (int c = 0; c < NCHUNK; ++c, ++q) {
    const int slot = (int)(q % PD_SLOTS);
    mbar_wait(&full[slot], (uint32_t)((q / PD_SLOTS) & 1));
    const uint4* w = reinterpret_cast<const uint4*>(ring + (size_t)slot * PD_CHUNK) + (size_t)warp * RPW * (K / 8);
#pragma unroll
    for (int j = 0; j < RPW; ++j) {
      float s = 0.f;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint4 wv = w[j * (K / 8) + lane + 32 * u];
        const __half2* h = reinterpret_cast<const __half2*>(&wv);
        float d = 0.f;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(h[e]);
          d = fmaf(f.x, xr[u * 8 + 2 * e], d);
          d = fmaf(f.y, xr[u * 8 + 2 * e + 1], d);
        }
        s += d;
      }
      emit(c * RCH + warp * RPW + j, warp_sum(s));
    }
    __syncthreads();   // the slot is consumed: refill it with the chunk PD_SLOTS further on
    if (threadIdx.x == 0) st.issue(q + PD_SLOTS, ring, full);
  }
}

struct PoseArgs {
  ap_pose_decoder_params p;
  int T;
  float* out;
  __half* kv;
  float* trace;   // pose_decoder_kernel<NC, true> only: fp32 [T, PD_TRACE_STAGES * layers + 1, 512]
};

// With TRACE, the kernel stores the input of every stage of every layer, so that a test can check each stage on its own
// inputs: row (i, 5 l + k) of step i, layer l holds k = 0 the layer input x, 1 q, 2 the attention output of all heads,
// 3 the LN2 output (linear1's input), 4 linear2 + bias + residual (LN3's input); row (i, 5 layers) the pose head's input.
// The vectors are identical in every CTA, so CTA 0 stores them; q lives in the head owner's CTA (h < 8), which stores
// its 64 entries. `if constexpr` keeps the production instantiations free of it: the 16-CTA kernel sits at the
// 128-register cap.
constexpr int PD_TRACE_STAGES = 5;
template <bool TRACE>
__device__ __forceinline__ void trace_store(const PoseArgs& a, bool who, int i, int row, int e, float v) {
  if constexpr (TRACE) {
    if (who) a.trace[((size_t)i * (PD_TRACE_STAGES * a.p.layers + 1) + row) * PD_E + e] = v;
  }
}

template <int NC, bool TRACE>
__global__ void __launch_bounds__(PD_THREADS, 1) pose_decoder_kernel(const PoseArgs args) {
  using S = PoseShape<NC>;
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  extern __shared__ __align__(128) char dyn[];   // [PD_SLOTS][PD_CHUNK] weight ring | [2][PFLOATS] parameter blocks
  char* ring = dyn;
  float* pbuf = reinterpret_cast<float*>(dyn + (size_t)PD_SLOTS * PD_CHUNK);
  __shared__ __align__(8) uint64_t full[PD_SLOTS];
  __shared__ __align__(8) uint64_t pbar[2];
  __shared__ __align__(16) float xs[PD_E];        // x: the current token's activation (local copy)
  __shared__ __align__(16) float hs[PD_E];        // remote-written: out_proj / linear2 output + residual
  __shared__ __align__(16) float as_[PD_E];       // remote-written: attention output of all heads
  __shared__ __align__(16) float fs[PD_FF];       // remote-written: ReLU(linear1)
  __shared__ __align__(16) float qkv[3][PD_D];    // remote-written: q, k, v of this CTA's head (CTAs < 8)
  __shared__ __align__(16) float sc[PD_MAX_T];    // attention scores / probabilities
  __shared__ __align__(16) float pv[PD_PV_GROUPS][PD_D];
  __shared__ float red[2 * PD_WARPS];
  __shared__ float pose[8];

  const ap_pose_decoder_params& p = args.p;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t rank = cluster_rank();
  const int L = p.layers, T = args.T, od = p.out_dim;
  const PoseStream<NC> st{&p, (int)rank, (long long)T * L * S::CPL};
  long long q = 0;   // next chunk to consume
  BlockReduce br{red};

  if (tid == 0) {
    for (int s = 0; s < PD_SLOTS; ++s) mbar_init(&full[s], 1);
    mbar_init(&pbar[0], 1);
    mbar_init(&pbar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  griddep_wait();   // cross is written by the preceding GEMM
  if (tid == 0) {
    for (int s = 0; s < PD_SLOTS; ++s) st.issue(s, ring, full);
    st.issue_params(0, pbuf, pbar, T);
    st.issue_params(1, pbuf, pbar, T);
  }
  // token 0 = pose_map(0) = pose_map's bias
  float tok = __ldg(p.pose_map_b + tid);
  // every CTA of the cluster must be running before anyone stores into its shared memory
  cluster_arrive();
  cluster_wait();

#pragma unroll 1
  for (int i = 0; i < T; ++i) {
    xs[tid] = tok + (__ldg(p.pe + (size_t)i * PD_E + tid) + __ldg(p.id_row + tid));
#pragma unroll 1
    for (int l = 0; l < L; ++l) {
      const long long g = (long long)i * L + l;
      if (l > 0) {
        const float* pp = pbuf + ((g - 1) & 1) * S::PFLOATS;
        xs[tid] = layer_norm(hs[tid], pp + 4 * PD_E, pp + 5 * PD_E, p.eps, br);
      }
      trace_store<TRACE>(args, rank == 0, i, PD_TRACE_STAGES * l, tid, xs[tid]);
      __syncthreads();
      // the block of layer g - 1 has been read for the last time (its LN3 ran above, or at the end of the last step)
      if (tid == 0 && g >= 1) st.issue_params(g + 1, pbuf, pbar, T);
      const float* pp = pbuf + (g & 1) * S::PFLOATS;
      mbar_wait(&pbar[g & 1], (uint32_t)((g >> 1) & 1));
      // ---- A: in_proj rows -> q/k/v of the owning head's CTA
      gemv_phase<PD_E, S::NA>(xs, ring, full, q, st, [&](int r, float o) {
        if (lane == 0) {
          const int row = (int)rank * S::BQ + r;   // 0 .. 1535: (q|k|v) x head x dim
          const int which = row / PD_E, head = (row % PD_E) / PD_D, d = row % PD_D;
          dsmem_st(dsmem_addr(&qkv[which][d], (uint32_t)head), o + pp[S::P_BQ + r]);
        }
      });
      cluster_arrive();
      cluster_wait();
      // ---- B: attention, one head per CTA
      if (rank < PD_HEADS) {
        const int h = (int)rank;
        __half* kc = args.kv + (((size_t)l * 2 + 0) * PD_HEADS + h) * (size_t)T * PD_D;
        __half* vc = args.kv + (((size_t)l * 2 + 1) * PD_HEADS + h) * (size_t)T * PD_D;
        if (tid < 2 * PD_D) {
          const int which = 1 + tid / PD_D, d = tid % PD_D;
          (which == 1 ? kc : vc)[(size_t)i * PD_D + d] = __float2half_rn(qkv[which][d]);
        }
        trace_store<TRACE>(args, tid < PD_D, i, PD_TRACE_STAGES * l + 1, h * PD_D + (tid & (PD_D - 1)),
                           qkv[0][tid & (PD_D - 1)]);
        __syncthreads();
        const float* mrow = p.mask + ((size_t)h * p.mask_len + i) * p.mask_len;
        float m = -INFINITY;
        for (int j = tid; j <= i; j += PD_THREADS) {
          const uint4* kr = reinterpret_cast<const uint4*>(kc + (size_t)j * PD_D);
          float s = 0.f;
#pragma unroll
          for (int u = 0; u < PD_D / 8; ++u) s += dot8(__ldcg(kr + u), &qkv[0][u * 8]);
          s = s * 0.125f + __ldg(mrow + j);
          sc[j] = s;
          m = fmaxf(m, s);
        }
        m = br.max(m);
        float z = 0.f;
        for (int j = tid; j <= i; j += PD_THREADS) {
          const float e = expf(sc[j] - m);
          sc[j] = e;
          z += e;
        }
        z = br.sum(z);   // its __syncthreads also publishes sc[]
        {
          const int c = tid & 7, gq = tid >> 3;   // 8 dims of key j = gq, gq + 64, ...
          float acc[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll 4
          for (int j = gq; j <= i; j += PD_PV_GROUPS) {
            const uint4 u = __ldcg(reinterpret_cast<const uint4*>(vc + (size_t)j * PD_D) + c);
            const __half2* hv = reinterpret_cast<const __half2*>(&u);
            const float pj = sc[j];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 f = __half22float2(hv[k]);
              acc[2 * k] = fmaf(pj, f.x, acc[2 * k]);
              acc[2 * k + 1] = fmaf(pj, f.y, acc[2 * k + 1]);
            }
          }
#pragma unroll
          for (int k = 0; k < 8; ++k) pv[gq][c * 8 + k] = acc[k];
        }
        __syncthreads();
        {   // per dim: 8 partial sums over 8 groups each, then their sum (fixed order)
          static_assert(PD_PV_GROUPS == 64 && PD_THREADS == 8 * PD_D, "two-level P.V reduction");
          const int d = tid & (PD_D - 1), qq = tid >> 6;
          float s = pv[qq * 8][d];
#pragma unroll
          for (int k = 1; k < 8; ++k) s += pv[qq * 8 + k][d];
          __syncthreads();
          pv[qq][d] = s;
          __syncthreads();
        }
        {
          const int d = tid & (PD_D - 1);
          float s = pv[0][d];
#pragma unroll
          for (int k = 1; k < 8; ++k) s += pv[k][d];
          s = s / z;
          for (int rk = tid >> 6; rk < NC; rk += PD_THREADS / PD_D) dsmem_st(dsmem_addr(&as_[h * PD_D + d], (uint32_t)rk), s);
        }
      }
      cluster_arrive();
      cluster_wait();
      trace_store<TRACE>(args, rank == 0, i, PD_TRACE_STAGES * l + 2, tid, as_[tid]);
      // ---- C: out_proj rows + bias + residual
      gemv_phase<PD_E, S::NCo>(as_, ring, full, q, st, [&](int r, float o) {
        const int row = (int)rank * S::BO + r;
        const float y = xs[row] + (o + pp[S::P_BO + r]);
        if (lane < NC) dsmem_st(dsmem_addr(&hs[row], (uint32_t)lane), y);
      });
      cluster_arrive();
      cluster_wait();
      // ---- D: LN1, + cross, LN2 (redundant), then linear1 rows + ReLU
      {
        float y = layer_norm(hs[tid], pp + 0 * PD_E, pp + 1 * PD_E, p.eps, br);
        y = y + pp[S::P_CR + tid];
        xs[tid] = layer_norm(y, pp + 2 * PD_E, pp + 3 * PD_E, p.eps, br);
        trace_store<TRACE>(args, rank == 0, i, PD_TRACE_STAGES * l + 3, tid, xs[tid]);
        __syncthreads();
        gemv_phase<PD_E, S::ND>(xs, ring, full, q, st, [&](int r, float o) {
          const int row = (int)rank * S::B1 + r;
          const float y1 = fmaxf(o + pp[S::P_B1 + r], 0.f);
          if (lane < NC) dsmem_st(dsmem_addr(&fs[row], (uint32_t)lane), y1);
        });
      }
      cluster_arrive();
      cluster_wait();
      // ---- E: linear2 rows + bias + residual
      gemv_phase<PD_FF, S::NE>(fs, ring, full, q, st, [&](int r, float o) {
        const int row = (int)rank * S::B2 + r;
        const float y = xs[row] + (o + pp[S::P_B2 + r]);
        if (lane < NC) dsmem_st(dsmem_addr(&hs[row], (uint32_t)lane), y);
      });
      cluster_arrive();
      cluster_wait();
      trace_store<TRACE>(args, rank == 0, i, PD_TRACE_STAGES * l + 4, tid, hs[tid]);
    }
    // ---- pose head and next token, redundantly in every CTA (no remote stores: hs is not written again before the next
    // step's phase C, two barriers away)
    {
      const float* pp = pbuf + (((long long)i * L + L - 1) & 1) * S::PFLOATS;
      xs[tid] = layer_norm(hs[tid], pp + 4 * PD_E, pp + 5 * PD_E, p.eps, br);
      trace_store<TRACE>(args, rank == 0, i, PD_TRACE_STAGES * L, tid, xs[tid]);
      __syncthreads();
      if (warp < od) {
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < PD_E / 32; ++u) s = fmaf(__ldg(p.pose_map_r_w + (size_t)warp * PD_E + u * 32 + lane), xs[u * 32 + lane], s);
        s = warp_sum(s) + __ldg(p.pose_map_r_b + warp);
        if (lane == 0) {
          pose[warp] = s;
          if (rank == 0) args.out[(size_t)i * od + warp] = s;
        }
      }
      __syncthreads();
      float t = 0.f;
#pragma unroll 1
      for (int o = 0; o < od; ++o) t = fmaf(__ldg(p.pose_map_w + (size_t)tid * od + o), pose[o], t);
      tok = t + __ldg(p.pose_map_b + tid);
    }
  }
  // Every chunk and parameter block issued has been waited for (the issue functions stop at the call's last one), so no
  // bulk copy is in flight. The last remote stores (phase E of the last layer) precede the last cluster barrier: no CTA's
  // shared memory is accessed by another CTA after this point, so the CTAs may exit independently.
}

// Cluster size per device, chosen once: 16 CTAs if the device can co-schedule a cluster of 16 with this kernel's resources
// (a non-portable size), else 8; AP_POSE_CTAS=8|16 asks for one size instead (both sizes compute identical bytes; the
// override lets one device test the 8-CTA kernel). 0 = not chosen yet, < 0 = minus the size that cannot run.
constexpr int PD_MAX_DEVICES = 64;
static int g_pose_ctas[PD_MAX_DEVICES] = {0};

template <int NC, bool TRACE>
static bool allow_cluster_smem() {   // the non-portable cluster size and the dynamic shared memory of one instantiation
  if (NC > 8 && cudaFuncSetAttribute(pose_decoder_kernel<NC, TRACE>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) !=
                    cudaSuccess)
    return false;
  return cudaFuncSetAttribute(pose_decoder_kernel<NC, TRACE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)PoseShape<NC>::SMEM) == cudaSuccess;
}

template <int NC>
static int max_active_clusters() {
  if (!allow_cluster_smem<NC, false>()) return 0;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(NC);
  cfg.blockDim = dim3(PD_THREADS);
  cfg.dynamicSmemBytes = PoseShape<NC>::SMEM;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = NC;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, pose_decoder_kernel<NC, false>, &cfg) != cudaSuccess) n = 0;
  return n;
}

static int pose_ctas(int* out) {
  int dev = 0;
  AP_CHECK_CUDA(cudaGetDevice(&dev));
  AP_REQUIRE(dev >= 0 && dev < PD_MAX_DEVICES, "pose_decoder: device %d out of range", dev);
  if (g_pose_ctas[dev] == 0) {
    const char* want = getenv("AP_POSE_CTAS");
    AP_REQUIRE(!want || !strcmp(want, "8") || !strcmp(want, "16"), "pose_decoder: AP_POSE_CTAS=%s must be 8 or 16", want);
    if (want && !strcmp(want, "8"))
      g_pose_ctas[dev] = max_active_clusters<8>() > 0 ? 8 : -8;
    else if (want)
      g_pose_ctas[dev] = max_active_clusters<16>() > 0 ? 16 : -16;
    else
      g_pose_ctas[dev] = max_active_clusters<16>() > 0 ? 16 : (max_active_clusters<8>() > 0 ? 8 : -8);
    cudaGetLastError();   // a refused query must not leave an error behind for the next launch
  }
  if (g_pose_ctas[dev] < 0)
    return fail(AP_ERR_CUDA, "pose_decoder: the device cannot co-schedule a cluster of %d CTAs", -g_pose_ctas[dev]);
  *out = g_pose_ctas[dev];
  return AP_OK;
}

template <int NC, bool TRACE>
static cudaError_t launch_decoder(const PoseArgs& args, void* stream) {
  if (TRACE && !allow_cluster_smem<NC, TRACE>()) {   // the test hook sets its own attributes, at its own launches
    const cudaError_t e = cudaGetLastError();
    return e != cudaSuccess ? e : cudaErrorInvalidConfiguration;
  }
  return launch_pdl(pose_decoder_kernel<NC, TRACE>, dim3(NC), dim3(PD_THREADS), PoseShape<NC>::SMEM,
                    (cudaStream_t)stream, NC, args);
}

// ap_pose_decoder_f16 (trace == nullptr) and its traced test hook: one validation, one launch.
static int pose_decoder(const ap_pose_decoder_params* params, int T, void* kv_cache, float* out, float* trace,
                        void* stream) {
  AP_REQUIRE(params && kv_cache && out, "pose_decoder: null pointer");
  const ap_pose_decoder_params& p = *params;
  AP_REQUIRE(p.w_qkv && p.w_out && p.w_ff1 && p.w_ff2 && p.vec && p.pose_map_w && p.pose_map_b && p.pose_map_r_w &&
                 p.pose_map_r_b && p.pe && p.id_row && p.mask && p.cross,
             "pose_decoder: null parameter pointer");
  AP_REQUIRE(p.embed_dim == PD_E && p.heads == PD_HEADS && p.ffn_dim == PD_FF,
             "pose_decoder: only E = %d, %d heads, FFN %d are supported (got E = %d, %d heads, FFN %d)", PD_E, PD_HEADS,
             PD_FF, p.embed_dim, p.heads, p.ffn_dim);
  AP_REQUIRE(p.layers >= 1, "pose_decoder: layers = %d must be >= 1", p.layers);
  AP_REQUIRE(p.out_dim >= 1 && p.out_dim <= 8, "pose_decoder: out_dim = %d must be in [1, 8]", p.out_dim);
  AP_REQUIRE(T >= 1 && T <= p.mask_len && T <= p.pe_len && T <= PD_MAX_T,
             "pose_decoder: T = %d must be in [1, min(mask_len %d, pe_len %d, %d)]", T, p.mask_len, p.pe_len, PD_MAX_T);
  AP_REQUIRE(p.eps > 0.f, "pose_decoder: eps must be > 0");
  const void* a16[] = {p.w_qkv, p.w_out, p.w_ff1, p.w_ff2, p.vec, p.cross, kv_cache};
  for (const void* q : a16) AP_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0, "pose_decoder: the weights, vec, cross "
                                       "and the KV cache must be 16-byte aligned");
  const float* a4[] = {p.pose_map_w, p.pose_map_b, p.pose_map_r_w, p.pose_map_r_b, p.pe, p.id_row, p.mask, out, trace};
  for (const float* q : a4) AP_REQUIRE((reinterpret_cast<uintptr_t>(q) & 3) == 0, "pose_decoder: fp32 operands must be "
                                       "4-byte aligned");
  int nc = 0;
  int rc = pose_ctas(&nc);
  if (rc) return rc;
  PoseArgs args{p, T, out, reinterpret_cast<__half*>(kv_cache), trace};
  cudaError_t e = nc == 16 ? (trace ? launch_decoder<16, true>(args, stream) : launch_decoder<16, false>(args, stream))
                           : (trace ? launch_decoder<8, true>(args, stream) : launch_decoder<8, false>(args, stream));
  if (e != cudaSuccess)
    return fail(AP_ERR_CUDA, "launch pose_decoder_kernel<%d%s>: %s", nc, trace ? ", trace" : "", cudaGetErrorString(e));
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

}  // namespace ap

using namespace ap;

extern "C" int ap_pose_decoder_ctas(int* ctas) {
  AP_REQUIRE(ctas, "pose_decoder_ctas: null pointer");
  return pose_ctas(ctas);
}

extern "C" int ap_pose_decoder_f16(const ap_pose_decoder_params* params, int T, void* kv_cache, float* out, void* stream) {
  return pose_decoder(params, T, kv_cache, out, nullptr, stream);
}

extern "C" int ap_pose_decoder_trace_f16(const ap_pose_decoder_params* params, int T, void* kv_cache, float* out,
                                         float* trace, void* stream) {
  AP_REQUIRE(trace, "pose_decoder_trace: null trace pointer");
  return pose_decoder(params, T, kv_cache, out, trace, stream);
}
