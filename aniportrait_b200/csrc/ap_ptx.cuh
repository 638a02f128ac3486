// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma ordering and descriptors.
// Everything here is hand-written for Hopper H100; nothing is portable to other archs on purpose.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace ap {

// Programmatic dependent launch (see ap_host.h::launch_pdl): let the next kernel be scheduled / wait for the previous one.
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// erf-GELU with ONE MUFU op: erfc(z) = 2^-q(z), q(z) = z * P6(z) fitted to -log2(erfc z) on [0, 4.3] (max relative error of
// erfc 4.2e-5, |error of GELU| <= 1.1e-6: an order of magnitude below the fp16 resolution of the output). With
// z = |x| / sqrt2 clamped to 4.3 (erfc(4.3) = 1.2e-9):  gelu(x) = max(x, 0) - 0.5 |x| erfc(z).
// The previous Abramowitz-Stegun 7.1.26 form needed rcp + ex2; at K = 320 the GEGLU epilogue (16 K outputs per tile and
// CTA) kept the 16-per-clock MUFU pipe busy for 2048 clocks against 2560 clocks of MMA. Shared by the GEGLU and GELU GEMM
// epilogues, the BatchNorm apply and the wav2vec2 positional convolution.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fminf(fabsf(x) * 0.70710678118654752f, 4.3f);
  float q = fmaf(1.686094986e-05f, z, -4.376256625e-04f);
  q = fmaf(q, z, 4.960034474e-03f);
  q = fmaf(q, z, -3.321249048e-02f);
  q = fmaf(q, z, 1.515097036e-01f);
  q = fmaf(q, z, 9.176268788e-01f);
  q = fmaf(q, z, 1.627959694e+00f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-q * z));
  return fmaxf(x, 0.f) - z * 0.70710678118654752f * e;
}

// CLIP's quick_gelu, x * sigmoid(1.702 x) = x / (1 + 2^(-1.702 log2(e) x)): one ex2 and one rcp on the MUFU pipe (relative
// error ~2e-7 each). For x << 0 the exponential overflows to +inf and rcp(inf) = 0, so the result is a signed zero, as in
// torch. Used by the AP_GEMM_QUICK_GELU epilogue.
__device__ __forceinline__ float quick_gelu(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -2.4554669595930157f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.f + e));
  return x * r;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "elect.sync _|P1, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}\n"
      : "=r"(pred));
  return pred;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}\n"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done;
}
// Bounded wait: a protocol bug must trap (kernel error) instead of hanging the GPU box.
#ifndef AP_MBAR_TIMEOUT_CYCLES
#define AP_MBAR_TIMEOUT_CYCLES (8000000000ll)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > AP_MBAR_TIMEOUT_CYCLES) {
      printf("ap: mbarrier timeout block=(%d,%d) thread=%d bar=0x%x parity=%u\n", blockIdx.x, blockIdx.y, threadIdx.x,
             smem_u32(bar), parity);
      __trap();
    }
  }
}

// The same bound without the diagnostic print: a function call inside a wgmma pipeline makes ptxas serialise the
// warpgroup MMAs, so the MMA consumers use this one.
__device__ __forceinline__ void mbar_wait_quiet(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > AP_MBAR_TIMEOUT_CYCLES) __trap();
}

// ----------------------------------------------------------------------------------------------
// TMA tiled loads (global -> shared, completion on an mbarrier)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
          "r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// TMA tiled stores (shared -> global, bulk async-group completion). OOB parts of the box are clipped.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): ordering, shared-memory operand descriptors, register reallocation
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving reads or writes of accumulator registers across an asynchronous wgmma.
template <int N>
__device__ __forceinline__ void reg_fence(float* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
template <uint32_t kRegs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <uint32_t kRegs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// K-major, 128B-swizzled operand tile as TMA writes it (rows at 128 B pitch, 8-row groups 1024 B apart).
// Fields of the sm_90 matrix descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout [62,64) (1 = SWIZZLE_128B).
// Advancing 16 fp16 (32 B) along K inside the swizzle atom is +2 on the descriptor.
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;            // LBO (unused for swizzled K-major) = 1
  d |= static_cast<uint64_t>(1024 >> 4) << 32;    // SBO = 1024 B between 8-row groups
  d |= static_cast<uint64_t>(1) << 62;            // SWIZZLE_128B
  return d;
}
// MN-major, 128B-swizzled operand (the contiguous dim is M/N: 64 fp16 per 128 B row; k rows at 128 B pitch,
// 8-k groups 1024 B apart; further 64-wide MN atoms LBO apart).
__device__ __forceinline__ uint64_t wgmma_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace ap
