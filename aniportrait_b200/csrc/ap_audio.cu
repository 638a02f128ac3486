// wav2vec2 audio-encoder kernels that are not GEMM-shaped: the first feature-extractor convolution over the raw waveform,
// the linear time resampler between the feature extractor and the projection, and the grouped positional convolution.
//
// Replaces, in transformers' Wav2Vec2Model as the reference runs it (src/audio_models/wav2vec2.py:30-64,
// src/audio_models/torch_utils.py:16-19): conv_layers[0].conv (Conv1d(1, 512, 10, 5, bias=False)), the
// F.interpolate(mode="linear", align_corners=True) of linear_interpolation, and pos_conv_embed
// (Conv1d(768, 768, 128, padding=64, groups=16) -> SamePad -> GELU) with the residual add of Wav2Vec2Encoder.forward.
// The strided conv layers 1-6, the projection and the 12 transformer layers run on the wgmma GEMM (ap_gemm.cu), the
// GroupNorm of layer 0 on the BatchNorm kernel (ap_stem.cu), LayerNorm and attention on their own kernels.
//
// All three are small next to the GEMMs (the positional convolution is 2.8 GFLOP for a 10 s clip, the others stream a few
// MB). Every output element is summed in a fixed order: results are bit-reproducible run to run.
#include "ap_host.h"
#include "ap_ptx.cuh"

namespace ap {

// ---------------------------------------------------------------------------------------------------------
// Stem: out[t, c] = sum_k w[c, k] * wave[5 t + k], k < 10. Block = Cout / 2 threads (two channels each, weights in
// registers) x STEM_FR frames; the block's waveform window sits in shared memory. fp32 math, fp16 output.
// ---------------------------------------------------------------------------------------------------------
constexpr int STEM_K = 10, STEM_S = 5, STEM_FR = 16;

__global__ void __launch_bounds__(512)
conv1d_stem_kernel(const float* __restrict__ wave, long long samples, const float* __restrict__ w, long long T0, int Cout,
                   __half* __restrict__ out) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  __shared__ float xs[STEM_FR * STEM_S + STEM_K];
  const int c = 2 * threadIdx.x;
  float w0[STEM_K], w1[STEM_K];
#pragma unroll
  for (int k = 0; k < STEM_K; ++k) {
    w0[k] = __ldg(w + (long long)c * STEM_K + k);
    w1[k] = __ldg(w + (long long)(c + 1) * STEM_K + k);
  }
  griddep_wait();
  const long long t0 = (long long)blockIdx.x * STEM_FR;
  for (int i = threadIdx.x; i < STEM_FR * STEM_S + STEM_K; i += blockDim.x) {
    const long long s = t0 * STEM_S + i;
    xs[i] = s < samples ? __ldg(wave + s) : 0.f;
  }
  __syncthreads();
  for (int f = 0; f < STEM_FR; ++f) {
    const long long t = t0 + f;
    if (t >= T0) break;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int k = 0; k < STEM_K; ++k) {
      const float v = xs[f * STEM_S + k];
      a0 = fmaf(w0[k], v, a0);
      a1 = fmaf(w1[k], v, a1);
    }
    *reinterpret_cast<__half2*>(out + t * Cout + c) = __floats2half2_rn(a0, a1);
  }
}

// ---------------------------------------------------------------------------------------------------------
// Linear resampling of rows (align_corners=True), with torch's index arithmetic: src = scale * i in fp32,
// i0 = min(floor(src), T_in - 1), lambda = clamp(src - i0, 0, 1), out = (1 - lambda) x[i0] + lambda x[i0 + (i0 < T_in - 1)].
// One thread per 8 channels of an output row.
// ---------------------------------------------------------------------------------------------------------
__global__ void resample_rows_linear_kernel(const __half* __restrict__ x, long long T_in, int C, float scale,
                                            __half* __restrict__ out, long long T_out) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int vecs = C >> 3;
  const long long n = T_out * vecs;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
    const long long i = idx / vecs;
    const int v = (int)(idx % vecs);
    const float src = scale * (float)i;
    long long i0 = (long long)floorf(src);
    if (i0 > T_in - 1) i0 = T_in - 1;
    const float l1 = fminf(fmaxf(src - (float)i0, 0.f), 1.f), l0 = 1.f - l1;
    const long long i1 = i0 + (i0 < T_in - 1 ? 1 : 0);
    const uint4 u0 = __ldg(reinterpret_cast<const uint4*>(x + i0 * C) + v);
    const uint4 u1 = __ldg(reinterpret_cast<const uint4*>(x + i1 * C) + v);
    const __half2* h0 = reinterpret_cast<const __half2*>(&u0);
    const __half2* h1 = reinterpret_cast<const __half2*>(&u1);
    uint4 o;
    __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = __half22float2(h0[j]), b = __half22float2(h1[j]);
      o2[j] = __floats2half2_rn(__fadd_rn(__fmul_rn(a.x, l0), __fmul_rn(b.x, l1)),
                                __fadd_rn(__fmul_rn(a.y, l0), __fmul_rn(b.y, l1)));
    }
    reinterpret_cast<uint4*>(out + i * C)[v] = o;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Positional convolution, out[t, g*48 + o] = x[t, g*48 + o] + gelu(bias + sum_{tap, c} w[g*48 + o, tap, c] x[t + tap - K/2, g*48 + c]).
// Per group an implicit GEMM M = T, N = 48, K = 48 * taps on mma.sync m16n8k16. Block = one group x PC_BM = 32 output
// rows, 4 warps = 2 row halves x 2 column halves (16 rows x 24 columns, 3 n-tiles each). The block's input window
// (PC_BM + K - 1 rows x 48 channels, zero outside [0, T)) is loaded once into shared memory (row stride 56 halves: the
// 8 rows x 4 words of an A fragment hit 32 distinct banks); the B fragments come straight from the L2-resident packed
// weight [C][K][48]. The residual is read back from the window.
// ---------------------------------------------------------------------------------------------------------
constexpr int PC_CPG = 48, PC_BM = 32, PC_LD = 56;

__device__ __forceinline__ void mma_16816_f16(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                              uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(128)
pos_conv1d_gelu_kernel(const __half* __restrict__ x, long long T, int C, int K, const __half* __restrict__ w,
                       const float* __restrict__ bias, __half* __restrict__ out) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  extern __shared__ __align__(16) __half xs[];   // [PC_BM + K - 1][PC_LD]
  const int g = blockIdx.y;
  const long long t0 = (long long)blockIdx.x * PC_BM;
  const int half_k = K / 2;
  const int rows = PC_BM + K - 1;
  for (int i = threadIdx.x; i < rows * (PC_CPG / 8); i += blockDim.x) {
    const int r = i / (PC_CPG / 8), v = i % (PC_CPG / 8);
    const long long t = t0 - half_k + r;
    uint4 u = make_uint4(0u, 0u, 0u, 0u);
    if (t >= 0 && t < T) u = __ldg(reinterpret_cast<const uint4*>(x + t * C + g * PC_CPG) + v);
    *reinterpret_cast<uint4*>(xs + r * PC_LD + v * 8) = u;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = (warp & 1) * 16;
  const int nt0 = (warp >> 1) * 3;
  const int qr = lane >> 2, qc = (lane & 3) * 2;
  float acc[3][4];
#pragma unroll
  for (int j = 0; j < 3; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  const long long kk = (long long)K * PC_CPG;   // weight row length
  const __half* wrow[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) wrow[j] = w + ((long long)g * PC_CPG + (nt0 + j) * 8 + qr) * kk + qc;
  for (int tap = 0; tap < K; ++tap) {
    const __half* ar0 = xs + (m0 + qr + tap) * PC_LD + qc;
    const __half* ar1 = ar0 + 8 * PC_LD;
#pragma unroll
    for (int ks = 0; ks < PC_CPG / 16; ++ks) {
      const int c = ks * 16;
      const uint32_t a0 = *reinterpret_cast<const uint32_t*>(ar0 + c);
      const uint32_t a1 = *reinterpret_cast<const uint32_t*>(ar1 + c);
      const uint32_t a2 = *reinterpret_cast<const uint32_t*>(ar0 + c + 8);
      const uint32_t a3 = *reinterpret_cast<const uint32_t*>(ar1 + c + 8);
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const __half* wb = wrow[j] + tap * PC_CPG + c;
        const uint32_t b0 = __ldg(reinterpret_cast<const unsigned int*>(wb));
        const uint32_t b1 = __ldg(reinterpret_cast<const unsigned int*>(wb + 8));
        mma_16816_f16(acc[j], a0, a1, a2, a3, b0, b1);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int n = (nt0 + j) * 8 + qc;
    const int ch = g * PC_CPG + n;
    const float2 b = *reinterpret_cast<const float2*>(bias + ch);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + qr + 8 * h;
      const long long t = t0 + m;
      if (t >= T) continue;
      const float2 r = __half22float2(*reinterpret_cast<const __half2*>(xs + (m + half_k) * PC_LD + n));
      const float v0 = r.x + gelu_erf(acc[j][2 * h] + b.x);
      const float v1 = r.y + gelu_erf(acc[j][2 * h + 1] + b.y);
      *reinterpret_cast<__half2*>(out + t * C + ch) = __floats2half2_rn(v0, v1);
    }
  }
}

}  // namespace ap

using namespace ap;

extern "C" int ap_conv1d_stem_f32(const float* wave, long long samples, const float* w, int Cout, void* out,
                                  void* stream) {
  AP_REQUIRE(wave && w && out, "conv1d_stem: null pointer");
  AP_REQUIRE(samples >= STEM_K, "conv1d_stem: %lld samples give no output frame (need >= %d)", samples, STEM_K);
  AP_REQUIRE(Cout % 64 == 0 && Cout <= 1024, "conv1d_stem: Cout=%d must be a multiple of 64, <= 1024", Cout);
  AP_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0, "conv1d_stem: out must be 4-byte aligned");
  const long long T0 = (samples - STEM_K) / STEM_S + 1;
  AP_LAUNCH((conv1d_stem_kernel), (unsigned)((T0 + STEM_FR - 1) / STEM_FR), Cout / 2, 0, (cudaStream_t)stream, wave, samples,
            w, T0, Cout, (__half*)out);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_resample_rows_linear_f16(const void* x, long long T_in, int C, void* out, long long T_out, void* stream) {
  AP_REQUIRE(x && out, "resample_rows_linear: null pointer");
  AP_REQUIRE(T_in > 0 && T_out > 0 && C > 0 && C % 8 == 0, "resample_rows_linear: bad shape T_in=%lld T_out=%lld C=%d", T_in,
             T_out, C);
  AP_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 && x != out,
             "resample_rows_linear: x/out must be distinct 16-byte aligned buffers");
  const float scale = T_out > 1 ? (float)(T_in - 1) / (float)(T_out - 1) : 0.f;
  const long long n = T_out * (C / 8);
  long long blocks = (n + 255) / 256;
  if (blocks > num_sms() * 8LL) blocks = num_sms() * 8LL;
  AP_LAUNCH((resample_rows_linear_kernel), (unsigned)blocks, 256, 0, (cudaStream_t)stream, (const __half*)x, T_in, C, scale,
            (__half*)out, T_out);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_pos_conv1d_gelu_f16(const void* x, long long T, int C, int groups, int K, const void* w,
                                      const float* bias, void* out, void* stream) {
  AP_REQUIRE(x && w && bias && out, "pos_conv1d_gelu: null pointer");
  AP_REQUIRE(x != out, "pos_conv1d_gelu: out must not alias x");
  AP_REQUIRE(T > 0 && groups > 0 && C == groups * PC_CPG, "pos_conv1d_gelu: C=%d must be %d channels per group x %d groups",
             C, PC_CPG, groups);
  AP_REQUIRE(K >= 2 && K % 2 == 0 && K <= 256, "pos_conv1d_gelu: K=%d must be even and <= 256", K);
  AP_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(out) & 3) == 0 && (reinterpret_cast<uintptr_t>(bias) & 7) == 0,
             "pos_conv1d_gelu: misaligned pointer");
  const size_t smem = (size_t)(PC_BM + K - 1) * PC_LD * sizeof(__half);
  AP_LAUNCH((pos_conv1d_gelu_kernel), dim3((unsigned)((T + PC_BM - 1) / PC_BM), (unsigned)groups), 128, smem,
            (cudaStream_t)stream, (const __half*)x, T, C, K, (const __half*)w, bias, (__half*)out);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}
