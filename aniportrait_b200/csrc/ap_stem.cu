// PoseGuider building blocks that are not GEMM-shaped: train-mode BatchNorm (+ReLU / GELU) over channels-last activations and the
// small-channel (3..64) k3/k4 convolutions of its stem.
//
// Replaces nn.BatchNorm2d in TRAIN mode (the reference never calls .eval() on the PoseGuider: batch statistics over the
// (frames, H, W) of the window, biased variance, eps 1e-5) + nn.ReLU, and the nn.Conv2d layers with 3/16/32 input
// channels (reference src/models/pose_guider.py:19-46,124-131). The 64..1280-channel 3x3 convolutions of the same module run on
// the wgmma implicit-GEMM kernel (ap_gemm.cu).
//
// Both are HBM / CUDA-core work: 1.3 GFLOP per frame in total for the stem convolutions, one read + one write of the
// activation for the BatchNorm apply, one extra read for its statistics. Reductions are two-stage and order-fixed (no
// floating-point atomics), so results are bit-reproducible.
#include "ap_host.h"
#include "ap_ptx.cuh"

namespace ap {

// ---------------------------------------------------------------------------------------------------------
// BatchNorm, batch statistics. x: [rows, C] fp16 (rows = frames*H*W), C % 8 == 0.
// Stage 1: block = (C/8) * k threads, each thread owns 8 channels and strides over the block's rows; per-channel
//          {sum, sumsq} partials per block.   Stage 2: one thread per channel adds the partials in double, in block order,
//          and emits the affine pair a = gamma * rstd, b = beta - mean * a.   Stage 3: y = act(a x + b).
// For one clip, wav2vec2's GroupNorm(512 groups, 512 channels) over time is exactly this per-channel batch normalisation
// over the [T0, 512] rows of its first convolution (act = GELU).
// ---------------------------------------------------------------------------------------------------------
__global__ void bn_stats_kernel(const __half* __restrict__ x, long long rows, int C, int rows_per_block,
                                float2* __restrict__ partials) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int vecs = C >> 3;
  const int k = blockDim.x / vecs;
  const int cv = threadIdx.x % vecs;
  const int rl = threadIdx.x / vecs;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = min(r0 + (long long)rows_per_block, rows);
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  if (rl < k) {
    const __half* base = x + cv * 8;
#pragma unroll 4
    for (long long r = r0 + rl; r < r1; r += k) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(base + r * C));
      const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h2[j]);
        s[2 * j] += f.x; q[2 * j] += f.x * f.x;
        s[2 * j + 1] += f.y; q[2 * j + 1] += f.y * f.y;
      }
    }
  }
  extern __shared__ float2 sh[];  // [k][C]
  if (rl < k) {
#pragma unroll
    for (int j = 0; j < 8; ++j) sh[rl * C + cv * 8 + j] = make_float2(s[j], q[j]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float as = 0.f, aq = 0.f;
    for (int r = 0; r < k; ++r) {
      const float2 v = sh[r * C + c];
      as += v.x;
      aq += v.y;
    }
    partials[(long long)blockIdx.x * C + c] = make_float2(as, aq);
  }
}

__global__ void bn_finalize_kernel(const float2* __restrict__ partials, int chunks, int C, double inv_rows, float eps,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float2* __restrict__ ab) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0, q = 0.0;
  for (int i = 0; i < chunks; ++i) {
    const float2 v = partials[(long long)i * C + c];
    s += v.x;
    q += v.y;
  }
  const double mean = s * inv_rows;
  const double var = fmax(q * inv_rows - mean * mean, 0.0);   // biased variance, as F.batch_norm(training=True) normalises
  const double a = (double)gamma[c] / sqrt(var + (double)eps);
  ab[c] = make_float2((float)a, (float)((double)beta[c] - mean * a));
}

template <int ACT>   // 0 none, 1 ReLU, 2 GELU (erf)
__global__ void bn_apply_kernel(const __half* __restrict__ x, long long n_vec, int C, const float2* __restrict__ ab,
                                __half* __restrict__ y) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int vecs = C >> 3;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % vecs) * 8;
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(x) + i);
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
    uint4 o;
    __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h2[j]);
      const float2 p0 = __ldg(ab + c0 + 2 * j), p1 = __ldg(ab + c0 + 2 * j + 1);
      float v0 = fmaf(f.x, p0.x, p0.y), v1 = fmaf(f.y, p1.x, p1.y);
      if (ACT == 1) {
        v0 = fmaxf(v0, 0.f);
        v1 = fmaxf(v1, 0.f);
      } else if (ACT == 2) {
        v0 = gelu_erf(v0);
        v1 = gelu_erf(v1);
      }
      o2[j] = __floats2half2_rn(v0, v1);
    }
    reinterpret_cast<uint4*>(y)[i] = o;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Direct convolution for few channels. x: [Nf, H, W, CIN] fp16, w: [Cout, K, K, CIN] fp16, out: [Nf, Ho, Wo, Cout].
// Thread = one output pixel x COUT_T output channels (fp32 accumulators); the block's weight slab [K*K][CIN][COUT_T] sits in
// shared memory as fp32 and is read with warp-broadcast 16-byte loads; the input pixel's CIN channels arrive as 16-byte
// global loads (neighbouring threads read neighbouring pixels: coalesced, taps hit L1).
// ---------------------------------------------------------------------------------------------------------
template <int CIN, int K, int S, int COUT_T>
__global__ void __launch_bounds__(128)
conv_direct_kernel(const __half* __restrict__ x, const __half* __restrict__ w, const float* __restrict__ bias,
                   __half* __restrict__ out, int Nf, int H, int W, int Ho, int Wo, int Cout, int pad) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  __shared__ __align__(16) float ws[K * K * CIN * COUT_T];
  const int co0 = blockIdx.y * COUT_T;
  for (int i = threadIdx.x; i < K * K * CIN * COUT_T; i += blockDim.x) {
    const int co = i % COUT_T;
    const int ci = (i / COUT_T) % CIN;
    const int tap = i / (COUT_T * CIN);
    ws[i] = __half2float(w[((long long)(co0 + co) * (K * K) + tap) * CIN + ci]);
  }
  __syncthreads();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)Nf * Ho * Wo;
  if (pix >= total) return;
  const int ox = (int)(pix % Wo);
  const int oy = (int)((pix / Wo) % Ho);
  const int n = (int)(pix / ((long long)Wo * Ho));
  float acc[COUT_T];
#pragma unroll
  for (int j = 0; j < COUT_T; ++j) acc[j] = bias ? __ldg(bias + co0 + j) : 0.f;
  const __half* xin = x + (long long)n * H * W * CIN;
#pragma unroll
  for (int ky = 0; ky < K; ++ky) {
    const int iy = oy * S - pad + ky;
    if (iy < 0 || iy >= H) continue;
#pragma unroll
    for (int kx = 0; kx < K; ++kx) {
      const int ix = ox * S - pad + kx;
      if (ix < 0 || ix >= W) continue;
      const uint4* src = reinterpret_cast<const uint4*>(xin + ((long long)iy * W + ix) * CIN);
      const float* wt = ws + (ky * K + kx) * CIN * COUT_T;
#pragma unroll
      for (int c8 = 0; c8 < CIN / 8; ++c8) {
        const uint4 u = __ldg(src + c8);
        const __half2* h2 = reinterpret_cast<const __half2*>(&u);
        float xv[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h2[j]);
          xv[2 * j] = f.x;
          xv[2 * j + 1] = f.y;
        }
#pragma unroll
        for (int ci = 0; ci < 8; ++ci) {
          const float4* w4 = reinterpret_cast<const float4*>(wt + (c8 * 8 + ci) * COUT_T);
#pragma unroll
          for (int j = 0; j < COUT_T / 4; ++j) {
            const float4 wv = w4[j];
            acc[4 * j + 0] = fmaf(xv[ci], wv.x, acc[4 * j + 0]);
            acc[4 * j + 1] = fmaf(xv[ci], wv.y, acc[4 * j + 1]);
            acc[4 * j + 2] = fmaf(xv[ci], wv.z, acc[4 * j + 2]);
            acc[4 * j + 3] = fmaf(xv[ci], wv.w, acc[4 * j + 3]);
          }
        }
      }
    }
  }
  __half* dst = out + pix * Cout + co0;
#pragma unroll
  for (int q = 0; q < COUT_T / 8; ++q) {
    __half2 o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = __floats2half2_rn(acc[q * 8 + 2 * j], acc[q * 8 + 2 * j + 1]);
    *reinterpret_cast<uint4*>(dst + q * 8) = *reinterpret_cast<uint4*>(o);
  }
}

template <int CIN, int K, int S, int COUT_T>
static int launch_conv_direct(const void* x, const void* w, const float* bias, void* out, int Nf, int H, int W, int Ho,
                              int Wo, int Cout, int pad, cudaStream_t stream) {
  const long long total = (long long)Nf * Ho * Wo;
  dim3 grid((unsigned)((total + 127) / 128), (unsigned)(Cout / COUT_T));
  AP_LAUNCH((conv_direct_kernel<CIN, K, S, COUT_T>), grid, 128, 0, stream, (const __half*)x, (const __half*)w, bias, (__half*)out,
                                                                  Nf, H, W, Ho, Wo, Cout, pad);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

}  // namespace ap

using namespace ap;

extern "C" int ap_batchnorm_train_nhwc_f16(const void* x, long long rows, int C, const float* gamma, const float* beta,
                                           float eps, int act, float* workspace, long long workspace_floats, void* out,
                                           void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  AP_REQUIRE(x && out && gamma && beta && workspace, "batchnorm: null pointer");
  AP_REQUIRE(act >= AP_ACT_NONE && act <= AP_ACT_GELU, "batchnorm: activation %d is not one of AP_ACT_*", act);
  AP_REQUIRE(rows > 0 && C > 0 && C % 8 == 0 && C / 8 <= 256, "batchnorm: C=%d must be a multiple of 8, <= 2048", C);
  AP_REQUIRE(aligned16(x) && aligned16(out), "batchnorm: x and out must be 16-byte aligned");
  const int vecs = C / 8;
  int k = 256 / vecs;
  if (k < 1) k = 1;
  const int threads = vecs * k;
  AP_REQUIRE((size_t)k * C * sizeof(float2) <= 48 * 1024, "batchnorm: C=%d too wide for the reduction buffer", C);
  // at most AP_BN_MAX_BLOCKS partial rows; at least 8 rows per row-lane
  long long rpb = 8LL * k;
  const long long min_rpb = (rows + AP_BN_MAX_BLOCKS - 1) / AP_BN_MAX_BLOCKS;
  if (rpb < min_rpb) rpb = (min_rpb + k - 1) / k * k;
  AP_REQUIRE(rpb <= 0x7fffffff, "batchnorm: too many rows");
  const int chunks = (int)((rows + rpb - 1) / rpb);
  AP_REQUIRE(2LL * ((long long)chunks * C + C) <= workspace_floats,
             "batchnorm: workspace too small (%lld floats needed)", 2LL * ((long long)chunks * C + C));
  float2* partials = reinterpret_cast<float2*>(workspace);
  float2* ab = partials + (long long)chunks * C;
  AP_LAUNCH((bn_stats_kernel), chunks, threads, sizeof(float2) * (size_t)k * C, stream, (const __half*)x, rows, C, (int)rpb, partials);
  AP_CHECK_CUDA(cudaGetLastError());
  AP_LAUNCH((bn_finalize_kernel), (C + 127) / 128, 128, 0, stream, partials, chunks, C, 1.0 / (double)rows, eps, gamma, beta, ab);
  AP_CHECK_CUDA(cudaGetLastError());
  const long long n_vec = rows * vecs;
  long long blocks = (n_vec + 255) / 256;
  if (blocks > num_sms() * 16LL) blocks = num_sms() * 16LL;
  if (act == 1) AP_LAUNCH((bn_apply_kernel<1>), (unsigned)blocks, 256, 0, stream, (const __half*)x, n_vec, C, ab, (__half*)out);
  else if (act == 2) AP_LAUNCH((bn_apply_kernel<2>), (unsigned)blocks, 256, 0, stream, (const __half*)x, n_vec, C, ab, (__half*)out);
  else AP_LAUNCH((bn_apply_kernel<0>), (unsigned)blocks, 256, 0, stream, (const __half*)x, n_vec, C, ab, (__half*)out);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}

extern "C" int ap_conv2d_direct_nhwc_f16(const void* x, int Cin, int Nf, int H, int W, const void* w, int Cout, int K,
                                         int stride, int pad, const float* bias, void* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  AP_REQUIRE(x && w && out, "conv2d_direct: null pointer");
  AP_REQUIRE(Nf > 0 && H > 0 && W > 0, "conv2d_direct: bad shape");
  AP_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "conv2d_direct: x/out must be 16-byte aligned");
  const int Ho = (H + 2 * pad - K) / stride + 1, Wo = (W + 2 * pad - K) / stride + 1;
  AP_REQUIRE(Ho > 0 && Wo > 0, "conv2d_direct: empty output");
#define AP_DC(CIN_, K_, S_, CT_)                                                                            \
  if (Cin == CIN_ && K == K_ && stride == S_ && Cout % CT_ == 0)                                            \
    return launch_conv_direct<CIN_, K_, S_, CT_>(x, w, bias, out, Nf, H, W, Ho, Wo, Cout, pad, stream);
  AP_DC(8, 3, 1, 8)
  AP_DC(8, 4, 2, 16)
  AP_DC(16, 3, 1, 16)
  AP_DC(16, 4, 2, 16)
  AP_DC(32, 3, 1, 16)
  AP_DC(32, 4, 2, 16)
#undef AP_DC
  return fail(AP_ERR_INVALID,
              "conv2d_direct: unsupported (Cin=%d, K=%d, stride=%d, Cout=%d): Cin in {8,16,32}, (K,stride) in {(3,1),(4,2)}, "
              "Cout a multiple of 16 (8 for Cin=8,K=3)", Cin, K, stride, Cout);
}
