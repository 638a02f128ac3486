// CLIP vision encoder: the patch extraction that turns the patch-embedding Conv2d(3, C, P, stride P) into a GEMM.
//
// transformers' CLIPVisionEmbeddings computes conv(pixels).flatten(2).transpose(1, 2), prepends class_embedding and adds
// the position table. Here one pass writes the A operand [B * (1 + G^2), kpad]: a CLS row (a single 1.0 in column 3 P^2,
// where the packed weight holds class_embedding) followed by the image's patches in flatten(2) order, each row the patch's
// (c, ky, kx) pixels in Conv2d.weight.reshape(C, -1) order, zero padded to kpad. The GEMM (ap_gemm.cu) then yields
// class token + patch embeddings in one launch, with the tiled position table as its residual. The transformer layers
// run on the GEMM, LayerNorm and attention kernels.
#include "ap_host.h"
#include "ap_ptx.cuh"

namespace ap {

__device__ __forceinline__ float load_px(const __half* p, long long i) { return __half2float(p[i]); }
__device__ __forceinline__ float load_px(const float* p, long long i) { return __ldg(p + i); }

// One thread per 8 consecutive output columns of a row (one 16-byte store).
template <typename T>
__global__ void patchify_nchw_kernel(const T* __restrict__ px, int H, int W, int P, int Gw, int tokens, int kpad,
                                     long long rows, __half* __restrict__ out) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int vecs = kpad >> 3;
  const int kdata = 3 * P * P;
  const long long n = rows * vecs;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / vecs;
    const int k0 = (int)(idx % vecs) * 8;
    const long long b = r / tokens;
    const int t = (int)(r % tokens);
    __align__(16) __half o[8];
    if (t == 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = __float2half_rn(k0 + j == kdata ? 1.f : 0.f);
    } else {
      const int gy = (t - 1) / Gw, gx = (t - 1) % Gw;
      const T* img = px + b * 3LL * H * W;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = k0 + j;
        float v = 0.f;
        if (k < kdata) {
          const int c = k / (P * P), rem = k % (P * P);
          const int y = gy * P + rem / P, x = gx * P + rem % P;
          v = load_px(img, ((long long)c * H + y) * W + x);
        }
        o[j] = __float2half_rn(v);
      }
    }
    *reinterpret_cast<uint4*>(out + r * kpad + k0) = *reinterpret_cast<const uint4*>(o);
  }
}

}  // namespace ap

using namespace ap;

extern "C" int ap_patchify_nchw_f16(const void* pixels, int in_f32, int B, int H, int W, int patch, void* out, int kpad,
                                    void* stream) {
  AP_REQUIRE(pixels && out, "patchify: null pointer");
  AP_REQUIRE(B > 0 && patch > 0 && H > 0 && W > 0 && H % patch == 0 && W % patch == 0,
             "patchify: bad shape B=%d H=%d W=%d patch=%d (H, W must be multiples of the patch)", B, H, W, patch);
  AP_REQUIRE(kpad % 64 == 0 && kpad > 3 * patch * patch, "patchify: kpad=%d must be a multiple of 64 above 3*patch^2=%d",
             kpad, 3 * patch * patch);
  AP_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "patchify: out must be 16-byte aligned");
  const int Gw = W / patch;
  const int tokens = 1 + (H / patch) * Gw;
  const long long rows = (long long)B * tokens;
  const long long n = rows * (kpad / 8);
  long long blocks = (n + 255) / 256;
  if (blocks > num_sms() * 8LL) blocks = num_sms() * 8LL;
  if (in_f32) {
    AP_LAUNCH((patchify_nchw_kernel<float>), (unsigned)blocks, 256, 0, (cudaStream_t)stream, (const float*)pixels, H, W,
              patch, Gw, tokens, kpad, rows, (__half*)out);
  } else {
    AP_LAUNCH((patchify_nchw_kernel<__half>), (unsigned)blocks, 256, 0, (cudaStream_t)stream, (const __half*)pixels, H, W,
              patch, Gw, tokens, kpad, rows, (__half*)out);
  }
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}
