// The comparison grid of the scripts (torch.cat of the tiles, then save_videos_grid's make_grid + `(x * 255).astype(uint8)`
// per frame, reference src/utils/util.py:87-104) as uint8 frames, every frame of every tile in one launch.
#include <stdint.h>

#include "ap_host.h"
#include "ap_ptx.cuh"
#include "ap_u8.cuh"

namespace ap {

constexpr int kGridThreads = 256;

struct GridTiles {
  ap_grid_tile t[AP_GRID_MAX_TILES];
};

__device__ __forceinline__ unsigned grid_sample(const ap_grid_tile& tl, int t, int y, int x, int c) {
  const long long off = t * tl.stride_t + y * tl.stride_h + x * tl.stride_w + (tl.bgr ? 2 - c : c) * tl.stride_c;
  if (tl.dtype == AP_GRID_U8) return __ldg(static_cast<const uint8_t*>(tl.data) + off);
  if (tl.dtype == AP_GRID_F16) return to_u8(__ldg(static_cast<const __half*>(tl.data) + off), 0);
  return to_u8(__ldg(static_cast<const float*>(tl.data) + off), 0);
}

// One thread per group of 4 neighbouring pixels of a grid row; with GW % 4 == 0 (every row starts on a 4-byte boundary)
// their 12 bytes go out as three 4-byte stores.
__global__ void __launch_bounds__(kGridThreads)
video_grid_u8_kernel(const __grid_constant__ GridTiles tiles, int B, int xmaps, int T, int H, int W, int GH, int GW,
                     int packed, uint8_t* __restrict__ out) {
  griddep_launch_dependents();   // PDL: see ap_host.h::launch_pdl
  griddep_wait();
  const int G = (GW + 3) / 4;
  const long long total = (long long)T * GH * G;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
    const int gx = (int)(g % G) * 4;
    const long long r = g / G;
    const int gy = (int)(r % GH);
    const int t = (int)(r / GH);
    // the cell row of this grid row: B = 1 has no padding (make_grid returns the tile itself)
    int cell_row = 0, y = gy;
    if (B > 1) {
      const int yy = gy - 2;
      cell_row = yy >= 0 && yy % (H + 2) < H ? yy / (H + 2) : -1;
      y = yy % (H + 2);
    }
    unsigned px[4][3];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      px[k][0] = px[k][1] = px[k][2] = 0;
      const int gxk = gx + k;
      if (cell_row < 0 || gxk >= GW) continue;
      int cell = 0, x = gxk;
      if (B > 1) {
        const int xx = gxk - 2;
        if (xx < 0 || xx % (W + 2) >= W) continue;
        cell = cell_row * xmaps + xx / (W + 2);
        x = xx % (W + 2);
        if (cell >= B) continue;
      }
      const ap_grid_tile& tl = tiles.t[cell];
#pragma unroll
      for (int c = 0; c < 3; ++c) px[k][c] = grid_sample(tl, t, y, x, c);
    }
    uint8_t* o = out + (r * GW + gx) * 3;
    if (packed) {
      uint32_t* o4 = reinterpret_cast<uint32_t*>(o);
      o4[0] = px[0][0] | (px[0][1] << 8) | (px[0][2] << 16) | (px[1][0] << 24);
      o4[1] = px[1][1] | (px[1][2] << 8) | (px[2][0] << 16) | (px[2][1] << 24);
      o4[2] = px[2][2] | (px[3][0] << 8) | (px[3][1] << 16) | (px[3][2] << 24);
    } else {
      for (int k = 0; k < 4 && gx + k < GW; ++k)
        for (int c = 0; c < 3; ++c) o[3 * k + c] = (uint8_t)px[k][c];
    }
  }
}

}  // namespace ap

extern "C" int ap_video_grid_u8(const ap_grid_tile* tiles, int B, int n_rows, int T, int H, int W, void* out,
                                void* stream) {
  AP_REQUIRE(tiles && out && T > 0 && H > 0 && W > 0 && n_rows > 0, "video_grid_u8: bad arguments");
  AP_REQUIRE(B >= 1 && B <= AP_GRID_MAX_TILES, "video_grid_u8: %d tiles, expected 1 to %d", B, AP_GRID_MAX_TILES);
  ap::GridTiles gt{};
  for (int i = 0; i < B; ++i) {
    const ap_grid_tile& tl = tiles[i];
    AP_REQUIRE(tl.data, "video_grid_u8: tile %d has no data", i);
    AP_REQUIRE(tl.dtype == AP_GRID_U8 || tl.dtype == AP_GRID_F16 || tl.dtype == AP_GRID_F32,
               "video_grid_u8: tile %d has unknown dtype %d", i, tl.dtype);
    gt.t[i] = tl;
  }
  const int xmaps = B == 1 ? 1 : (n_rows < B ? n_rows : B);
  const int ymaps = (B + xmaps - 1) / xmaps;
  const long long GH = B == 1 ? H : (long long)ymaps * (H + 2) + 2;
  const long long GW = B == 1 ? W : (long long)xmaps * (W + 2) + 2;
  AP_REQUIRE(GH <= 65535 && GW <= 65535, "video_grid_u8: grid frame %lldx%lld is too large", GW, GH);
  const bool packed = GW % 4 == 0 && ((uintptr_t)out & 3) == 0;
  const long long groups = (long long)T * GH * ((GW + 3) / 4);
  long long grid = (groups + ap::kGridThreads - 1) / ap::kGridThreads;
  const long long cap = (long long)ap::num_sms() * 16;
  if (grid > cap) grid = cap;
  AP_LAUNCH(ap::video_grid_u8_kernel, (unsigned)grid, ap::kGridThreads, 0, (cudaStream_t)stream, gt, B, xmaps, T, H, W,
            (int)GH, (int)GW, packed ? 1 : 0, (uint8_t*)out);
  AP_CHECK_CUDA(cudaGetLastError());
  return AP_OK;
}
