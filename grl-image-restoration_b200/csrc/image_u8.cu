// image_u8.cu -- 8-bit HWC images in and out of the fp32 CHW planes the network and the metrics work on (the closed forms
// are grl_image_u8.h).
//
// Both kernels are HBM-bound layout transposes over 32 x 32 pixel tiles of one image (grid.z = B), staged in shared
// memory by grl_pixel_tile.cuh so that every global load and store is coalesced.
#include "grl_common.cuh"
#include "grl_image_u8.h"
#include "grl_pixel_tile.cuh"

namespace grl {

namespace {

// (B, H, W, C) uint8 -> (B, C, H, W) fp32 = k / 255
__global__ void __launch_bounds__(kTile * kTileRows, kTileMinBlocks)
    u8_to_f32_kernel(const uint8_t* __restrict__ src, int H, int W, int C, float* __restrict__ dst) {
  __shared__ PixelTile tile;
  const long long plane = (long long)H * W;
  const int y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;
  const int rows = min(kTile, H - y0), cols = min(kTile, W - x0);
  const uint8_t* s = src + (long long)blockIdx.z * plane * C + ((long long)y0 * W + x0) * C;
  tile_load_u8(tile, rows, cols * C, [&](int r, int i) { return s[(long long)r * W * C + i]; });
  __syncthreads();
  float* d = dst + (long long)blockIdx.z * C * plane + (long long)y0 * W + x0 + threadIdx.x;
  tile_store_f32(tile, rows, cols, C, [&](int c, int r, float v) { d[c * plane + (long long)r * W] = v; });
}

// (B, C, H, W) fp32 -> (B, H, W, C) uint8 = round8(v)
__global__ void __launch_bounds__(kTile * kTileRows, kTileMinBlocks)
    f32_to_u8_kernel(const float* __restrict__ src, int C, int H, int W, uint8_t* __restrict__ dst) {
  __shared__ PixelTile tile;
  const long long plane = (long long)H * W;
  const int y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;
  const int rows = min(kTile, H - y0), cols = min(kTile, W - x0);
  const float* s = src + (long long)blockIdx.z * C * plane + (long long)y0 * W + x0 + threadIdx.x;
  tile_load_f32(tile, rows, cols, C, [&](int c, int r) { return s[c * plane + (long long)r * W]; });
  __syncthreads();
  uint8_t* d = dst + (long long)blockIdx.z * plane * C + ((long long)y0 * W + x0) * C;
  tile_store_u8(tile, rows, cols * C, [&](int r, int i, uint8_t v) { d[(long long)r * W * C + i] = v; });
}

int check_image(const void* src, const void* dst, int B, int H, int W, int C, const char* what) {
  GRL_REQUIRE(src && dst, "%s: null argument", what);
  GRL_REQUIRE(B >= 0 && H > 0 && W > 0 && C >= 1 && C <= kTileMaxC, "%s: bad shape B=%d H=%d W=%d C=%d (C must be 1..%d)",
              what, B, H, W, C, kTileMaxC);
  GRL_REQUIRE(B <= 65535 && H <= 65535 * kTile, "%s: B=%d / H=%d exceed the grid", what, B, H);
  return GRL_OK;
}

}  // namespace

}  // namespace grl

using namespace grl;

extern "C" {

int grl_u8_to_f32(const uint8_t* src, int B, int H, int W, int C, float* dst, void* stream) {
  const int rc = check_image(src, dst, B, H, W, C, "u8_to_f32");
  if (rc != GRL_OK || B == 0) return rc;
  const dim3 grid(ceil_div(W, kTile), ceil_div(H, kTile), B);
  u8_to_f32_kernel<<<grid, dim3(kTile, kTileRows), 0, (cudaStream_t)stream>>>(src, H, W, C, dst);
  GRL_LAUNCH_CHECK("u8_to_f32_kernel");
  return GRL_OK;
}

int grl_f32_to_u8(const float* src, int B, int C, int H, int W, uint8_t* dst, void* stream) {
  const int rc = check_image(src, dst, B, H, W, C, "f32_to_u8");
  if (rc != GRL_OK || B == 0) return rc;
  const dim3 grid(ceil_div(W, kTile), ceil_div(H, kTile), B);
  f32_to_u8_kernel<<<grid, dim3(kTile, kTileRows), 0, (cudaStream_t)stream>>>(src, C, H, W, dst);
  GRL_LAUNCH_CHECK("f32_to_u8_kernel");
  return GRL_OK;
}

int grl_u8_to_f32_host(const uint8_t* src, int B, int H, int W, int C, float* dst) {
  GRL_REQUIRE(src && dst && B >= 0 && H > 0 && W > 0 && C >= 1, "u8_to_f32_host: bad arguments B=%d H=%d W=%d C=%d", B, H, W, C);
  const size_t plane = (size_t)H * W;
  for (size_t b = 0; b < (size_t)B; ++b)
    for (size_t i = 0; i < plane; ++i)
      for (int c = 0; c < C; ++c) dst[(b * C + c) * plane + i] = u8_unit(src[(b * plane + i) * C + c]);
  return GRL_OK;
}

int grl_f32_to_u8_host(const float* src, int B, int C, int H, int W, uint8_t* dst) {
  GRL_REQUIRE(src && dst && B >= 0 && H > 0 && W > 0 && C >= 1, "f32_to_u8_host: bad arguments B=%d C=%d H=%d W=%d", B, C, H, W);
  const size_t plane = (size_t)H * W;
  for (size_t b = 0; b < (size_t)B; ++b)
    for (size_t i = 0; i < plane; ++i)
      for (int c = 0; c < C; ++c) dst[(b * plane + i) * C + c] = (uint8_t)round8(src[(b * C + c) * plane + i]);
  return GRL_OK;
}

}  // extern "C"
