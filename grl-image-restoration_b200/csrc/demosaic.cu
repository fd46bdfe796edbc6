// demosaic.cu -- dm_matlab (utils/utils_mosaic.py:36-111) as one bandwidth-bound kernel: packed RGGB planes
// (B, 4, h, w) -> RGB (B, 3, 2h, 2w) fp32.
//
// A CTA owns a 16 x 64 pixel tile of one image.  It stages the tile's mosaic plus a 2-pixel halo (reflect applied while
// loading) in shared memory, then every thread evaluates the closed form of grl_demosaic.h on 2 x 2 pixels, reading its
// 5 x 5 neighbourhood from the staged tile.  threadIdx.x walks a row of the tile, so every global store is a coalesced
// 128-byte row segment.
#include "grl_common.cuh"
#include "grl_demosaic.h"

namespace grl {

namespace {

constexpr int kTY = 16, kTX = 64, kHalo = 2;
constexpr int kSY = kTY + 2 * kHalo, kSX = kTX + 2 * kHalo;
constexpr int kThreadsX = 32, kThreadsY = 8;

struct DmTile {
  const float* s;  // staged mosaic, row pitch kSX, (0, 0) = tile pixel (-2, -2)
  int ly, lx;
  __device__ __forceinline__ float operator()(int dy, int dx) const { return s[(ly + kHalo + dy) * kSX + lx + kHalo + dx]; }
};

__global__ void __launch_bounds__(kThreadsX * kThreadsY) demosaic_kernel(const float* __restrict__ cfa4, int h, int w,
                                                                          float* __restrict__ out) {
  __shared__ float tile[kSY * kSX];
  const int H = 2 * h, W = 2 * w;
  const int y0 = blockIdx.y * kTY, x0 = blockIdx.x * kTX;
  const float* planes = cfa4 + (long long)blockIdx.z * 4 * h * w;
  const int tid = threadIdx.y * kThreadsX + threadIdx.x;
  for (int e = tid; e < kSY * kSX; e += kThreadsX * kThreadsY) {
    const int r = e / kSX, cl = e - r * kSX;
    const int Y = y0 - kHalo + r, X = x0 - kHalo + cl;
    if (Y <= H + 1 && X <= W + 1) {  // rows / columns past that are never read by a pixel inside the image
      const int Yr = dm_reflect(Y, H), Xr = dm_reflect(X, W);
      tile[e] = planes[((long long)((Yr & 1) * 2 + (Xr & 1)) * h + (Yr >> 1)) * w + (Xr >> 1)];
    }
  }
  __syncthreads();
  const long long plane = (long long)H * W;
  float* dst = out + (long long)blockIdx.z * 3 * plane;
#pragma unroll
  for (int i = 0; i < kTY / kThreadsY; ++i) {
    const int ly = threadIdx.y + i * kThreadsY, Y = y0 + ly;
    if (Y >= H) break;
#pragma unroll
    for (int j = 0; j < kTX / kThreadsX; ++j) {
      const int lx = threadIdx.x + j * kThreadsX, X = x0 + lx;
      if (X >= W) continue;
      const DmTile m{tile, ly, lx};
#pragma unroll
      for (int c = 0; c < 3; ++c) dst[c * plane + (long long)Y * W + X] = dm_value(c, Y & 1, X & 1, m);
    }
  }
}

}  // namespace

}  // namespace grl

using namespace grl;

extern "C" {

int grl_demosaic_host(const float* cfa4, int B, int h, int w, float* out) {
  GRL_REQUIRE(cfa4 && out && B >= 0 && h >= 2 && w >= 2, "demosaic_host: bad arguments B=%d h=%d w=%d", B, h, w);
  const int H = 2 * h, W = 2 * w;
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < 3; ++c)
      for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x)
          out[(((size_t)b * 3 + c) * H + y) * W + x] = dm_pixel(cfa4 + (size_t)b * 4 * h * w, h, w, c, y, x);
  return GRL_OK;
}

int grl_demosaic_f32(const float* cfa4, int B, int h, int w, float* out, void* stream) {
  GRL_REQUIRE(cfa4 && out, "demosaic: null argument");
  GRL_REQUIRE(B > 0 && h >= 2 && w >= 2, "demosaic: packed RGGB planes must be (B, 4, h, w) with B >= 1 and h, w >= 2, got "
              "B=%d h=%d w=%d", B, h, w);
  GRL_REQUIRE(B <= 65535 && 2LL * h <= 0x7fffffffLL / (2LL * w), "demosaic: shape out of range (B=%d h=%d w=%d)", B, h, w);
  const dim3 grid(ceil_div(2 * w, kTX), ceil_div(2 * h, kTY), B);
  demosaic_kernel<<<grid, dim3(kThreadsX, kThreadsY), 0, (cudaStream_t)stream>>>(cfa4, h, w, out);
  GRL_LAUNCH_CHECK("demosaic_kernel");
  return GRL_OK;
}

}  // extern "C"
