// dataset_u8.cu -- the demosaicking command's packed Bayer input and the gray JPEG command's MATLAB luma, made on the
// device from clean 8-bit RGB images, from the closed forms of grl_dataset_u8.h.
//
// Both are pixel maps, so a launch takes up to kDatasetPerLaunch images of any sizes, their descriptors by value in the
// kernel parameters: blockIdx.y picks the image, the x blocks stride over its work items (a 2 x 2 quad for the mosaic, a
// pixel for the luma).  Consecutive threads read consecutive source bytes and write consecutive destination elements of
// each plane.  No workspace, no host sync; a longer list takes several launches on the caller's stream.
#include "grl_common.cuh"
#include "grl_dataset_u8.h"

namespace grl {

namespace {

constexpr int kDatasetPerLaunch = 128;  // 128 x 24 bytes of descriptors: 3 KB of the 4 KB of kernel parameters
constexpr int kDatasetThreads = 256, kDatasetMaxBlocksX = 512;

struct DatasetList {
  const uint8_t* src[kDatasetPerLaunch];
  void* dst[kDatasetPerLaunch];
  int H[kDatasetPerLaunch], W[kDatasetPerLaunch];  // of the source image
};
static_assert(sizeof(DatasetList) <= 4096, "kernel parameters");

__global__ void __launch_bounds__(kDatasetThreads) mosaic_kernel(const DatasetList L) {
  const int img = blockIdx.y, W = L.W[img], h = L.H[img] >> 1, w = W >> 1;
  const long long quads = (long long)h * w;
  const uint8_t* src = L.src[img];
  float* dst = static_cast<float*>(L.dst[img]);
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(q / w), x = (int)(q - (long long)y * w);
#pragma unroll
    for (int p = 0; p < 4; ++p) dst[p * quads + q] = mosaic_value(src, W, p, y, x);
  }
}

__global__ void __launch_bounds__(kDatasetThreads) luma_kernel(const DatasetList L) {
  const int img = blockIdx.y;
  const long long n = (long long)L.H[img] * L.W[img];
  const uint8_t* src = L.src[img];
  uint8_t* dst = static_cast<uint8_t*>(L.dst[img]);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = luma_y(src[3 * i], src[3 * i + 1], src[3 * i + 2]);
}

// Every image: an (H, W, 3) uint8 source and its destination, (4, H / 2, W / 2) fp32 planes (mosaic) or (H, W, 1) uint8
// (luma).  An empty destination (a source of one row or column, mosaic) may have a null pointer.
int check_dataset(const GrlImageRef* src, const GrlImageRef* dst, int n, bool mosaic, const char* what) {
  GRL_REQUIRE(n >= 0 && ((src && dst) || n == 0), "%s: null image list (n = %d)", what, n);
  for (int i = 0; i < n; ++i) {
    const GrlImageRef &s = src[i], &d = dst[i];
    const int kind = mosaic ? GRL_IMAGE_RGGB : GRL_IMAGE_U8, dh = mosaic ? s.H / 2 : s.H, dw = mosaic ? s.W / 2 : s.W;
    GRL_REQUIRE(s.kind == GRL_IMAGE_U8 && d.kind == kind, "%s: image %d: kinds %d / %d, need GRL_IMAGE_U8 -> %s", what, i,
                s.kind, d.kind, mosaic ? "GRL_IMAGE_RGGB" : "GRL_IMAGE_U8");
    GRL_REQUIRE(s.H >= 1 && s.W >= 1 && d.H == dh && d.W == dw, "%s: image %d: sizes %d x %d -> %d x %d, need %d x %d",
                what, i, s.H, s.W, d.H, d.W, dh, dw);
    GRL_REQUIRE((long long)s.H * s.W * 3 <= 0x7fffffffLL, "%s: image %d: %d x %d x 3 bytes is too large", what, i, s.H,
                s.W);
    GRL_REQUIRE(s.data && (d.data || (long long)d.H * d.W == 0), "%s: image %d: null data", what, i);
  }
  return GRL_OK;
}

int launch_dataset(const GrlImageRef* src, const GrlImageRef* dst, int n, bool mosaic, cudaStream_t st) {
  DatasetList L;
  for (int i0 = 0; i0 < n; i0 += kDatasetPerLaunch) {
    const int m = n - i0 < kDatasetPerLaunch ? n - i0 : kDatasetPerLaunch;
    long long most = 0;
    for (int j = 0; j < m; ++j) {
      const GrlImageRef &s = src[i0 + j], &d = dst[i0 + j];
      L.src[j] = static_cast<const uint8_t*>(s.data);
      L.dst[j] = d.data;
      L.H[j] = s.H;
      L.W[j] = s.W;
      const long long items = (long long)d.H * d.W;
      most = items > most ? items : most;
    }
    if (most == 0) continue;
    const dim3 grid(ceil_div(most, kDatasetThreads) < kDatasetMaxBlocksX ? ceil_div(most, kDatasetThreads)
                                                                         : kDatasetMaxBlocksX, m);
    if (mosaic) {
      mosaic_kernel<<<grid, kDatasetThreads, 0, st>>>(L);
      GRL_LAUNCH_CHECK("mosaic_kernel");
    } else {
      luma_kernel<<<grid, kDatasetThreads, 0, st>>>(L);
      GRL_LAUNCH_CHECK("luma_kernel");
    }
  }
  return GRL_OK;
}

}  // namespace

}  // namespace grl

using namespace grl;

extern "C" {

int grl_mosaic_u8(const GrlImageRef* src, const GrlImageRef* dst, int n, void* stream) {
  const int rc = check_dataset(src, dst, n, true, "mosaic_u8");
  return rc != GRL_OK ? rc : launch_dataset(src, dst, n, true, (cudaStream_t)stream);
}

int grl_luma_u8(const GrlImageRef* src, const GrlImageRef* dst, int n, void* stream) {
  const int rc = check_dataset(src, dst, n, false, "luma_u8");
  return rc != GRL_OK ? rc : launch_dataset(src, dst, n, false, (cudaStream_t)stream);
}

int grl_mosaic_host(const uint8_t* img, int H, int W, float* out) {
  GRL_REQUIRE(H >= 1 && W >= 1 && img && (out || (H / 2) * (W / 2) == 0), "mosaic_host: bad arguments (%d x %d)", H, W);
  const int h = H / 2, w = W / 2;
  for (int p = 0; p < 4; ++p)
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) out[((long long)p * h + y) * w + x] = mosaic_value(img, W, p, y, x);
  return GRL_OK;
}

int grl_luma_host(const uint8_t* rgb, int64_t n, uint8_t* out) {
  GRL_REQUIRE(n >= 0 && ((rgb && out) || n == 0), "luma_host: bad arguments (n = %lld)", (long long)n);
  for (int64_t i = 0; i < n; ++i) out[i] = luma_y(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
  return GRL_OK;
}

}  // extern "C"
