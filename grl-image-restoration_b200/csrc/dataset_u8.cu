// dataset_u8.cu -- the demosaicking command's packed Bayer input and the gray JPEG command's MATLAB luma, made on the
// device from clean 8-bit RGB images, from the closed forms of grl_dataset_u8.h.
//
// Both are pixel maps, so a launch takes up to kDatasetPerLaunch images of any sizes, their records by value in the
// kernel parameters (grl_param_list.cuh): blockIdx.y picks the image, the x blocks stride over its work items (a 2 x 2
// quad for the mosaic, a pixel for the luma).  Consecutive threads read consecutive source bytes and write consecutive
// destination elements of each plane.  No workspace, no host sync.
#include "grl_common.cuh"
#include "grl_dataset_u8.h"
#include "grl_param_list.cuh"

namespace grl {

namespace {

constexpr int kDatasetPerLaunch = 128;
constexpr int kDatasetThreads = 256, kDatasetMaxBlocksX = 512;

struct DatasetRecord {  // 24 bytes: 128 (source, destination) GrlImageRef pairs would not fit the kernel parameters
  const uint8_t* src;
  void* dst;
  int H, W;  // of the source image
};
using DatasetRecords = ParamList<DatasetRecord, kDatasetPerLaunch>;

__global__ void __launch_bounds__(kDatasetThreads) mosaic_kernel(const DatasetRecords L) {
  const DatasetRecord& im = L.at[blockIdx.y];
  const int W = im.W, h = im.H >> 1, w = W >> 1;
  const long long quads = (long long)h * w;
  const uint8_t* src = im.src;
  float* dst = static_cast<float*>(im.dst);
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(q / w), x = (int)(q - (long long)y * w);
#pragma unroll
    for (int p = 0; p < 4; ++p) dst[p * quads + q] = mosaic_value(src, W, p, y, x);
  }
}

__global__ void __launch_bounds__(kDatasetThreads) luma_kernel(const DatasetRecords L) {
  const DatasetRecord& im = L.at[blockIdx.y];
  const long long n = (long long)im.H * im.W;
  const uint8_t* src = im.src;
  uint8_t* dst = static_cast<uint8_t*>(im.dst);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = luma_y(src[3 * i], src[3 * i + 1], src[3 * i + 2]);
}

// Every image: an (H, W, 3) uint8 source and its destination, (4, H / 2, W / 2) fp32 planes (mosaic) or (H, W, 1) uint8
// (luma).  An empty destination (a source of one row or column, mosaic) may have a null pointer.
int check_dataset(const GrlImageRef* src, const GrlImageRef* dst, int n, bool mosaic, const char* what) {
  return check_u8_pairs(
      src, dst, n, mosaic ? GRL_IMAGE_RGGB : GRL_IMAGE_U8,
      [&](const GrlImageRef& s) { return mosaic ? make_int2(s.H / 2, s.W / 2) : make_int2(s.H, s.W); },
      [&](const GrlImageRef& s, int i) -> int {
        GRL_REQUIRE((long long)s.H * s.W * 3 <= 0x7fffffffLL, "%s: image %d: %d x %d x 3 bytes is too large", what, i,
                    s.H, s.W);
        return GRL_OK;
      },
      what);
}

int launch_dataset(const GrlImageRef* src, const GrlImageRef* dst, int n, bool mosaic, cudaStream_t st) {
  const auto add = [&](DatasetRecord& r, int, int i) {
    r = {static_cast<const uint8_t*>(src[i].data), dst[i].data, src[i].H, src[i].W};
    return (long long)dst[i].H * dst[i].W;
  };
  return launch_list<DatasetRecords>(n, add, [&](const DatasetRecords& L, int, int m) -> int {
    long long most = 0;  // work items of the launch's largest image
    for (int j = 0; j < m; ++j) {
      const int h = mosaic ? L.at[j].H >> 1 : L.at[j].H, w = mosaic ? L.at[j].W >> 1 : L.at[j].W;
      most = (long long)h * w > most ? (long long)h * w : most;
    }
    const dim3 grid(ceil_div(most, kDatasetThreads) < kDatasetMaxBlocksX ? ceil_div(most, kDatasetThreads)
                                                                         : kDatasetMaxBlocksX, m);
    if (mosaic) {
      mosaic_kernel<<<grid, kDatasetThreads, 0, st>>>(L);
      GRL_LAUNCH_CHECK("mosaic_kernel");
    } else {
      luma_kernel<<<grid, kDatasetThreads, 0, st>>>(L);
      GRL_LAUNCH_CHECK("luma_kernel");
    }
    return GRL_OK;
  });
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
