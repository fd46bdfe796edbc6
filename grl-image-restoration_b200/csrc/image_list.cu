// image_list.cu -- a list of differently sized images in and out of one padded batch (GRL.forward_list): the pad-gather
// writes check_image_size of every image into a (n, C, Hp, Wp) fp32 batch, the crop-scatter writes each image's corner of
// the batch's output to its own tensor.
//
// Both are HBM-bound and tiled like image_u8.cu: a CTA of 32 x 8 threads owns a 32 x 32 pixel tile of one image of the
// list (grid.z = image).  The image descriptors (GrlImageRef) travel by value in the kernel parameters, at most
// kListPerLaunch per launch, so a call needs no device copy of them.  8-bit pixels are staged in shared memory by
// grl_pixel_tile.cuh; fp32 planes and packed RGGB planes are read straight from global memory, one thread per output
// column.
#include "grl_common.cuh"
#include "grl_demosaic.h"
#include "grl_image_u8.h"
#include "grl_pixel_tile.cuh"

namespace grl {

namespace {

constexpr int kListPerLaunch = 128;  // 128 x 24-byte refs: 3 KB of the 4 KB of kernel parameters

struct ListRefs {
  GrlImageRef im[kListPerLaunch];
};

// check_image_size on one axis: the source index of padded index p on an axis of n samples, reflected on the bottom /
// right (F.pad "reflect": 2 (n - 1) - p), or -1 in the zero padding.
__device__ __forceinline__ int pad_source(int p, int n, bool reflect) {
  if (p < n) return p;
  return reflect ? 2 * (n - 1) - p : -1;
}

// F.pad(..., "reflect") needs every pad smaller than its axis; otherwise the reference pads both axes with zeros.
__host__ __device__ __forceinline__ bool reflects(int H, int W, int Hp, int Wp) { return Hp - H < H && Wp - W < W; }

// Source readers of the fp32 gather: the network image's size, and its channel c at pixel (y, x).
struct PlanesReader {  // (C, H, W) fp32 planes
  __device__ static int height(const GrlImageRef& im) { return im.H; }
  __device__ static int width(const GrlImageRef& im) { return im.W; }
  __device__ static float read(const GrlImageRef& im, int c, int y, int x) {
    return static_cast<const float*>(im.data)[((long long)c * im.H + y) * im.W + x];
  }
};
struct RggbReader {  // (4, h, w) packed RGGB planes of a (2h, 2w) image, demosaiced on the fly (grl_demosaic.h)
  __device__ static int height(const GrlImageRef& im) { return 2 * im.H; }
  __device__ static int width(const GrlImageRef& im) { return 2 * im.W; }
  __device__ static float read(const GrlImageRef& im, int c, int y, int x) {
    return dm_pixel(static_cast<const float*>(im.data), im.H, im.W, c, y, x);
  }
};

template <class Reader>
__global__ void __launch_bounds__(kTile * kTileRows) gather_planes_kernel(const ListRefs refs, int C, int Hp, int Wp,
                                                                           float* __restrict__ out) {
  const GrlImageRef& im = refs.im[blockIdx.z];
  const int H = Reader::height(im), W = Reader::width(im);
  const bool reflect = reflects(H, W, Hp, Wp);
  const int y0 = blockIdx.y * kTile, x = blockIdx.x * kTile + threadIdx.x;
  if (x >= Wp) return;
  const int xs = pad_source(x, W, reflect);
  const long long plane = (long long)Hp * Wp;
  float* o = out + (long long)blockIdx.z * C * plane + x;
  for (int r = threadIdx.y; r < kTile && y0 + r < Hp; r += kTileRows) {
    const int y = y0 + r, ys = pad_source(y, H, reflect);
    for (int c = 0; c < C; ++c) o[c * plane + (long long)y * Wp] = (ys < 0 || xs < 0) ? 0.f : Reader::read(im, c, ys, xs);
  }
}

// (H, W, C) uint8 -> padded (C, Hp, Wp) fp32 = k / 255; the zero padding is the byte 0, i.e. +0.f.
__global__ void __launch_bounds__(kTile * kTileRows, kTileMinBlocks)
    gather_u8_kernel(const ListRefs refs, int C, int Hp, int Wp, float* __restrict__ out) {
  __shared__ PixelTile tile;
  const GrlImageRef& im = refs.im[blockIdx.z];
  const int H = im.H, W = im.W;
  const bool reflect = reflects(H, W, Hp, Wp);
  const int y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;
  const int rows = min(kTile, Hp - y0), cols = min(kTile, Wp - x0);
  const uint8_t* s = static_cast<const uint8_t*>(im.data);
  tile_load_u8(tile, rows, cols * C, [&](int r, int i) -> uint8_t {
    const int px = i / C, c = i - px * C;
    const int ys = pad_source(y0 + r, H, reflect), xs = pad_source(x0 + px, W, reflect);
    return (ys < 0 || xs < 0) ? 0 : s[((long long)ys * W + xs) * C + c];
  });
  __syncthreads();
  const long long plane = (long long)Hp * Wp;
  float* d = out + (long long)blockIdx.z * C * plane + (long long)y0 * Wp + x0 + threadIdx.x;
  tile_store_f32(tile, rows, cols, C, [&](int c, int r, float v) { d[c * plane + (long long)r * Wp] = v; });
}

// y (n, C, Hy, Wy) -> the top-left (H, W) of image z as (C, H, W) fp32 planes
__global__ void __launch_bounds__(kTile * kTileRows, kTileMinBlocks)
    crop_planes_kernel(const float* __restrict__ y, int C, int Hy, int Wy, const ListRefs refs) {
  const GrlImageRef& im = refs.im[blockIdx.z];
  const int H = im.H, W = im.W;
  const int y0 = blockIdx.y * kTile, x = blockIdx.x * kTile + threadIdx.x;
  if (x >= W) return;
  const long long plane = (long long)Hy * Wy;
  const float* s = y + (long long)blockIdx.z * C * plane + x;
  float* d = static_cast<float*>(im.data) + x;
  for (int r = threadIdx.y; r < kTile && y0 + r < H; r += kTileRows)
    for (int c = 0; c < C; ++c) d[((long long)c * H + y0 + r) * W] = s[c * plane + (long long)(y0 + r) * Wy];
}

// ... as (H, W, C) uint8 = round8(v) (grl_f32_to_u8)
__global__ void __launch_bounds__(kTile * kTileRows, kTileMinBlocks)
    crop_u8_kernel(const float* __restrict__ y, int C, int Hy, int Wy, const ListRefs refs) {
  __shared__ PixelTile tile;
  const GrlImageRef& im = refs.im[blockIdx.z];
  const int H = im.H, W = im.W;
  const int y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;
  if (y0 >= H || x0 >= W) return;  // the grid covers the launch's largest image
  const int rows = min(kTile, H - y0), cols = min(kTile, W - x0);
  const long long plane = (long long)Hy * Wy;
  const float* s = y + (long long)blockIdx.z * C * plane + (long long)y0 * Wy + x0 + threadIdx.x;
  tile_load_f32(tile, rows, cols, C, [&](int c, int r) { return s[c * plane + (long long)r * Wy]; });
  __syncthreads();
  uint8_t* d = static_cast<uint8_t*>(im.data) + ((long long)y0 * W + x0) * C;
  tile_store_u8(tile, rows, cols * C, [&](int r, int i, uint8_t v) { d[(long long)r * W * C + i] = v; });
}

// The checks both entry points make before anything launches; *kind receives the list's kind.
int check_list(const GrlImageRef* images, int n, int C, int Hmax, int Wmax, bool gather, int* kind, const char* what) {
  GRL_REQUIRE(n >= 0 && (images || n == 0), "%s: null image list (n = %d)", what, n);
  GRL_REQUIRE(C >= 1 && C <= kTileMaxC, "%s: C = %d outside 1..%d", what, C, kTileMaxC);
  GRL_REQUIRE(Hmax >= 1 && Wmax >= 1 && Hmax <= 65535 * kTile, "%s: bad batch size %d x %d", what, Hmax, Wmax);
  *kind = n ? images[0].kind : GRL_IMAGE_F32;
  for (int i = 0; i < n; ++i) {
    const GrlImageRef& im = images[i];
    const bool known = im.kind == GRL_IMAGE_F32 || im.kind == GRL_IMAGE_U8 || (gather && im.kind == GRL_IMAGE_RGGB);
    GRL_REQUIRE(known, "%s: image %d: unknown kind %d (%s)", what, i, im.kind,
                gather ? "GRL_IMAGE_F32, _U8 or _RGGB" : "GRL_IMAGE_F32 or _U8");
    GRL_REQUIRE(im.kind == *kind, "%s: image %d has kind %d, image 0 kind %d: one kind per call", what, i, im.kind, *kind);
    GRL_REQUIRE(im.data, "%s: image %d: null data", what, i);
    const bool rggb = im.kind == GRL_IMAGE_RGGB;
    GRL_REQUIRE(im.H >= (rggb ? 2 : 1) && im.W >= (rggb ? 2 : 1), "%s: image %d: bad size %d x %d%s", what, i, im.H, im.W,
                rggb ? " (packed RGGB planes need h, w >= 2)" : "");
    GRL_REQUIRE(!rggb || C == 3, "%s: packed RGGB planes demosaic to C = 3, got C = %d", what, C);
    const long long H = rggb ? 2LL * im.H : im.H, W = rggb ? 2LL * im.W : im.W;
    GRL_REQUIRE(H <= Hmax && W <= Wmax, "%s: image %d (%lld x %lld) is bigger than the batch's %d x %d", what, i, H, W, Hmax,
                Wmax);
  }
  return GRL_OK;
}

ListRefs refs_of(const GrlImageRef* images, int m) {
  ListRefs refs = {};
  for (int j = 0; j < m; ++j) refs.im[j] = images[j];
  return refs;
}

}  // namespace

}  // namespace grl

using namespace grl;

extern "C" {

int grl_list_gather(const GrlImageRef* images, int n, int C, int Hp, int Wp, float* out, void* stream) {
  int kind;
  const int rc = check_list(images, n, C, Hp, Wp, true, &kind, "list_gather");
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(out || n == 0, "list_gather: null output");
  const cudaStream_t st = (cudaStream_t)stream;
  const long long per_image = (long long)C * Hp * Wp;
  for (int i0 = 0; i0 < n; i0 += kListPerLaunch) {
    const int m = min(kListPerLaunch, n - i0);
    const ListRefs refs = refs_of(images + i0, m);
    const dim3 grid(ceil_div(Wp, kTile), ceil_div(Hp, kTile), m), block(kTile, kTileRows);
    float* o = out + i0 * per_image;
    if (kind == GRL_IMAGE_U8) {
      gather_u8_kernel<<<grid, block, 0, st>>>(refs, C, Hp, Wp, o);
      GRL_LAUNCH_CHECK("gather_u8_kernel");
    } else if (kind == GRL_IMAGE_RGGB) {
      gather_planes_kernel<RggbReader><<<grid, block, 0, st>>>(refs, C, Hp, Wp, o);
      GRL_LAUNCH_CHECK("gather_planes_kernel<RggbReader>");
    } else {
      gather_planes_kernel<PlanesReader><<<grid, block, 0, st>>>(refs, C, Hp, Wp, o);
      GRL_LAUNCH_CHECK("gather_planes_kernel<PlanesReader>");
    }
  }
  return GRL_OK;
}

int grl_list_crop(const float* y, int n, int C, int Hy, int Wy, const GrlImageRef* images, void* stream) {
  int kind;
  const int rc = check_list(images, n, C, Hy, Wy, false, &kind, "list_crop");
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(y || n == 0, "list_crop: null input");
  const cudaStream_t st = (cudaStream_t)stream;
  const long long per_image = (long long)C * Hy * Wy;
  for (int i0 = 0; i0 < n; i0 += kListPerLaunch) {
    const int m = min(kListPerLaunch, n - i0);
    const ListRefs refs = refs_of(images + i0, m);
    int H = 1, W = 1;
    for (int j = 0; j < m; ++j) H = max(H, refs.im[j].H), W = max(W, refs.im[j].W);
    const dim3 grid(ceil_div(W, kTile), ceil_div(H, kTile), m), block(kTile, kTileRows);
    const float* s = y + i0 * per_image;
    if (kind == GRL_IMAGE_U8) {
      crop_u8_kernel<<<grid, block, 0, st>>>(s, C, Hy, Wy, refs);
      GRL_LAUNCH_CHECK("crop_u8_kernel");
    } else {
      crop_planes_kernel<<<grid, block, 0, st>>>(s, C, Hy, Wy, refs);
      GRL_LAUNCH_CHECK("crop_planes_kernel");
    }
  }
  return GRL_OK;
}

}  // extern "C"
