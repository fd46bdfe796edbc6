// image_list.cu -- a list of differently sized images in and out of one padded batch (GRL.forward_list): the pad-gather
// writes check_image_size of every image into a (n, C, Hp, Wp) fp32 batch, the crop-scatter writes each image's corner of
// the batch's output to its own tensor.  The tiled version (tiling.forward_tile_list) cuts the tiles of a list of images
// into such a batch and blends the batch's outputs into each image's accumulator (grl_tiles.h).
//
// Both are HBM-bound and tiled like image_u8.cu: a CTA of 32 x 8 threads owns a 32 x 32 pixel tile of one image of the
// list (grid.z = image).  The descriptors (GrlImageRef, GrlTileRef, GrlTileImage) travel by value in the kernel
// parameters (grl_param_list.cuh), so a call needs no device copy of them.  8-bit pixels are staged in shared memory by
// grl_pixel_tile.cuh; fp32 planes and packed RGGB planes are read straight from global memory, one thread per output
// column.
#include "grl_common.cuh"
#include "grl_demosaic.h"
#include "grl_image_u8.h"
#include "grl_param_list.cuh"
#include "grl_pixel_tile.cuh"
#include "grl_tiles.h"

namespace grl {

namespace {

// Per launch: 128 x 24-byte GrlImageRef, 96 x 40-byte GrlTileRef or 80 x 48-byte GrlTileImage, and at most a pointer
// and four ints besides.
constexpr int kOtherParams = sizeof(float*) + 4 * sizeof(int);
using ImageRecords = ParamList<GrlImageRef, 128, kOtherParams>;
using TileRecords = ParamList<GrlTileRef, 96, kOtherParams>;
using BlendRecords = ParamList<GrlTileImage, 80, kOtherParams>;

// The region a gather pads into one batch entry: a whole image of a list, or the t x t window at (y0, x0) of a tile's
// source, in the frame the network sees.
struct Window {
  GrlImageRef im;
  int y0, x0, h, w;
};
template <class Reader>
__device__ __forceinline__ Window window(const ImageRecords& refs, int z) {
  const GrlImageRef& im = refs.at[z];
  return {im, 0, 0, Reader::height(im), Reader::width(im)};
}
template <class Reader>
__device__ __forceinline__ Window window(const TileRecords& refs, int z) {
  const GrlTileRef& t = refs.at[z];
  return {t.src, t.y0, t.x0, t.t, t.t};
}

// check_image_size on one axis: the source index of padded index p on an axis of n samples, reflected on the bottom /
// right (F.pad "reflect": 2 (n - 1) - p), or -1 in the zero padding.
__device__ __forceinline__ int pad_source(int p, int n, bool reflect) {
  if (p < n) return p;
  return reflect ? 2 * (n - 1) - p : -1;
}

// F.pad(..., "reflect") needs every pad smaller than its axis; otherwise the reference pads both axes with zeros.
GRL_HD bool reflects(int H, int W, int Hp, int Wp) { return Hp - H < H && Wp - W < W; }

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

// Refs: ImageRecords (whole images) or TileRecords (tile windows).
template <class Reader, class Refs>
__global__ void __launch_bounds__(kTile * kTileRows) gather_planes_kernel(const Refs refs, int C, int Hp, int Wp,
                                                                           float* __restrict__ out) {
  const Window win = window<Reader>(refs, blockIdx.z);
  const bool reflect = reflects(win.h, win.w, Hp, Wp);
  const int y0 = blockIdx.y * kTile, x = blockIdx.x * kTile + threadIdx.x;
  if (x >= Wp) return;
  const int xs = pad_source(x, win.w, reflect);
  const long long plane = (long long)Hp * Wp;
  float* o = out + (long long)blockIdx.z * C * plane + x;
  for (int r = threadIdx.y; r < kTile && y0 + r < Hp; r += kTileRows) {
    const int y = y0 + r, ys = pad_source(y, win.h, reflect);
    for (int c = 0; c < C; ++c)
      o[c * plane + (long long)y * Wp] = (ys < 0 || xs < 0) ? 0.f : Reader::read(win.im, c, win.y0 + ys, win.x0 + xs);
  }
}

// (H, W, C) uint8 -> padded (C, Hp, Wp) fp32 = k / 255; the zero padding is the byte 0, i.e. +0.f.
template <class Refs>
__global__ void __launch_bounds__(kTile * kTileRows, kTileMinBlocks)
    gather_u8_kernel(const Refs refs, int C, int Hp, int Wp, float* __restrict__ out) {
  __shared__ PixelTile tile;
  const Window win = window<PlanesReader>(refs, blockIdx.z);  // uint8 images: (H, W) is the frame
  const int W = win.im.W;
  const bool reflect = reflects(win.h, win.w, Hp, Wp);
  const int y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;
  const int rows = min(kTile, Hp - y0), cols = min(kTile, Wp - x0);
  const uint8_t* s = static_cast<const uint8_t*>(win.im.data);
  tile_load_u8(tile, rows, cols * C, [&](int r, int i) -> uint8_t {
    const int px = i / C, c = i - px * C;
    const int ys = pad_source(y0 + r, win.h, reflect), xs = pad_source(x0 + px, win.w, reflect);
    return (ys < 0 || xs < 0) ? 0 : s[((long long)(win.y0 + ys) * W + win.x0 + xs) * C + c];
  });
  __syncthreads();
  const long long plane = (long long)Hp * Wp;
  float* d = out + (long long)blockIdx.z * C * plane + (long long)y0 * Wp + x0 + threadIdx.x;
  tile_store_f32(tile, rows, cols, C, [&](int c, int r, float v) { d[c * plane + (long long)r * Wp] = v; });
}

// y (n, C, Hy, Wy) -> the top-left (H, W) of image z as (C, H, W) fp32 planes
__global__ void __launch_bounds__(kTile * kTileRows, kTileMinBlocks)
    crop_planes_kernel(const float* __restrict__ y, int C, int Hy, int Wy, const ImageRecords refs) {
  const GrlImageRef& im = refs.at[blockIdx.z];
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
    crop_u8_kernel(const float* __restrict__ y, int C, int Hy, int Wy, const ImageRecords refs) {
  __shared__ PixelTile tile;
  const GrlImageRef& im = refs.at[blockIdx.z];
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

// The checks of one image of a list: *kind is the list's kind (image 0's); max_h / max_w bound its frame (0: no bound).
int check_image(const GrlImageRef& im, int i, int C, bool gather, int kind, int max_h, int max_w, const char* what) {
  const bool known = im.kind == GRL_IMAGE_F32 || im.kind == GRL_IMAGE_U8 || (gather && im.kind == GRL_IMAGE_RGGB);
  GRL_REQUIRE(known, "%s: image %d: unknown kind %d (%s)", what, i, im.kind,
              gather ? "GRL_IMAGE_F32, _U8 or _RGGB" : "GRL_IMAGE_F32 or _U8");
  GRL_REQUIRE(im.kind == kind, "%s: image %d has kind %d, image 0 kind %d: one kind per call", what, i, im.kind, kind);
  GRL_REQUIRE(im.data, "%s: image %d: null data", what, i);
  const bool rggb = im.kind == GRL_IMAGE_RGGB;
  GRL_REQUIRE(im.H >= (rggb ? 2 : 1) && im.W >= (rggb ? 2 : 1), "%s: image %d: bad size %d x %d%s", what, i, im.H, im.W,
              rggb ? " (packed RGGB planes need h, w >= 2)" : "");
  GRL_REQUIRE(!rggb || C == 3, "%s: packed RGGB planes demosaic to C = 3, got C = %d", what, C);
  const long long H = rggb ? 2LL * im.H : im.H, W = rggb ? 2LL * im.W : im.W;
  GRL_REQUIRE(!max_h || (H <= max_h && W <= max_w), "%s: image %d (%lld x %lld) is bigger than the batch's %d x %d", what, i,
              H, W, max_h, max_w);
  return GRL_OK;
}

// The checks both list entry points make before anything launches; *kind receives the list's kind.
int check_list(const GrlImageRef* images, int n, int C, int Hmax, int Wmax, bool gather, int* kind, const char* what) {
  int rc = check_list_args(n, images != nullptr, "image", what);
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(C >= 1 && C <= kTileMaxC, "%s: C = %d outside 1..%d", what, C, kTileMaxC);
  GRL_REQUIRE(Hmax >= 1 && Wmax >= 1 && Hmax <= 65535 * kTile, "%s: bad batch size %d x %d", what, Hmax, Wmax);
  *kind = n ? images[0].kind : GRL_IMAGE_F32;
  for (int i = 0; i < n; ++i) {
    rc = check_image(images[i], i, C, gather, *kind, Hmax, Wmax, what);
    if (rc != GRL_OK) return rc;
  }
  return GRL_OK;
}

// ---------------------------------------------------------------------------------------------- tiled inference
// Every covering tile of a launch, in origin order, is added to the accumulator as E = E + o: the reference adds the
// tiles one slice add_ at a time, so a pixel's sum is rounded after every tile in that order.  A thread owns one output
// column of one image and walks kTile / kTileRows rows of it; the tile outputs it reads are rows of the batch's output.
__global__ void __launch_bounds__(kTile * kTileRows) tile_accumulate_kernel(const float* __restrict__ y, int C, int Hy, int Wy, int s, const BlendRecords refs) {
  const GrlTileImage& im = refs.at[blockIdx.z];
  const TileAxis ay = tile_axis(im.H, im.t, im.overlap), ax = tile_axis(im.W, im.t, im.overlap);
  // the tile rows this launch holds of the image and the output rows they cover
  const int kr0 = im.k0 / ax.n, kr1 = (im.k1 - 1) / ax.n;
  const int Ybeg = tile_origin(ay, kr0) * s, Yend = (tile_origin(ay, kr1) + im.t) * s;
  const int Wo = im.W * s, X = blockIdx.x * kTile + threadIdx.x, Yt = blockIdx.y * kTile;
  if (X >= Wo || Yt >= Yend || Yt + kTile <= Ybeg) return;
  const int c_lo = tile_first(ax, X / s), c_hi = tile_last(ax, X / s);
  const long long plane = (long long)im.H * s * Wo, yplane = (long long)Hy * Wy;
  for (int Y = max(Yt, Ybeg) + (int)threadIdx.y; Y < min(Yt + kTile, Yend); Y += kTileRows) {
    const int r_lo = max(tile_first(ay, Y / s), kr0), r_hi = min(tile_last(ay, Y / s), kr1);
    const int k_lo = max(r_lo * ax.n + c_lo, im.k0), k_hi = min(r_hi * ax.n + c_hi, im.k1 - 1);
    if (k_lo > k_hi) continue;  // no tile of this launch can cover the pixel
    for (int c = 0; c < C; ++c) {
      float* e = im.E + c * plane + (long long)Y * Wo + X;
      float v = *e;
      for (int kr = r_lo; kr <= r_hi; ++kr) {
        const long long row = (long long)(Y - tile_origin(ay, kr) * s) * Wy;
        for (int kc = c_lo; kc <= c_hi; ++kc) {
          const int k = kr * ax.n + kc;
          if (k < im.k0 || k >= im.k1) continue;
          v = v + y[((long long)(im.slot + k - im.k0) * C + c) * yplane + row + X - tile_origin(ax, kc) * s];
        }
      }
      *e = v;
    }
  }
}

// The reference's W at output pixel (Y, X): the number of tiles covering it, an exact float.
__device__ __forceinline__ float tile_count(const TileAxis& ay, const TileAxis& ax, int Y, int X, int s) {
  const int r = Y / s, c = X / s;
  return (float)((tile_last(ay, r) - tile_first(ay, r) + 1) * (tile_last(ax, c) - tile_first(ax, c) + 1));
}

// E / W in place (E.div_(W) with a tensor W is an IEEE division).
__global__ void __launch_bounds__(kTile * kTileRows, kTileMinBlocks)
    tile_finish_f32_kernel(int C, int s, const BlendRecords refs) {
  const GrlTileImage& im = refs.at[blockIdx.z];
  const TileAxis ay = tile_axis(im.H, im.t, im.overlap), ax = tile_axis(im.W, im.t, im.overlap);
  const int Ho = im.H * s, Wo = im.W * s, X = blockIdx.x * kTile + threadIdx.x, Yt = blockIdx.y * kTile;
  if (X >= Wo || Yt >= Ho) return;
  const long long plane = (long long)Ho * Wo;
  for (int Y = Yt + threadIdx.y; Y < min(Yt + kTile, Ho); Y += kTileRows) {
    const float n = tile_count(ay, ax, Y, X, s);
    float* e = im.E + (long long)Y * Wo + X;
    for (int c = 0; c < C; ++c) e[c * plane] = __fdiv_rn(e[c * plane], n);
  }
}

// ... as (H*s, W*s, C) uint8 = round8(E / W) (grl_f32_to_u8 of the reference's result)
__global__ void __launch_bounds__(kTile * kTileRows, kTileMinBlocks)
    tile_finish_u8_kernel(int C, int s, const BlendRecords refs) {
  __shared__ PixelTile tile;
  const GrlTileImage& im = refs.at[blockIdx.z];
  const TileAxis ay = tile_axis(im.H, im.t, im.overlap), ax = tile_axis(im.W, im.t, im.overlap);
  const int Ho = im.H * s, Wo = im.W * s, Y0 = blockIdx.y * kTile, X0 = blockIdx.x * kTile;
  if (Y0 >= Ho || X0 >= Wo) return;  // the grid covers the launch's largest image
  const int rows = min(kTile, Ho - Y0), cols = min(kTile, Wo - X0);
  const long long plane = (long long)Ho * Wo;
  const float* e = im.E + (long long)Y0 * Wo + X0 + threadIdx.x;
  tile_load_f32(tile, rows, cols, C, [&](int c, int r) {
    return __fdiv_rn(e[c * plane + (long long)r * Wo], tile_count(ay, ax, Y0 + r, X0 + threadIdx.x, s));
  });
  __syncthreads();
  uint8_t* d = im.out_u8 + ((long long)Y0 * Wo + X0) * C;
  tile_store_u8(tile, rows, cols * C, [&](int r, int i, uint8_t v) { d[(long long)r * Wo * C + i] = v; });
}

// The checks of one image's blend state.
int check_blend(const GrlTileImage& im, int i, int s, const char* what) {
  GRL_REQUIRE(im.E, "%s: image %d: null accumulator", what, i);
  GRL_REQUIRE(im.H >= 1 && im.W >= 1 && (long long)im.H * s <= 65535 * kTile && (long long)im.W * s <= (1 << 30),
              "%s: image %d: bad size %d x %d at scale %d", what, i, im.H, im.W, s);
  GRL_REQUIRE(im.t >= 1 && im.t <= im.H && im.t <= im.W && im.overlap >= 0 && im.overlap < im.t,
              "%s: image %d: tile %d, overlap %d: needs 0 <= overlap < tile <= min(H, W) = %d", what, i, im.t, im.overlap,
              im.H < im.W ? im.H : im.W);
  return GRL_OK;
}

// The kTile x kTile tiles of the largest image of a launch's m records at scale s, one grid.z per record.
template <class List>
dim3 tile_grid(const List& L, int m, int s) {
  int H = 1, W = 1;
  for (int j = 0; j < m; ++j) H = max(H, L.at[j].H), W = max(W, L.at[j].W);
  return dim3(ceil_div((long long)W * s, kTile), ceil_div((long long)H * s, kTile), m);
}

// The pad-gather of n images or tile windows into (n, C, Hp, Wp), every source of `kind`.
template <class List, class Item>
int gather(const Item* items, int n, int kind, int C, int Hp, int Wp, float* out, cudaStream_t st) {
  const auto add = [&](Item& r, int, int i) {
    r = items[i];
    return 1LL;
  };
  return launch_list<List>(n, add, [&](const List& L, int i0, int m) -> int {
    const dim3 grid(ceil_div(Wp, kTile), ceil_div(Hp, kTile), m), block(kTile, kTileRows);
    float* o = out + i0 * (long long)C * Hp * Wp;
    if (kind == GRL_IMAGE_U8)
      gather_u8_kernel<List><<<grid, block, 0, st>>>(L, C, Hp, Wp, o);
    else if (kind == GRL_IMAGE_RGGB)
      gather_planes_kernel<RggbReader, List><<<grid, block, 0, st>>>(L, C, Hp, Wp, o);
    else
      gather_planes_kernel<PlanesReader, List><<<grid, block, 0, st>>>(L, C, Hp, Wp, o);
    GRL_LAUNCH_CHECK("gather kernel");
    return GRL_OK;
  });
}

// The blend of m images: the batch y's tile outputs added to their accumulators, or (finish) E / count.
int blend(const float* y, int C, int Hy, int Wy, int s, const GrlTileImage* images, int m, bool finish,
          cudaStream_t st) {
  const bool u8 = m && images[0].out_u8;
  const auto add = [&](GrlTileImage& r, int, int i) {
    r = images[i];
    return 1LL;
  };
  return launch_list<BlendRecords>(m, add, [&](const BlendRecords& L, int, int mm) -> int {
    const dim3 grid = tile_grid(L, mm, s), block(kTile, kTileRows);
    if (!finish)
      tile_accumulate_kernel<<<grid, block, 0, st>>>(y, C, Hy, Wy, s, L);
    else if (u8)
      tile_finish_u8_kernel<<<grid, block, 0, st>>>(C, s, L);
    else
      tile_finish_f32_kernel<<<grid, block, 0, st>>>(C, s, L);
    GRL_LAUNCH_CHECK("tile blend kernel");
    return GRL_OK;
  });
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
  return gather<ImageRecords>(images, n, kind, C, Hp, Wp, out, (cudaStream_t)stream);
}

int grl_list_crop(const float* y, int n, int C, int Hy, int Wy, const GrlImageRef* images, void* stream) {
  int kind;
  const int rc = check_list(images, n, C, Hy, Wy, false, &kind, "list_crop");
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(y || n == 0, "list_crop: null input");
  const cudaStream_t st = (cudaStream_t)stream;
  const auto add = [&](GrlImageRef& r, int, int i) {
    r = images[i];
    return 1LL;
  };
  return launch_list<ImageRecords>(n, add, [&](const ImageRecords& L, int i0, int m) -> int {
    const dim3 grid = tile_grid(L, m, 1), block(kTile, kTileRows);
    const float* s = y + i0 * (long long)C * Hy * Wy;
    if (kind == GRL_IMAGE_U8)
      crop_u8_kernel<<<grid, block, 0, st>>>(s, C, Hy, Wy, L);
    else
      crop_planes_kernel<<<grid, block, 0, st>>>(s, C, Hy, Wy, L);
    GRL_LAUNCH_CHECK("crop kernel");
    return GRL_OK;
  });
}

int grl_tile_gather(const GrlTileRef* tiles, int n, int C, int Hp, int Wp, float* out, void* stream) {
  const char* what = "tile_gather";
  int rc = check_list_args(n, tiles != nullptr, "tile", what);
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(C >= 1 && C <= kTileMaxC, "%s: C = %d outside 1..%d", what, C, kTileMaxC);
  GRL_REQUIRE(Hp >= 1 && Wp >= 1 && Hp <= 65535 * kTile, "%s: bad batch size %d x %d", what, Hp, Wp);
  GRL_REQUIRE(out || n == 0, "%s: null output", what);
  const int kind = n ? tiles[0].src.kind : GRL_IMAGE_F32;
  for (int i = 0; i < n; ++i) {
    const GrlTileRef& t = tiles[i];
    rc = check_image(t.src, i, C, true, kind, 0, 0, what);
    if (rc != GRL_OK) return rc;
    const int k = t.src.kind == GRL_IMAGE_RGGB ? 2 : 1;
    GRL_REQUIRE(t.t >= 1 && t.t <= Hp && t.t <= Wp, "%s: tile %d: side %d outside 1..min(Hp, Wp) = %d", what, i, t.t,
                Hp < Wp ? Hp : Wp);
    GRL_REQUIRE(t.y0 >= 0 && t.x0 >= 0 && (long long)t.y0 + t.t <= (long long)k * t.src.H &&
                    (long long)t.x0 + t.t <= (long long)k * t.src.W,
                "%s: tile %d: window %d x %d at (%d, %d) is outside the %lld x %lld image", what, i, t.t, t.t, t.y0, t.x0,
                (long long)k * t.src.H, (long long)k * t.src.W);
  }
  return gather<TileRecords>(tiles, n, kind, C, Hp, Wp, out, (cudaStream_t)stream);
}

int grl_tile_accumulate(const float* y, int n, int C, int Hy, int Wy, int scale, const GrlTileImage* images, int m,
                        void* stream) {
  const char* what = "tile_accumulate";
  int rc = check_list_args(m, images != nullptr, "image", what);
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(C >= 1 && C <= kTileMaxC, "%s: C = %d outside 1..%d", what, C, kTileMaxC);
  GRL_REQUIRE(scale >= 1 && n >= 0 && Hy >= 1 && Wy >= 1, "%s: bad batch (n %d, %d x %d) or scale %d", what, n, Hy, Wy,
              scale);
  GRL_REQUIRE(y || m == 0, "%s: null input", what);
  for (int i = 0; i < m; ++i) {
    const GrlTileImage& im = images[i];
    rc = check_blend(im, i, scale, what);
    if (rc != GRL_OK) return rc;
    const long long tiles = (long long)tile_axis(im.H, im.t, im.overlap).n * tile_axis(im.W, im.t, im.overlap).n;
    GRL_REQUIRE(im.k0 >= 0 && im.k0 < im.k1 && im.k1 <= tiles, "%s: image %d: tiles [%d, %d) outside its %lld tiles", what, i,
                im.k0, im.k1, tiles);
    GRL_REQUIRE(im.slot >= 0 && (long long)im.slot + im.k1 - im.k0 <= n, "%s: image %d: slots %d + %d past the batch of %d",
                what, i, im.slot, im.k1 - im.k0, n);
    GRL_REQUIRE((long long)im.t * scale <= Hy && (long long)im.t * scale <= Wy,
                "%s: image %d: tile output %d x %d is bigger than the batch's %d x %d", what, i, im.t * scale, im.t * scale,
                Hy, Wy);
  }
  return blend(y, C, Hy, Wy, scale, images, m, false, (cudaStream_t)stream);
}

int grl_tile_finish(const GrlTileImage* images, int m, int C, int scale, void* stream) {
  const char* what = "tile_finish";
  int rc = check_list_args(m, images != nullptr, "image", what);
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(C >= 1 && C <= kTileMaxC, "%s: C = %d outside 1..%d", what, C, kTileMaxC);
  GRL_REQUIRE(scale >= 1, "%s: bad scale %d", what, scale);
  const bool u8 = m && images[0].out_u8;
  for (int i = 0; i < m; ++i) {
    rc = check_blend(images[i], i, scale, what);
    if (rc != GRL_OK) return rc;
    GRL_REQUIRE(!images[i].out_u8 == !u8, "%s: image %d: uint8 output %s, image 0's %s: one output kind per call", what,
                i, images[i].out_u8 ? "set" : "NULL", u8 ? "set" : "NULL");
  }
  return blend(nullptr, C, 0, 0, scale, images, m, true, (cudaStream_t)stream);
}

}  // extern "C"
