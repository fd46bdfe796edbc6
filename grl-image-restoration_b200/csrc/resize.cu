// resize.cu -- the SR dataset's online LR image (data/datasets/restoration_sr.py:127-141: imresize(modcrop(img_gt) / 255,
// 1 / scale)) for batches of float32 planes and lists of 8-bit images: MATLAB's bicubic downscale by 2, 3 or 4 with
// antialiasing (utils/matlab_functions.py:92-188), from the closed forms of grl_resize.h, bit for bit equal to the host
// copy grl_imresize_f32_host.
//
// One CTA per kResizeTH x kResizeTW output tile of one image, all channels in turn.  Per channel the H pass writes the
// float32 column sums of the tile's output rows over the s (kResizeTW - 1) + T input columns its W pass reads into shared
// memory; after a barrier the W pass reads its T taps from there.  A launch takes up to kResizePerLaunch images of any
// sizes: their records and first-tile numbers travel by value in the kernel parameters (grl_param_list.cuh), and a CTA
// finds its image with record_of.  No workspace, no host sync.
#include <vector>

#include "grl_common.cuh"
#include "grl_image_u8.h"
#include "grl_param_list.cuh"
#include "grl_resize.h"

namespace grl {

namespace {

constexpr int kResizePerLaunch = 64;
constexpr int kResizeTH = 16, kResizeTW = 32, kResizeThreads = 256;

struct ResizeRecord {
  const void* src;
  float* dst;
  int H, W;  // of the source image
};
struct ResizeStarts {
  int tile0[kResizePerLaunch + 1];  // image j's tiles are CTAs tile0[j] .. tile0[j + 1] - 1
};
struct ResizeTaps {
  float w[kResizeMaxTaps];
};
using ResizeRecords =
    ParamList<ResizeRecord, kResizePerLaunch, sizeof(ResizeStarts) + sizeof(ResizeTaps) + 2 * sizeof(int)>;
static_assert(kResizeThreads >= 256, "one thread per entry of the k / 255 table");

// (C, H, W) float32 planes
struct F32Img {
  const float* p;
  int H, W, C;
  static __device__ F32Img at(const void* p, int H, int W, int C, const float*) {
    return {static_cast<const float*>(p), H, W, C};
  }
  __device__ float operator()(int c, int y, int x) const { return p[((long long)c * H + y) * W + x]; }
};
// (H, W, C) uint8 pixels, k / 255 as to_tensor gives it, looked up in the CTA's table unit[k] = u8_unit(k)
struct U8Img {
  const uint8_t* p;
  int H, W, C;
  const float* unit;
  static __device__ U8Img at(const void* p, int H, int W, int C, const float* unit) {
    return {static_cast<const uint8_t*>(p), H, W, C, unit};
  }
  __device__ float operator()(int c, int y, int x) const { return unit[p[((long long)y * W + x) * C + c]]; }
};

__host__ __device__ int resize_tiles(int H, int W, int s) {
  const int h = (H + s - 1) / s, w = (W + s - 1) / s;
  return ((h + kResizeTH - 1) / kResizeTH) * ((w + kResizeTW - 1) / kResizeTW);
}

template <class Img, int S>
__global__ void __launch_bounds__(kResizeThreads) imresize_kernel(const ResizeRecords L, const ResizeStarts X,
                                                                   const ResizeTaps taps, int m, int C) {
  constexpr int T = resize_taps_of(S), c0 = resize_offset(S), kCols = S * (kResizeTW - 1) + T;
  __shared__ float t[kResizeTH][kCols];
  __shared__ float unit[256];
  if (threadIdx.x < 256) unit[threadIdx.x] = u8_unit(threadIdx.x);  // read by U8Img after the first barrier only
  const int j = record_of(X.tile0, m, blockIdx.x);
  const ResizeRecord& im = L.at[j];
  const int H = im.H, W = im.W, h = (H + S - 1) / S, w = (W + S - 1) / S;
  const int tiles_x = (w + kResizeTW - 1) / kResizeTW, tile = blockIdx.x - X.tile0[j];
  const int oy0 = tile / tiles_x * kResizeTH, ox0 = tile % tiles_x * kResizeTW;
  const int nh = min(kResizeTH, h - oy0), nw = min(kResizeTW, w - ox0), ncols = S * (nw - 1) + T;
  const Img img = Img::at(im.src, H, W, C, unit);
  __syncthreads();
  float* dst = im.dst;
  for (int c = 0; c < C; ++c) {
    for (int i = threadIdx.x; i < nh * ncols; i += kResizeThreads) {
      const int r = i / ncols, xl = i - r * ncols;
      const int x = resize_index(S * ox0 + c0 + xl, W), y0 = S * (oy0 + r) + c0;
      float v[T];
#pragma unroll
      for (int k = 0; k < T; ++k) v[k] = img(c, resize_index(y0 + k, H), x);
      t[r][xl] = resize_dot(taps.w, v, T);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nh * kResizeTW; i += kResizeThreads) {
      const int r = i / kResizeTW, ox = i - r * kResizeTW;
      if (ox < nw) dst[((long long)c * h + oy0 + r) * w + ox0 + ox] = resize_dot(taps.w, &t[r][S * ox], T);
    }
    __syncthreads();
  }
}

int check_resize_geometry(int H, int W, int C, int s, const char* what, int i) {
  GRL_REQUIRE(resize_fits(H, s) && resize_fits(W, s), "%s: image %d: %d x %d is too small for scale 1/%d: the symmetric "
              "padding needs (%d, %d) rows and (%d, %d) columns, more than the image has (the reference fails there too)",
              what, i, H, W, s, resize_geom(H, s).pad_s, resize_geom(H, s).pad_e, resize_geom(W, s).pad_s,
              resize_geom(W, s).pad_e);
  GRL_REQUIRE((long long)H * W * C <= 0x7fffffffLL, "%s: image %d: %d x %d x %d samples is too large", what, i, H, W, C);
  return GRL_OK;
}

int check_scale(int s, const char* what) {
  GRL_REQUIRE(s == 2 || s == 3 || s == 4, "%s: scale 1/%d, only 1/2, 1/3 and 1/4 are supported", what, s);
  return GRL_OK;
}

// Runs n images, image i's record from record(i).
template <class Img, int S, class Record>
int launch_resize(int n, int C, Record record, cudaStream_t st) {
  ResizeStarts X;
  ResizeTaps taps;
  resize_taps(S, taps.w);
  const auto add = [&](ResizeRecord& r, int, int i) {
    r = record(i);
    return (long long)resize_tiles(r.H, r.W, S);
  };
  return launch_list<ResizeRecords>(n, add, [&](const ResizeRecords& L, int, int m) -> int {
    long long total = 0;
    for (int j = 0; j < m; ++j) {
      X.tile0[j] = (int)total;
      total += resize_tiles(L.at[j].H, L.at[j].W, S);
    }
    GRL_REQUIRE(total <= 0x7fffffffLL, "imresize: %lld tiles in one launch", total);
    X.tile0[m] = (int)total;
    imresize_kernel<Img, S><<<(unsigned)total, kResizeThreads, 0, st>>>(L, X, taps, m, C);
    GRL_LAUNCH_CHECK("imresize_kernel");
    return GRL_OK;
  });
}

template <class Img, class Record>
int launch_resize(int n, int C, int s, Record record, cudaStream_t st) {
  if (s == 2) return launch_resize<Img, 2>(n, C, record, st);
  if (s == 3) return launch_resize<Img, 3>(n, C, record, st);
  return launch_resize<Img, 4>(n, C, record, st);
}

}  // namespace

}  // namespace grl

using namespace grl;

extern "C" {

int grl_imresize_taps_host(int n, int s, float* taps, int32_t* geometry) {
  int rc = check_scale(s, "imresize_taps_host");
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(taps && geometry, "imresize_taps_host: null argument");
  GRL_REQUIRE(n >= 1 && resize_fits(n, s), "imresize_taps_host: length %d is too small for scale 1/%d: the symmetric "
              "padding needs (%d, %d) samples (the reference fails there too)", n, s, resize_geom(n, s).pad_s,
              resize_geom(n, s).pad_e);
  const ResizeGeom g = resize_geom(n, s);
  resize_taps(s, taps);
  const int32_t v[5] = {g.T, g.c, g.out, g.pad_s, g.pad_e};
  for (int i = 0; i < 5; ++i) geometry[i] = v[i];
  return GRL_OK;
}

int grl_imresize_f32_host(const float* x, int B, int C, int H, int W, int s, float* y) {
  int rc = check_scale(s, "imresize_f32_host");
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(B >= 0 && C >= 1 && C <= 8, "imresize_f32_host: B = %d, C = %d (1 <= C <= 8)", B, C);
  GRL_REQUIRE((x && y) || B == 0, "imresize_f32_host: null argument");
  rc = check_resize_geometry(H, W, C, s, "imresize_f32_host", 0);
  if (rc != GRL_OK) return rc;
  const ResizeGeom gh = resize_geom(H, s), gw = resize_geom(W, s);
  const int h = gh.out, w = gw.out, T = gh.T;
  float taps[kResizeMaxTaps], v[kResizeMaxTaps];
  resize_taps(s, taps);
  std::vector<float> t((size_t)h * W);
  for (long long p = 0; p < (long long)B * C; ++p) {
    const float* src = x + p * H * W;
    float* dst = y + p * h * w;
    for (int oy = 0; oy < h; ++oy)
      for (int xx = 0; xx < W; ++xx) {
        for (int k = 0; k < T; ++k) v[k] = src[(long long)resize_index(s * oy + gh.c + k, H) * W + xx];
        t[(long long)oy * W + xx] = resize_dot(taps, v, T);
      }
    for (int oy = 0; oy < h; ++oy)
      for (int ox = 0; ox < w; ++ox) {
        for (int k = 0; k < T; ++k) v[k] = t[(long long)oy * W + resize_index(s * ox + gw.c + k, W)];
        dst[(long long)oy * w + ox] = resize_dot(taps, v, T);
      }
  }
  return GRL_OK;
}

int grl_imresize_f32(const float* x, int B, int C, int H, int W, int s, float* y, void* stream) {
  int rc = check_scale(s, "imresize_f32");
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(B >= 0 && C >= 1 && C <= 8, "imresize_f32: B = %d, C = %d (1 <= C <= 8)", B, C);
  GRL_REQUIRE((x && y) || B == 0, "imresize_f32: null argument");
  rc = check_resize_geometry(H, W, C, s, "imresize_f32", 0);
  if (rc != GRL_OK) return rc;
  const long long in = (long long)C * H * W, out = (long long)C * ((H + s - 1) / s) * ((W + s - 1) / s);
  return launch_resize<F32Img>(B, C, s, [&](int b) { return ResizeRecord{x + b * in, y + b * out, H, W}; },
                               (cudaStream_t)stream);
}

int grl_imresize_u8_list(const GrlImageRef* src, const GrlImageRef* dst, int n, int C, int s, void* stream) {
  int rc = check_scale(s, "imresize_u8_list");
  if (rc != GRL_OK) return rc;
  GRL_REQUIRE(C == 1 || C == 3, "imresize_u8_list: C = %d, an 8-bit image here is gray (C = 1) or RGB (C = 3)", C);
  rc = check_u8_pairs(
      src, dst, n, GRL_IMAGE_F32, [&](const GrlImageRef& a) { return make_int2((a.H + s - 1) / s, (a.W + s - 1) / s); },
      [&](const GrlImageRef& a, int i) { return check_resize_geometry(a.H, a.W, C, s, "imresize_u8_list", i); },
      "imresize_u8_list");
  if (rc != GRL_OK) return rc;
  return launch_resize<U8Img>(n, C, s, [&](int i) {
    return ResizeRecord{src[i].data, static_cast<float*>(dst[i].data), src[i].H, src[i].W};
  }, (cudaStream_t)stream);
}

}  // extern "C"
