// jpeg.cu -- the JPEG test command's degraded input (jpeg_compress, data/datasets/restoration_jpeg.py:62-79) for a list
// of 8-bit images: the pixels of a baseline encode at quality q followed by the default decode, bit for bit, from the
// closed forms of grl_jpeg.h.
//
// Two kernels over flattened indices of the whole list (at most kJpegPerLaunch images per launch; the descriptors travel
// by value in the kernel parameters, as in image_list.cu):
//   jpeg_blocks_kernel  one thread per coded 8 x 8 block of every component: loads its samples (clamp-to-edge; a chroma
//                       block converts and downsamples its 16 x 16 image pixels), then FDCT -> quantise -> dequantise ->
//                       IDCT.  Gray: the decoded block is the output.  Colour: Y goes to an (H, W) workspace plane, Cb
//                       and Cr to (h2, w2) ones.
//   jpeg_rgb_kernel     colour only, one thread per output pixel: fancy-upsampled Cb / Cr (4 neighbours of each plane)
//                       and Y -> RGB.
// The upsampler reads chroma samples of up to four blocks, so the split keeps every block's IDCT done once; a fused
// kernel would redo the halo blocks' DCTs.
#include "grl_common.cuh"
#include "grl_jpeg.h"

namespace grl {

namespace {

constexpr int kJpegPerLaunch = 80;  // 80 x 40 bytes of descriptors + the tables: 3.3 KB of the 4 KB of kernel parameters
constexpr int kBlockThreads = 128, kPixelThreads = 256;

struct JpegList {
  const uint8_t* src[kJpegPerLaunch];
  uint8_t* dst[kJpegPerLaunch];
  uint8_t* ws[kJpegPerLaunch];       // colour: Y (H, W), then Cb and Cr (h2, w2)
  int H[kJpegPerLaunch], W[kJpegPerLaunch];
  int block0[kJpegPerLaunch + 1];    // first block / pixel of image i in the launch's flat index; [m] = the total
  int pixel0[kJpegPerLaunch + 1];
  uint8_t qt[2][64];                 // luma, chroma; natural order
};
static_assert(sizeof(JpegList) + 2 * sizeof(int) <= 4096, "kernel parameters");

// The image of flat index t: the last i < m with first[i] <= t.
__device__ __forceinline__ int find_image(const int* first, int m, int t) {
  int lo = 0, hi = m - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

GRL_HD long long blocks_of(int H, int W, int C) {
  const JpegImage im{nullptr, H, W, C};
  long long n = (long long)jpeg_blocks_y(im, 0) * jpeg_blocks_x(im, 0);
  if (C == 3) n += 2LL * jpeg_blocks_y(im, 1) * jpeg_blocks_x(im, 1);
  return n;
}

GRL_HD long long workspace_of(int H, int W, int C) {
  return C == 3 ? (long long)H * W + 2LL * ((H + 1) >> 1) * ((W + 1) >> 1) : 0;
}

__global__ void __launch_bounds__(kBlockThreads) jpeg_blocks_kernel(const JpegList L, int m, int C) {
  const int t = blockIdx.x * kBlockThreads + threadIdx.x;
  if (t >= L.block0[m]) return;
  const int i = find_image(L.block0, m, t);
  const JpegImage im{L.src[i], L.H[i], L.W[i], C};
  int k = t - L.block0[i], comp = 0;
  const int nluma = jpeg_blocks_y(im, 0) * jpeg_blocks_x(im, 0);
  if (k >= nluma) {
    const int nc = jpeg_blocks_y(im, 1) * jpeg_blocks_x(im, 1);
    comp = 1 + (k - nluma) / nc;
    k = (k - nluma) % nc;
  }
  const int nx = jpeg_blocks_x(im, comp), by = k / nx, bx = k - by * nx;
  const long long plane = (long long)im.H * im.W, cplane = (long long)im.h2() * im.w2();
  uint8_t* out = C == 1 ? L.dst[i] : L.ws[i] + (comp ? plane + (comp - 1) * cplane : 0);
  jpeg_component_block(im, comp, by, bx, L.qt[comp ? 1 : 0], out, comp ? im.w2() : im.W);
}

__global__ void __launch_bounds__(kPixelThreads) jpeg_rgb_kernel(const JpegList L, int m) {
  const int p = blockIdx.x * kPixelThreads + threadIdx.x;
  if (p >= L.pixel0[m]) return;
  const int i = find_image(L.pixel0, m, p);
  const int H = L.H[i], W = L.W[i], k = p - L.pixel0[i], y = k / W, x = k - y * W;
  const long long plane = (long long)H * W, cplane = (long long)((H + 1) >> 1) * ((W + 1) >> 1);
  const uint8_t* ws = L.ws[i];
  uint8_t rgb[3];
  jpeg_decode_pixel(ws, ws + plane, ws + plane + cplane, H, W, y, x, rgb);
  uint8_t* d = L.dst[i] + 3LL * k;
  d[0] = rgb[0];
  d[1] = rgb[1];
  d[2] = rgb[2];
}

int check_jpeg(const GrlImageRef* src, const GrlImageRef* dst, int n, int C, int quality, const char* what) {
  GRL_REQUIRE(n >= 0 && ((src && dst) || n == 0), "%s: null image list (n = %d)", what, n);
  GRL_REQUIRE(C == 1 || C == 3, "%s: C = %d, a JPEG image is gray (C = 1) or RGB (C = 3)", what, C);
  GRL_REQUIRE(quality >= 1 && quality <= 100, "%s: quality %d outside 1..100", what, quality);
  for (int i = 0; i < n; ++i) {
    const GrlImageRef &s = src[i], &d = dst[i];
    GRL_REQUIRE(s.kind == GRL_IMAGE_U8 && d.kind == GRL_IMAGE_U8, "%s: image %d: kinds %d / %d, need GRL_IMAGE_U8", what,
                i, s.kind, d.kind);
    GRL_REQUIRE(s.data && d.data, "%s: image %d: null data", what, i);
    GRL_REQUIRE(s.H >= 1 && s.W >= 1 && s.H == d.H && s.W == d.W, "%s: image %d: sizes %d x %d -> %d x %d", what, i, s.H,
                s.W, d.H, d.W);
    GRL_REQUIRE((long long)s.H * s.W <= 0x7fffffffLL / 2, "%s: image %d: %d x %d pixels is too large", what, i, s.H, s.W);
  }
  return GRL_OK;
}

}  // namespace

}  // namespace grl

using namespace grl;

extern "C" {

size_t grl_jpeg_workspace(const GrlImageRef* images, int n, int C) {
  size_t bytes = 0;
  for (int i = 0; images && i < n; ++i) bytes += (size_t)workspace_of(images[i].H, images[i].W, C);
  return bytes;
}

int grl_jpeg_quant_tables_host(int quality, int32_t* tables) {
  GRL_REQUIRE(tables, "jpeg_quant_tables_host: null output");
  GRL_REQUIRE(quality >= 1 && quality <= 100, "jpeg_quant_tables_host: quality %d outside 1..100", quality);
  for (int t = 0; t < 2; ++t)
    for (int k = 0; k < 64; ++k) tables[t * 64 + k] = jpeg_quant(quality, t, k);
  return GRL_OK;
}

int grl_jpeg_roundtrip_host(const uint8_t* src, int H, int W, int C, int quality, uint8_t* dst) {
  GRL_REQUIRE(src && dst, "jpeg_roundtrip_host: null argument");
  GRL_REQUIRE(H >= 1 && W >= 1 && (C == 1 || C == 3), "jpeg_roundtrip_host: bad shape %d x %d x %d", H, W, C);
  GRL_REQUIRE(quality >= 1 && quality <= 100, "jpeg_roundtrip_host: quality %d outside 1..100", quality);
  uint8_t qt[2][64];
  for (int t = 0; t < 2; ++t)
    for (int k = 0; k < 64; ++k) qt[t][k] = (uint8_t)jpeg_quant(quality, t, k);
  const JpegImage im{src, H, W, C};
  const long long plane = (long long)H * W, cplane = (long long)im.h2() * im.w2();
  uint8_t* ws = C == 3 ? new uint8_t[plane + 2 * cplane] : nullptr;
  for (int comp = 0; comp < (C == 3 ? 3 : 1); ++comp) {
    uint8_t* out = C == 1 ? dst : ws + (comp ? plane + (comp - 1) * cplane : 0);
    for (int by = 0; by < jpeg_blocks_y(im, comp); ++by)
      for (int bx = 0; bx < jpeg_blocks_x(im, comp); ++bx)
        jpeg_component_block(im, comp, by, bx, qt[comp ? 1 : 0], out, comp ? im.w2() : W);
  }
  if (C == 3) {
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x)
        jpeg_decode_pixel(ws, ws + plane, ws + plane + cplane, H, W, y, x, dst + 3 * ((long long)y * W + x));
    delete[] ws;
  }
  return GRL_OK;
}

int grl_jpeg_roundtrip_u8(const GrlImageRef* src, const GrlImageRef* dst, int n, int C, int quality, void* workspace,
                          size_t workspace_bytes, void* stream) {
  const int rc = check_jpeg(src, dst, n, C, quality, "jpeg_roundtrip_u8");
  if (rc != GRL_OK) return rc;
  const size_t need = grl_jpeg_workspace(src, n, C);
  GRL_REQUIRE(workspace || need == 0, "jpeg_roundtrip_u8: null workspace");
  if (workspace_bytes < need)
    return fail(GRL_ERR_WORKSPACE, "jpeg_roundtrip_u8: workspace of %zu bytes, need %zu", workspace_bytes, need);
  JpegList L;
  for (int t = 0; t < 2; ++t)
    for (int k = 0; k < 64; ++k) L.qt[t][k] = (uint8_t)jpeg_quant(quality, t, k);
  const cudaStream_t st = (cudaStream_t)stream;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  for (int i0 = 0; i0 < n;) {
    // A launch takes images while its flat block and pixel counts fit an int.
    int m = 0;
    long long blocks = 0, pixels = 0;
    while (i0 + m < n && m < kJpegPerLaunch) {
      const GrlImageRef& s = src[i0 + m];
      const long long b = blocks_of(s.H, s.W, C), p = (long long)s.H * s.W;
      if (m && (blocks + b > 0x7fffffffLL || pixels + p > 0x7fffffffLL)) break;
      L.src[m] = static_cast<const uint8_t*>(s.data);
      L.dst[m] = static_cast<uint8_t*>(dst[i0 + m].data);
      L.ws[m] = ws;
      L.H[m] = s.H;
      L.W[m] = s.W;
      L.block0[m] = (int)blocks;
      L.pixel0[m] = (int)pixels;
      ws += workspace_of(s.H, s.W, C);
      blocks += b;
      pixels += p;
      ++m;
    }
    L.block0[m] = (int)blocks;
    L.pixel0[m] = (int)pixels;
    jpeg_blocks_kernel<<<ceil_div(blocks, kBlockThreads), kBlockThreads, 0, st>>>(L, m, C);
    GRL_LAUNCH_CHECK("jpeg_blocks_kernel");
    if (C == 3) {
      jpeg_rgb_kernel<<<ceil_div(pixels, kPixelThreads), kPixelThreads, 0, st>>>(L, m);
      GRL_LAUNCH_CHECK("jpeg_rgb_kernel");
    }
    i0 += m;
  }
  return GRL_OK;
}

}  // extern "C"
