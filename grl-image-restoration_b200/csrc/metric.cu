// metric.cu -- the validation step's PSNR on the device in one pass (engines/base.py:255-268, utils/utils_image.py:8-11
// shave, :30-33 tensor_round, :43-80 rgb2ycbcr; utils/metrics/psnr.py:44-48).
//
// restored / target are (B, C, H, W) fp32 planes or (B, H, W, C) 8-bit pixels: every kernel is a template on the pixel
// reader of grl_image_u8.h, the rest of it is shared.  fp32 planes are rounded to the 8-bit grid (clamp to [0, 1], x255,
// round half to even like torch.round), `border` pixels are shaved on every side, and the squared error is accumulated
// EXACTLY as an integer (a rounded pixel is k/255; (k1 - k2)^2 <= 65025): the per-image sums are 64-bit integer atomics,
// so the result is independent of the block schedule.  C == 3 additionally accumulates the error of the luma of MATLAB's
// rgb2ycbcr (coefficients 65.481, 128.553, 24.966, offset 16, rounded to 8 bit).  HBM-bound: 2 x 4 bytes read per
// element from fp32 planes, 2 x 1 from 8-bit pixels.
// PSNR-B and SSIM (RGB and luma, float64 on the same 8-bit integers) follow below.
#include <algorithm>
#include <vector>

#include "grl_common.cuh"
#include "grl_image_u8.h"
#include "grl_ssim.h"

namespace grl {

// y = round(65.481/255 * R + 128.553/255 * G + 24.966/255 * B + 16) with R, G, B on the 0..255 grid
// (metrics.rgb_to_y: (img * 255) @ (coeff / 255) + 16, rounded)
GRL_HD float luma8(float r, float g, float b) {
  float acc = r * (65.481f / 255.0f);
  acc = fmaf(g, 128.553f / 255.0f, acc);
  acc = fmaf(b, 24.966f / 255.0f, acc);
  return rintf(acc + 16.0f);
}

template <class Img>
__global__ void psnr_sse_kernel(Img a, Img b, int C, int H, int W, int border,
                                unsigned long long* __restrict__ sse /* (B, 2): rgb, y */) {
  const int img = blockIdx.y;
  const int h = H - 2 * border, w = W - 2 * border;
  const long long n = (long long)h * w;
  const Img pa = a.img(img), pb = b.img(img);
  unsigned long long s_rgb = 0, s_y = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / w), x = (int)(i - (long long)y * w);
    const long long off = (long long)(y + border) * W + (x + border);
    float ra[3], rb[3];
    for (int c = 0; c < C; ++c) {
      const float va = pa(c, off), vb = pb(c, off);
      if (c < 3) ra[c] = va, rb[c] = vb;
      const int d = (int)va - (int)vb;
      s_rgb += (unsigned)(d * d);
    }
    if (C == 3) {
      const int d = (int)luma8(ra[0], ra[1], ra[2]) - (int)luma8(rb[0], rb[1], rb[2]);
      s_y += (unsigned)(d * d);
    }
  }
  // block reduction (integers: order-independent)
  __shared__ unsigned long long sh[2][32];
  for (int o = 16; o > 0; o >>= 1) {
    s_rgb += __shfl_xor_sync(0xffffffffu, s_rgb, o);
    s_y += __shfl_xor_sync(0xffffffffu, s_y, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sh[0][warp] = s_rgb, sh[1][warp] = s_y;
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    s_rgb = lane < nw ? sh[0][lane] : 0;
    s_y = lane < nw ? sh[1][lane] : 0;
    for (int o = 16; o > 0; o >>= 1) {
      s_rgb += __shfl_xor_sync(0xffffffffu, s_rgb, o);
      s_y += __shfl_xor_sync(0xffffffffu, s_y, o);
    }
    if (lane == 0) {
      atomicAdd(&sse[2 * img], s_rgb);
      atomicAdd(&sse[2 * img + 1], s_y);
    }
  }
}

__global__ void psnr_finalize_kernel(const unsigned long long* __restrict__ sse, int B, int C, long long n_pix,
                                     float* __restrict__ psnr_rgb, float* __restrict__ psnr_y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  // mean((a - b)^2) with a, b = k / 255
  const double m_rgb = (double)sse[2 * i] / (65025.0 * (double)n_pix * (double)C);
  psnr_rgb[i] = (float)(-10.0 * log10(m_rgb));
  if (psnr_y) psnr_y[i] = (C == 3) ? (float)(-10.0 * log10((double)sse[2 * i + 1] / (65025.0 * (double)n_pix))) : psnr_rgb[i];
}

// ---- PSNR-B (utils/metrics/psnrb.py:22-115) -------------------------------------------------------------------------
// Per image and per channel (the C channels, then the luma of luma8 for C == 3), five exact integer sums of squared 8-bit
// differences: the error against the target, and on the RESTORED image alone the differences of horizontal neighbours
// (x, x + 1) at block boundaries x = 7, 15, ... < W - 1 and elsewhere, and the same for vertical neighbours.
constexpr int kPsnrbSets = 4, kPsnrbSums = 5;  // sse, horizontal boundary, horizontal other, vertical boundary, vertical other

template <class Img>
__global__ void psnrb_sums_kernel(Img a, Img b, int C, int H, int W, unsigned long long* __restrict__ sums /* (B, 4, 5) */) {
  const int img = blockIdx.y;
  const long long n = (long long)H * W;
  const Img pa = a.img(img), pb = b.img(img);
  unsigned long long s[kPsnrbSets][kPsnrbSums] = {};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / W), x = (int)(i - (long long)y * W);
    const bool right = x < W - 1, down = y < H - 1;
    const bool hb = (x & 7) == 7, vb_ = (y & 7) == 7;  // on a block boundary
    float va[3] = {0.f, 0.f, 0.f}, vb[3] = {0.f, 0.f, 0.f}, vr[3] = {0.f, 0.f, 0.f}, vd[3] = {0.f, 0.f, 0.f};
    int d[4], e[4], f[4];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (c < C) {
        va[c] = pa(c, i), vb[c] = pb(c, i);
        if (right) vr[c] = pa(c, i + 1);
        if (down) vd[c] = pa(c, i + W);
      }
      d[c] = (int)va[c] - (int)vb[c], e[c] = right ? (int)va[c] - (int)vr[c] : 0, f[c] = down ? (int)va[c] - (int)vd[c] : 0;
    }
    d[3] = e[3] = f[3] = 0;
    if (C == 3) {
      const int ya = (int)luma8(va[0], va[1], va[2]);
      d[3] = ya - (int)luma8(vb[0], vb[1], vb[2]);
      if (right) e[3] = ya - (int)luma8(vr[0], vr[1], vr[2]);
      if (down) f[3] = ya - (int)luma8(vd[0], vd[1], vd[2]);
    }
#pragma unroll
    for (int c = 0; c < kPsnrbSets; ++c) {  // channels past C and the luma of C == 1 stay 0
      const unsigned e2 = (unsigned)(e[c] * e[c]), f2 = (unsigned)(f[c] * f[c]);
      s[c][0] += (unsigned)(d[c] * d[c]);
      s[c][1] += hb ? e2 : 0u;
      s[c][2] += hb ? 0u : e2;
      s[c][3] += vb_ ? f2 : 0u;
      s[c][4] += vb_ ? 0u : f2;
    }
  }
  __shared__ unsigned long long sh[kPsnrbSets * kPsnrbSums][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < kPsnrbSets * kPsnrbSums; ++k) {
    unsigned long long v = s[k / kPsnrbSums][k % kPsnrbSums];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sh[k][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < kPsnrbSets * kPsnrbSums) {
    unsigned long long v = 0;
    for (int w = 0; w < nw; ++w) v += sh[threadIdx.x][w];
    if (v) atomicAdd(&sums[(long long)img * kPsnrbSets * kPsnrbSums + threadIdx.x], v);
  }
}

// psnrb (psnrb.py:104-115) from the sums, in float64.  The normalisers are the reference's formulas (psnrb.py:85-95), not
// the number of summed positions: n_boundary_horiz = H * (W // 8 - 1) although arange(7, W - 1, 8) may hold one column
// more, and the non-boundary counts are the rest of H * (W - 1).  bef = 0 where boundary <= non-boundary.  Every channel
// gives 10 log10(1 / (mse + bef)); the result is their mean in dB.
__global__ void psnrb_finalize_kernel(const unsigned long long* __restrict__ sums, int B, int C, int H, int W,
                                      double* __restrict__ psnrb_rgb, double* __restrict__ psnrb_y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  const double nbh = (double)H * (W / 8 - 1), nbv = (double)W * (H / 8 - 1);
  const double nnh = (double)H * (W - 1) - nbh, nnv = (double)W * (H - 1) - nbv;
  const double scaler = log2(8.0) / log2((double)min(H, W));
  double v[kPsnrbSets];
  for (int c = 0; c < kPsnrbSets; ++c) {
    const unsigned long long* s = sums + ((long long)i * kPsnrbSets + c) * kPsnrbSums;
    const double mse = (double)s[0] / (65025.0 * H * W);
    const double bd = ((double)s[1] + (double)s[3]) / 65025.0 / (nbh + nbv);
    const double nd = ((double)s[2] + (double)s[4]) / 65025.0 / (nnh + nnv);
    const double bef = bd <= nd ? 0.0 : scaler * (bd - nd);
    v[c] = 10.0 * log10(1.0 / (mse + bef));
  }
  double t = 0.0;
  for (int c = 0; c < C; ++c) t += v[c];
  psnrb_rgb[i] = t / C;
  if (psnrb_y) psnrb_y[i] = C == 3 ? v[3] : psnrb_rgb[i];
}

// ---- SSIM (utils/metrics/ssim.py:17-85; the closed form is grl_ssim.h) -----------------------------------------------
// One CTA owns a 32 x 16 tile of output pixels of one image and produces every plane of it: the C channels and, for
// C == 3, the luma of luma8.  The 8-bit integers of the tile and its 5-pixel halo are staged once (42 x 26 per plane and
// image, 0 outside the image).  Per plane: the horizontal 11-tap sums of a, b, a^2, b^2, a b go to shared memory (one lane
// per staged row and four adjacent columns per thread, so a staged value is converted once for four outputs), then each
// thread takes the vertical sums and the map values of four rows of one column.  The tile's map values are summed in a
// fixed order into one float64 partial per (image, {channels, luma}, tile); ssim_finalize_kernel sums the partials of an
// image in a fixed order.  No atomics: the result depends neither on the schedule nor on the batch an image is part of.
// On paper the kernel is bound by the float64 pipe, not by HBM: about 145 DFMA per plane value against 24 bytes per pixel.
constexpr int kSsimTW = 32, kSsimTH = 16, kSsimThreads = 128;
constexpr int kSsimRows = kSsimTH + 2 * kSsimHalo;  // 26 staged rows
constexpr int kSsimCols = kSsimTW + 2 * kSsimHalo;  // 42 staged columns
constexpr int kSsimRowBytes = 44;                   // ... in rows of whole 32-bit words (the last two bytes hold 0)
constexpr int kSsimHStride = kSsimTW + 1;           // row stride of the horizontal sums: the lanes of a warp write one column
static_assert(kSsimRows <= 32 && kSsimTW == 32 && kSsimThreads == 4 * 32 && kSsimTH == 4 * 4, "thread mapping of ssim_tile_kernel");

// exact double of an integer 0 <= k < 2^32 without the conversion pipe: 2^52 + k is exact, minus 2^52
__device__ __forceinline__ double ssim_u2d(unsigned k) { return __hiloint2double(0x43300000, (int)k) - 4503599627370496.0; }

template <class Img>
__global__ void __launch_bounds__(kSsimThreads)
ssim_tile_kernel(Img a, Img b, int C, int H, int W, int border,
                 double* __restrict__ partial /* (B, 2, tiles) */, double* __restrict__ map_rgb, double* __restrict__ map_y) {
  __shared__ __align__(16) unsigned char sk[2][4][kSsimRows][kSsimRowBytes];
  __shared__ double hs[5][kSsimRows][kSsimHStride];
  __shared__ double red[2][kSsimThreads / 32];
  const int img = blockIdx.z, h = H - 2 * border, w = W - 2 * border;
  const int x0 = blockIdx.x * kSsimTW, y0 = blockIdx.y * kSsimTH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n = (long long)h * w;
  const Img pa = a.img(img), pb = b.img(img);

  // tensor_round + shave + luma, staged as bytes
  for (int i = threadIdx.x; i < kSsimRows * kSsimRowBytes; i += kSsimThreads) {
    const int r = i / kSsimRowBytes, c = i - r * kSsimRowBytes;
    const int y = y0 - kSsimHalo + r, x = x0 - kSsimHalo + c;
    const bool in = c < kSsimCols && y >= 0 && y < h && x >= 0 && x < w;
    const long long off = in ? (long long)(y + border) * W + (x + border) : 0;
    float va[3] = {0.f, 0.f, 0.f}, vb[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
      if (ch < C) {
        if (in) va[ch] = pa(ch, off), vb[ch] = pb(ch, off);
        sk[0][ch][r][c] = (unsigned char)va[ch], sk[1][ch][r][c] = (unsigned char)vb[ch];
      }
    if (C == 3) {
      sk[0][3][r][c] = in ? (unsigned char)luma8(va[0], va[1], va[2]) : 0;
      sk[1][3][r][c] = in ? (unsigned char)luma8(vb[0], vb[1], vb[2]) : 0;
    }
  }

  double sum_rgb = 0.0, sum_y = 0.0;
  const int planes = C == 3 ? 4 : C;
  for (int p = 0; p < planes; ++p) {
    __syncthreads();  // the staged bytes are written (p == 0); the previous plane's vertical pass has read hs
    if (lane < kSsimRows) {
      for (int xg = warp; xg < kSsimTW / 4; xg += kSsimThreads / 32) {  // outputs 4 xg .. 4 xg + 3 of staged row `lane`
        const unsigned* qa = reinterpret_cast<const unsigned*>(&sk[0][p][lane][4 * xg]);
        const unsigned* qb = reinterpret_cast<const unsigned*>(&sk[1][p][lane][4 * xg]);
        unsigned ua[4], ub[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) ua[j] = qa[j], ub[j] = qb[j];
        double va[14], vb[14];
#pragma unroll
        for (int j = 0; j < 14; ++j) {
          va[j] = ssim_u2d((ua[j >> 2] >> (8 * (j & 3))) & 0xffu);
          vb[j] = ssim_u2d((ub[j >> 2] >> (8 * (j & 3))) & 0xffu);
        }
#pragma unroll
        for (int q = 0; q < 5; ++q) {
          double v[14];
#pragma unroll
          for (int j = 0; j < 14; ++j)  // integers below 2^16: the products are exact
            v[j] = q == 0 ? va[j] : q == 1 ? vb[j] : q == 2 ? __dmul_rn(va[j], va[j]) : q == 3 ? __dmul_rn(vb[j], vb[j]) : __dmul_rn(va[j], vb[j]);
          double acc[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
          for (int t = 0; t < kSsimTaps; ++t)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[i] = dfma_rn(ssim_tap(t), v[i + t], acc[i]);
#pragma unroll
          for (int i = 0; i < 4; ++i) hs[q][lane][4 * xg + i] = acc[i];
        }
      }
    }
    __syncthreads();
    double s[5][4];  // column `lane`, rows 4 warp .. 4 warp + 3 of the tile
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      double r[14];
#pragma unroll
      for (int j = 0; j < 14; ++j) r[j] = hs[q][4 * warp + j][lane];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        double acc = 0.0;
#pragma unroll
        for (int t = 0; t < kSsimTaps; ++t) acc = dfma_rn(ssim_tap(t), r[i + t], acc);
        s[q][i] = acc;
      }
    }
    const int x = x0 + lane;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int y = y0 + 4 * warp + i;
      if (x < w && y < h) {
        const double m = ssim_map_value(s[0][i], s[1][i], s[2][i], s[3][i], s[4][i]);
        if (p < C) {
          sum_rgb += m;
          if (map_rgb) map_rgb[((long long)img * C + p) * n + (long long)y * w + x] = m;
        } else {
          sum_y += m;
          if (map_y) map_y[(long long)img * n + (long long)y * w + x] = m;
        }
      }
    }
  }
  // fixed-shape reduction: xor tree in the warp, then the four warps in order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum_rgb += __shfl_xor_sync(0xffffffffu, sum_rgb, o);
    sum_y += __shfl_xor_sync(0xffffffffu, sum_y, o);
  }
  if (lane == 0) red[0][warp] = sum_rgb, red[1][warp] = sum_y;
  __syncthreads();
  if (threadIdx.x < 2) {
    double t = 0.0;
    for (int k = 0; k < kSsimThreads / 32; ++k) t += red[threadIdx.x][k];
    const long long tiles = (long long)gridDim.x * gridDim.y, tile = (long long)blockIdx.y * gridDim.x + blockIdx.x;
    partial[((long long)img * 2 + threadIdx.x) * tiles + tile] = t;
  }
}

// Block (g, img): the mean of the map over the channels (g == 0) or over the luma plane (g == 1; for C != 3 the channels
// again, so ssim_y is a copy of ssim_rgb).  Thread t sums partials t, t + 256, ... in order, then a fixed tree.
__global__ void __launch_bounds__(256)
ssim_finalize_kernel(const double* __restrict__ partial, int C, long long tiles, long long n_pix, double* __restrict__ ssim_rgb,
                     double* __restrict__ ssim_y) {
  __shared__ double red[8];
  const int g = blockIdx.x, img = blockIdx.y;
  double* out = g == 0 ? ssim_rgb : ssim_y;
  if (!out) return;
  const bool luma = g == 1 && C == 3;
  const double* src = partial + ((long long)img * 2 + (luma ? 1 : 0)) * tiles;
  double t = 0.0;
  for (long long k = threadIdx.x; k < tiles; k += blockDim.x) t += src[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int k = 0; k < 8; ++k) v += red[k];
    out[img] = v / ((double)n_pix * (luma ? 1 : C));
  }
}

static long long ssim_tiles(int H, int W, int border) {
  return (long long)ceil_div(W - 2 * border, kSsimTW) * ceil_div(H - 2 * border, kSsimTH);
}

static bool ssim_shape_ok(int B, int C, int H, int W, int border) {
  return B >= 0 && (C == 1 || C == 3) && border >= 0 && H > 0 && W > 0 && 2LL * border < std::min(H, W);
}

#define GRL_SSIM_SHAPE(B, C, H, W, border)                                                                                     \
  do {                                                                                                                         \
    GRL_REQUIRE(C == 1 || C == 3, "ssim: needs C == 1 or 3, got %d", C);                                                       \
    GRL_REQUIRE(B >= 0 && border >= 0 && H > 0 && W > 0, "ssim: bad shape (%d,%d,%d,%d) border %d", B, C, H, W, border);       \
    GRL_REQUIRE(2LL * border < std::min(H, W), "ssim: border %d leaves no pixel of a %d x %d image", border, H, W);            \
  } while (0)

// The launches behind grl_psnr_f32 / grl_psnr_u8 and their siblings; a and b are the pixel readers of the two images.
template <class Img>
int psnr_run(Img a, Img b, int B, int C, int H, int W, int border, void* workspace, size_t workspace_bytes, float* psnr_rgb,
             float* psnr_y, void* stream) {
  GRL_REQUIRE(a.p && b.p && psnr_rgb, "psnr: null argument");
  GRL_REQUIRE(workspace && workspace_bytes >= sizeof(unsigned long long) * 2 * (size_t)(B > 0 ? B : 0),
              "psnr: workspace %zu bytes < %zu", workspace_bytes, sizeof(unsigned long long) * 2 * (size_t)(B > 0 ? B : 0));
  GRL_REQUIRE(B >= 0 && C >= 1 && C <= 4 && H > 2 * border && W > 2 * border && border >= 0, "psnr: bad shape (%d,%d,%d,%d) border %d",
              B, C, H, W, border);
  if (B == 0) return GRL_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* sse = (unsigned long long*)workspace;
  GRL_CUDA(cudaMemsetAsync(sse, 0, sizeof(unsigned long long) * 2 * (size_t)B, st));
  const long long n = (long long)(H - 2 * border) * (W - 2 * border);
  const int threads = 256;
  const int bx = (int)std::min<long long>((n + threads * 4 - 1) / (threads * 4), 592);  // ~4 CTAs per SM per image at most
  psnr_sse_kernel<<<dim3((unsigned)std::max(bx, 1), (unsigned)B), threads, 0, st>>>(a, b, C, H, W, border, sse);
  GRL_LAUNCH_CHECK("psnr_sse_kernel");
  psnr_finalize_kernel<<<(B + 127) / 128, 128, 0, st>>>(sse, B, C, n, psnr_rgb, psnr_y);
  GRL_LAUNCH_CHECK("psnr_finalize_kernel");
  return GRL_OK;
}

template <class Img>
int psnrb_run(Img a, Img b, int B, int C, int H, int W, void* workspace, size_t workspace_bytes, double* psnrb_rgb,
              double* psnrb_y, void* stream) {
  GRL_REQUIRE(a.p && b.p && psnrb_rgb, "psnrb: null argument");
  GRL_REQUIRE(workspace && workspace_bytes >= grl_psnrb_workspace(B), "psnrb: workspace %zu bytes < %zu", workspace_bytes,
              grl_psnrb_workspace(B));
  GRL_REQUIRE(B >= 0 && (C == 1 || C == 3), "psnrb: needs C == 1 or 3, got %d", C);
  GRL_REQUIRE(H >= 16 && W >= 16, "psnrb: needs at least 16 x 16 pixels (the blocking-effect factor divides 0 by 0 below), got %d x %d",
              H, W);
  if (B == 0) return GRL_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* sums = (unsigned long long*)workspace;
  GRL_CUDA(cudaMemsetAsync(sums, 0, grl_psnrb_workspace(B), st));
  const long long n = (long long)H * W;
  const int threads = 256;
  const int bx = (int)std::min<long long>((n + threads * 4 - 1) / (threads * 4), 592);
  psnrb_sums_kernel<<<dim3((unsigned)std::max(bx, 1), (unsigned)B), threads, 0, st>>>(a, b, C, H, W, sums);
  GRL_LAUNCH_CHECK("psnrb_sums_kernel");
  psnrb_finalize_kernel<<<(B + 127) / 128, 128, 0, st>>>(sums, B, C, H, W, psnrb_rgb, psnrb_y);
  GRL_LAUNCH_CHECK("psnrb_finalize_kernel");
  return GRL_OK;
}

template <class Img>
int ssim_run(Img a, Img b, int B, int C, int H, int W, int border, void* workspace, size_t workspace_bytes, double* ssim_rgb,
             double* ssim_y, double* map_rgb, double* map_y, void* stream) {
  GRL_REQUIRE(a.p && b.p && ssim_rgb, "ssim: null argument");
  GRL_SSIM_SHAPE(B, C, H, W, border);
  if (B == 0) return GRL_OK;
  GRL_REQUIRE(workspace && workspace_bytes >= grl_ssim_workspace(B, C, H, W, border), "ssim: workspace %zu bytes < %zu",
              workspace_bytes, grl_ssim_workspace(B, C, H, W, border));
  const cudaStream_t st = (cudaStream_t)stream;
  const int h = H - 2 * border, w = W - 2 * border;
  const int gx = ceil_div(w, kSsimTW), gy = ceil_div(h, kSsimTH);
  GRL_REQUIRE(gy <= 65535 && B <= 65535, "ssim: %d tile rows / %d images exceed the grid", gy, B);
  ssim_tile_kernel<<<dim3((unsigned)gx, (unsigned)gy, (unsigned)B), kSsimThreads, 0, st>>>(a, b, C, H, W, border,
                                                                                         (double*)workspace, map_rgb, map_y);
  GRL_LAUNCH_CHECK("ssim_tile_kernel");
  ssim_finalize_kernel<<<dim3(2, (unsigned)B), 256, 0, st>>>((const double*)workspace, C, (long long)gx * gy, (long long)h * w, ssim_rgb, ssim_y);
  GRL_LAUNCH_CHECK("ssim_finalize_kernel");
  return GRL_OK;
}

static F32Planes f32_planes(const float* p, int C, int H, int W) { return {p, (long long)H * W, C}; }
static U8Pixels u8_pixels(const uint8_t* p, int H, int W, int C) { return {p, (long long)H * W, C}; }

}  // namespace grl

using namespace grl;

extern "C" {

int grl_psnr_f32(const float* restored, const float* target, int B, int C, int H, int W, int border, void* workspace,
                 size_t workspace_bytes, float* psnr_rgb, float* psnr_y, void* stream) {
  return psnr_run(f32_planes(restored, C, H, W), f32_planes(target, C, H, W), B, C, H, W, border, workspace, workspace_bytes, psnr_rgb,
                  psnr_y, stream);
}

int grl_psnr_u8(const uint8_t* restored, const uint8_t* target, int B, int H, int W, int C, int border, void* workspace,
                size_t workspace_bytes, float* psnr_rgb, float* psnr_y, void* stream) {
  return psnr_run(u8_pixels(restored, H, W, C), u8_pixels(target, H, W, C), B, C, H, W, border, workspace, workspace_bytes, psnr_rgb,
                  psnr_y, stream);
}

size_t grl_psnrb_workspace(int B) { return sizeof(unsigned long long) * kPsnrbSets * kPsnrbSums * (size_t)(B > 0 ? B : 0); }

int grl_psnrb_f32(const float* restored, const float* target, int B, int C, int H, int W, void* workspace,
                  size_t workspace_bytes, double* psnrb_rgb, double* psnrb_y, void* stream) {
  return psnrb_run(f32_planes(restored, C, H, W), f32_planes(target, C, H, W), B, C, H, W, workspace, workspace_bytes, psnrb_rgb,
                   psnrb_y, stream);
}

int grl_psnrb_u8(const uint8_t* restored, const uint8_t* target, int B, int H, int W, int C, void* workspace,
                 size_t workspace_bytes, double* psnrb_rgb, double* psnrb_y, void* stream) {
  return psnrb_run(u8_pixels(restored, H, W, C), u8_pixels(target, H, W, C), B, C, H, W, workspace, workspace_bytes, psnrb_rgb,
                   psnrb_y, stream);
}

size_t grl_ssim_workspace(int B, int C, int H, int W, int border) {
  if (!ssim_shape_ok(B, C, H, W, border)) return 0;
  return sizeof(double) * 2 * (size_t)B * (size_t)ssim_tiles(H, W, border);
}

int grl_ssim_f32(const float* restored, const float* target, int B, int C, int H, int W, int border, void* workspace,
                 size_t workspace_bytes, double* ssim_rgb, double* ssim_y, double* map_rgb, double* map_y, void* stream) {
  return ssim_run(f32_planes(restored, C, H, W), f32_planes(target, C, H, W), B, C, H, W, border, workspace, workspace_bytes, ssim_rgb,
                  ssim_y, map_rgb, map_y, stream);
}

int grl_ssim_u8(const uint8_t* restored, const uint8_t* target, int B, int H, int W, int C, int border, void* workspace,
                size_t workspace_bytes, double* ssim_rgb, double* ssim_y, double* map_rgb, double* map_y, void* stream) {
  return ssim_run(u8_pixels(restored, H, W, C), u8_pixels(target, H, W, C), B, C, H, W, border, workspace, workspace_bytes, ssim_rgb,
                  ssim_y, map_rgb, map_y, stream);
}

int grl_ssim_taps_host(double* taps11) {
  GRL_REQUIRE(taps11, "ssim_taps_host: null output");
  for (int i = 0; i < kSsimTaps; ++i) taps11[i] = ssim_tap(i);
  return GRL_OK;
}

// The same computation on the CPU (HOST pointers): the scores and, when asked for, the maps.  Scratch is host memory.
int grl_ssim_host(const float* restored, const float* target, int B, int C, int H, int W, int border, double* ssim_rgb,
                  double* ssim_y, double* map_rgb, double* map_y) {
  GRL_REQUIRE(restored && target && ssim_rgb, "ssim_host: null argument");
  GRL_SSIM_SHAPE(B, C, H, W, border);
  const int h = H - 2 * border, w = W - 2 * border, planes = C == 3 ? 4 : C;
  const size_t n = (size_t)h * w, plane = (size_t)H * W;
  std::vector<double> ka(n), kb(n), src(n), hsum(n), sums[5];
  for (auto& s : sums) s.resize(n);
  for (int img = 0; img < B; ++img) {
    const float* pa = restored + (size_t)img * C * plane;
    const float* pb = target + (size_t)img * C * plane;
    double tot_rgb = 0.0, tot_y = 0.0;
    for (int p = 0; p < planes; ++p) {
      for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
          const size_t off = (size_t)(y + border) * W + (x + border);
          if (p < C) {
            ka[(size_t)y * w + x] = round8(pa[p * plane + off]), kb[(size_t)y * w + x] = round8(pb[p * plane + off]);
          } else {
            ka[(size_t)y * w + x] = luma8(round8(pa[off]), round8(pa[plane + off]), round8(pa[2 * plane + off]));
            kb[(size_t)y * w + x] = luma8(round8(pb[off]), round8(pb[plane + off]), round8(pb[2 * plane + off]));
          }
        }
      for (int q = 0; q < 5; ++q) {
        for (size_t i = 0; i < n; ++i)
          src[i] = q == 0 ? ka[i] : q == 1 ? kb[i] : q == 2 ? ka[i] * ka[i] : q == 3 ? kb[i] * kb[i] : ka[i] * kb[i];
        for (int y = 0; y < h; ++y)
          for (int x = 0; x < w; ++x) {
            double acc = 0.0;
            for (int t = 0; t < kSsimTaps; ++t) {
              const int xx = x - kSsimHalo + t;
              acc = dfma_rn(ssim_tap(t), xx >= 0 && xx < w ? src[(size_t)y * w + xx] : 0.0, acc);
            }
            hsum[(size_t)y * w + x] = acc;
          }
        for (int y = 0; y < h; ++y)
          for (int x = 0; x < w; ++x) {
            double acc = 0.0;
            for (int t = 0; t < kSsimTaps; ++t) {
              const int yy = y - kSsimHalo + t;
              acc = dfma_rn(ssim_tap(t), yy >= 0 && yy < h ? hsum[(size_t)yy * w + x] : 0.0, acc);
            }
            sums[q][(size_t)y * w + x] = acc;
          }
      }
      for (size_t i = 0; i < n; ++i) {
        const double m = ssim_map_value(sums[0][i], sums[1][i], sums[2][i], sums[3][i], sums[4][i]);
        if (p < C) {
          tot_rgb += m;
          if (map_rgb) map_rgb[((size_t)img * C + p) * n + i] = m;
        } else {
          tot_y += m;
          if (map_y) map_y[(size_t)img * n + i] = m;
        }
      }
    }
    ssim_rgb[img] = tot_rgb / ((double)n * C);
    if (ssim_y) ssim_y[img] = C == 3 ? tot_y / (double)n : ssim_rgb[img];
  }
  return GRL_OK;
}

}  // extern "C"
