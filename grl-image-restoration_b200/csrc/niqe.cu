// niqe.cu -- the per-block NIQE features of the blind-SR evaluator on the device (utils/metrics/niqe.py:566-576 ->
// calculate_niqe :493-546 -> niqe :400-490 -> compute_feature :373-397 -> estimate_aggd_param :341-370, imresize
// :241-338).  The multivariate-Gaussian distance that turns the features into a score is batched torch float64
// (metrics.niqe).
//
// Stages, each one kernel over all B images:
//   luma    tensor_round (or the bytes of 8-bit (B, H, W, 3) pixels), the BGR-weighted luma of grl_niqe.h, crop
//           `border`, crop to 96 * floor(. / 96) from the top left;
//   mscn    (img - mu) / (sigma + 1) with mu, E[img^2] the 7 x 7 window correlated with mode "nearest" (a shared-memory tile
//           with a 3-pixel halo); float64 accumulation stored to fp32 as scipy.ndimage.convolve does for an fp32 input,
//           then every step in fp32 with explicitly rounded operations (nvcc would contract them into FMAs otherwise).
//           A constant region gives exactly 0, which is what makes a flat block's features NaN (see feat);
//   half    MATLAB bicubic x0.5 with antialiasing of img / 255, times 255: 8 taps with symmetric padding per axis, two
//           separable passes, float64 accumulation stored to fp32;
//   feat    one CTA per (block, scale, image): the block in shared memory, the five AGGD fits (the block and its products
//           with the four np.roll shifts, which wrap inside the block) from float64 moments, the argmin over the 9801
//           entry r_gam table as a block reduction that keeps the lowest index, and the 18 features of the scale.
// An AGGD fit of a block without negative (or without positive) values has NaN moments; np.argmin then returns 0, so alpha
// is 0.2 and every other feature of that fit is NaN.  That is reproduced, not repaired.
#include <algorithm>

#include "grl_common.cuh"
#include "grl_image_u8.h"
#include "grl_niqe.h"
#include "grl_resize.h"  // resize_mirror: imresize's symmetric padding

namespace grl {

constexpr int kNiqeGam = 9801;  // gam = 0.2 : 0.001 : 10

struct NiqeWin {
  double w[49];  // scipy's footprint order: the flipped window, row-major
};
struct NiqeTaps {
  float w[8];
};

template <class Img>
__global__ void niqe_luma_kernel(Img x, int H, int W, int border, int Hc, int Wc, float* __restrict__ y) {
  const int img = blockIdx.y;
  const long long n = (long long)Hc * Wc;
  const Img p = x.img(img);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / Wc), c = (int)(i - (long long)r * Wc);
    const long long off = (long long)(r + border) * W + (c + border);
    y[img * n + i] = niqe_luma((int)p(0, off), (int)p(1, off), (int)p(2, off));
  }
}

constexpr int kTx = 32, kTy = 8;

__global__ void __launch_bounds__(kTx* kTy) niqe_mscn_kernel(const float* __restrict__ in, int H, int W, NiqeWin win,
                                                             float* __restrict__ out) {
  __shared__ float tile[kTy + 6][kTx + 6];
  const long long plane = (long long)H * W;
  const float* src = in + blockIdx.z * plane;
  const int x0 = blockIdx.x * kTx, y0 = blockIdx.y * kTy;
  for (int t = threadIdx.y * kTx + threadIdx.x; t < (kTy + 6) * (kTx + 6); t += kTx * kTy) {
    const int ty = t / (kTx + 6), tx = t - ty * (kTx + 6);
    const int gy = min(max(y0 + ty - 3, 0), H - 1), gx = min(max(x0 + tx - 3, 0), W - 1);  // mode "nearest"
    tile[ty][tx] = src[(long long)gy * W + gx];
  }
  __syncthreads();
  const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
  if (x >= W || y >= H) return;
  double m = 0.0, s = 0.0;
#pragma unroll
  for (int i = 0; i < 7; ++i)
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      const float v = tile[threadIdx.y + i][threadIdx.x + j];
      m = __dadd_rn(m, __dmul_rn((double)v, win.w[i * 7 + j]));
      s = __dadd_rn(s, __dmul_rn((double)__fmul_rn(v, v), win.w[i * 7 + j]));  // np.square(img) is fp32
    }
  const float mu = (float)m, e2 = (float)s;
  const float sigma = sqrtf(fabsf(__fsub_rn(e2, __fmul_rn(mu, mu))));
  const float v0 = tile[threadIdx.y + 3][threadIdx.x + 3];
  out[blockIdx.z * plane + (long long)y * W + x] = __fdiv_rn(__fsub_rn(v0, mu), __fadd_rn(sigma, 1.0f));
}

// vertical pass: t (B, H/2, W) = taps over rows of img / 255
__global__ void niqe_half_rows_kernel(const float* __restrict__ in, int H, int W, NiqeTaps taps, float* __restrict__ t) {
  const int Ho = H / 2, img = blockIdx.y;
  const long long n = (long long)Ho * W;
  const float* src = in + (long long)img * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(i / W), x = (int)(i - (long long)oy * W);
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float v = __fdiv_rn(src[(long long)resize_mirror(2 * oy - 3 + k, H) * W + x], 255.0f);  // img / 255.0 in fp32
      acc = __dadd_rn(acc, __dmul_rn((double)taps.w[k], (double)v));
    }
    t[img * n + i] = (float)acc;
  }
}

// horizontal pass: out (B, H/2, W/2) = 255 * taps over columns of t
__global__ void niqe_half_cols_kernel(const float* __restrict__ t, int H, int W, NiqeTaps taps, float* __restrict__ out) {
  const int Ho = H / 2, Wo = W / 2, img = blockIdx.y;
  const long long n = (long long)Ho * Wo;
  const float* src = t + (long long)img * Ho * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(i / Wo), ox = (int)(i - (long long)oy * Wo);
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) acc = __dadd_rn(acc, __dmul_rn((double)taps.w[k], (double)src[(long long)oy * W + resize_mirror(2 * ox - 3 + k, W)]));
    out[img * n + i] = __fmul_rn((float)acc, 255.0f);
  }
}

constexpr int kFeatThreads = 256;

struct Moments {
  double sl, sr, sa;
  int nl, nr;
};

__device__ double block_sum(double v, double* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  double r = 0.0;
  for (int w = 0; w < kFeatThreads / 32; ++w) r += sh[w];  // same order in every thread
  return r;
}

// One AGGD fit (estimate_aggd_param) of the block's values x(i, j), all threads; returns the table index and the stds.
template <class X>
__device__ int aggd_fit(const X& xf, int bs, const double* __restrict__ r_gam, double* sh_d, int* sh_i, double* lstd_out,
                        double* rstd_out) {
  double sl = 0.0, sr = 0.0, sa = 0.0, nl = 0.0, nr = 0.0;
  for (int p = threadIdx.x; p < bs * bs; p += kFeatThreads) {
    const float v = xf(p / bs, p % bs);
    const double d = (double)v, d2 = d * d;
    if (v < 0.f) sl += d2, nl += 1.0;
    if (v > 0.f) sr += d2, nr += 1.0;
    sa += fabs(d);
  }
  sl = block_sum(sl, sh_d), sr = block_sum(sr, sh_d), sa = block_sum(sa, sh_d);
  nl = block_sum(nl, sh_d), nr = block_sum(nr, sh_d);
  const double N = (double)bs * bs;
  const double lstd = sqrt(sl / nl), rstd = sqrt(sr / nr);  // an empty side: 0 / 0 = NaN, as np.mean of an empty array
  const double g = lstd / rstd;
  const double rhat = (sa / N) * (sa / N) / ((sl + sr) / N);
  const double rn = rhat * (g * g * g + 1.0) * (g + 1.0) / ((g * g + 1.0) * (g * g + 1.0));
  // argmin of (r_gam - rn)^2, lowest index on ties; all-NaN -> 0 (np.argmin returns the first NaN)
  double best = INFINITY;
  int bi = 0x7fffffff;
  if (!isnan(rn)) {
    for (int i = threadIdx.x; i < kNiqeGam; i += kFeatThreads) {
      const double e = r_gam[i] - rn, e2 = e * e;
      if (e2 < best) best = e2, bi = i;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob < best || (ob == best && oi < bi)) best = ob, bi = oi;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sh_d[warp] = best, sh_i[warp] = bi;
  __syncthreads();
  best = sh_d[0], bi = sh_i[0];
  for (int w = 1; w < kFeatThreads / 32; ++w)
    if (sh_d[w] < best || (sh_d[w] == best && sh_i[w] < bi)) best = sh_d[w], bi = sh_i[w];
  *lstd_out = lstd, *rstd_out = rstd;
  return isnan(rn) ? 0 : bi;
}

// feats (B, nbw * nbh, 36): row iw * nbh + ih (niqe.py:458-465 walks columns of blocks outermost), scale 1 in columns
// 0..17, scale 2 in 18..35.  tables (4, 9801): gam, r_gam, sqrt(G(1/a) / G(3/a)), G(2/a) / G(1/a).
__global__ void __launch_bounds__(kFeatThreads) niqe_feat_kernel(const float* __restrict__ m1, const float* __restrict__ m2,
                                                                 int nbh, int nbw, const double* __restrict__ tables,
                                                                 double* __restrict__ feats) {
  __shared__ float blk[96 * 96];
  __shared__ double sh_d[kFeatThreads / 32];
  __shared__ int sh_i[kFeatThreads / 32];
  const int r = blockIdx.x, scale = blockIdx.y, img = blockIdx.z;
  const int iw = r / nbh, ih = r - iw * nbh;
  const int bs = scale == 0 ? 96 : 48;
  const int Wm = nbw * bs, Hm = nbh * bs;
  const float* src = (scale == 0 ? m1 : m2) + (long long)img * Hm * Wm;
  for (int p = threadIdx.x; p < bs * bs; p += kFeatThreads)
    blk[p] = src[(long long)(ih * bs + p / bs) * Wm + iw * bs + p % bs];
  __syncthreads();
  const double* gam = tables;
  const double* r_gam = tables + kNiqeGam;
  const double* bfac = tables + 2 * kNiqeGam;
  const double* mfac = tables + 3 * kNiqeGam;
  double* f = feats + ((long long)img * gridDim.x + r) * 36 + scale * 18;
  double ls, rs;
  int a = aggd_fit([&](int i, int j) { return blk[i * bs + j]; }, bs, r_gam, sh_d, sh_i, &ls, &rs);
  if (threadIdx.x == 0) f[0] = gam[a], f[1] = (ls * bfac[a] + rs * bfac[a]) / 2.0;
  // np.roll(block, (di, dj), axis=(0, 1)): shifted(i, j) = block((i - di) mod bs, (j - dj) mod bs)
  const int shifts[4][2] = {{0, 1}, {1, 0}, {1, 1}, {1, -1}};
  for (int s = 0; s < 4; ++s) {
    const int di = shifts[s][0], dj = shifts[s][1];
    a = aggd_fit(
        [&](int i, int j) {
          const int si = (i - di + bs) % bs, sj = (j - dj + bs) % bs;
          return __fmul_rn(blk[i * bs + j], blk[si * bs + sj]);  // block * shifted_block in fp32
        },
        bs, r_gam, sh_d, sh_i, &ls, &rs);
    if (threadIdx.x == 0) {
      const double bl = ls * bfac[a], br = rs * bfac[a];
      f[2 + 4 * s] = gam[a], f[3 + 4 * s] = (br - bl) * mfac[a], f[4 + 4 * s] = bl, f[5 + 4 * s] = br;
    }
  }
}

static int grid_1d(long long n) { return (int)std::max<long long>(1, std::min<long long>((n + 255) / 256, 1184)); }

// imresize's weights for x0.5 with antialiasing (niqe.py:169-238): kernel width 8, distances 3.5 - k for the 8 taps that
// survive, 0.5 * cubic(0.5 * d) normalised by their sum.  Every value is a short dyadic fraction and the sum is exactly 1,
// so the fp32 weights are exact whatever the order of evaluation.
static void niqe_half_taps(float* w8) {
  double s = 0.0, c[8];
  for (int k = 0; k < 8; ++k) {
    const double x = fabs(0.5 * (3.5 - k)), x2 = x * x, x3 = x2 * x;
    const double cub = x <= 1.0 ? 1.5 * x3 - 2.5 * x2 + 1.0 : (x <= 2.0 ? -0.5 * x3 + 2.5 * x2 - 4.0 * x + 2.0 : 0.0);
    c[k] = 0.5 * cub;
    s += c[k];
  }
  for (int k = 0; k < 8; ++k) w8[k] = (float)(c[k] / s);
}

static size_t align256(size_t b) { return (b + 255) / 256 * 256; }

template <class Img>
int niqe_luma_run(Img x, int B, int C, int H, int W, int border, float* y, void* stream) {
  GRL_REQUIRE(x.p && y, "niqe_luma: null argument");
  GRL_REQUIRE(C == 3, "niqe: needs RGB images (C == 3), got C = %d", C);
  GRL_REQUIRE(B >= 0 && border >= 0 && H - 2 * border >= 96 && W - 2 * border >= 96,
              "niqe: needs at least 96 x 96 pixels after cropping border %d, got %d x %d", border, H, W);
  if (B == 0) return GRL_OK;
  const int Hc = (H - 2 * border) / 96 * 96, Wc = (W - 2 * border) / 96 * 96;
  niqe_luma_kernel<<<dim3(grid_1d((long long)Hc * Wc), B), 256, 0, (cudaStream_t)stream>>>(x, H, W, border, Hc, Wc, y);
  GRL_LAUNCH_CHECK("niqe_luma_kernel");
  return GRL_OK;
}

// The four stages on one workspace: luma, MSCN, x0.5 resize, MSCN of the resized image, features.
template <class Img>
int niqe_features_run(Img x, int B, int C, int H, int W, int border, const double* window49, const double* tables,
                      void* workspace, size_t workspace_bytes, double* feats, void* stream) {
  GRL_REQUIRE(x.p && window49 && tables && feats, "niqe: null argument");
  GRL_REQUIRE(C == 3, "niqe: needs RGB images (C == 3), got C = %d", C);
  GRL_REQUIRE(B >= 0 && border >= 0 && H - 2 * border >= 96 && W - 2 * border >= 96,
              "niqe: needs at least 96 x 96 pixels after cropping border %d, got %d x %d", border, H, W);
  if (B == 0) return GRL_OK;
  GRL_REQUIRE(workspace && workspace_bytes >= grl_niqe_workspace(B, H, W, border), "niqe: workspace %zu bytes < %zu",
              workspace_bytes, grl_niqe_workspace(B, H, W, border));
  const int Hc = (H - 2 * border) / 96 * 96, Wc = (W - 2 * border) / 96 * 96;
  char* p = (char*)workspace;
  float* y = (float*)p;
  p += align256(sizeof(float) * B * (size_t)Hc * Wc);
  float* m1 = (float*)p;
  p += align256(sizeof(float) * B * (size_t)Hc * Wc);
  float* t = (float*)p;
  p += align256(sizeof(float) * B * (size_t)(Hc / 2) * Wc);
  float* y2 = (float*)p;
  p += align256(sizeof(float) * B * (size_t)(Hc / 2) * (Wc / 2));
  float* m2 = (float*)p;
  int rc;
  if ((rc = niqe_luma_run(x, B, C, H, W, border, y, stream)) != GRL_OK) return rc;
  if ((rc = grl_niqe_mscn_f32(y, B, Hc, Wc, window49, m1, stream)) != GRL_OK) return rc;
  if ((rc = grl_niqe_half_f32(y, B, Hc, Wc, t, y2, stream)) != GRL_OK) return rc;
  if ((rc = grl_niqe_mscn_f32(y2, B, Hc / 2, Wc / 2, window49, m2, stream)) != GRL_OK) return rc;
  return grl_niqe_feat_f32(m1, m2, B, Hc / 96, Wc / 96, tables, feats, stream);
}

}  // namespace grl

using namespace grl;

extern "C" {

int grl_niqe_luma_host(const uint8_t* rgb, int64_t n, float* y) {
  GRL_REQUIRE(rgb && y && n >= 0, "niqe_luma_host: bad arguments");
  for (int64_t i = 0; i < n; ++i) y[i] = niqe_luma(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
  return GRL_OK;
}

int grl_niqe_half_taps_host(float* w8) {
  GRL_REQUIRE(w8, "niqe_half_taps_host: null output");
  niqe_half_taps(w8);
  return GRL_OK;
}

int grl_niqe_luma_f32(const float* restored, int B, int C, int H, int W, int border, float* y, void* stream) {
  return niqe_luma_run(F32Planes{restored, (long long)H * W, C}, B, C, H, W, border, y, stream);
}

int grl_niqe_luma_u8(const uint8_t* restored, int B, int H, int W, int C, int border, float* y, void* stream) {
  return niqe_luma_run(U8Pixels{restored, (long long)H * W, C}, B, C, H, W, border, y, stream);
}

int grl_niqe_mscn_f32(const float* img, int B, int H, int W, const double* window49, float* out, void* stream) {
  GRL_REQUIRE(img && out, "niqe_mscn: null argument");
  GRL_REQUIRE(B >= 0 && H >= 1 && W >= 1 && window49, "niqe_mscn: bad arguments B=%d H=%d W=%d", B, H, W);
  if (B == 0) return GRL_OK;
  NiqeWin win;
  for (int i = 0; i < 49; ++i) win.w[i] = window49[48 - i];  // convolve = correlate with the flipped window
  niqe_mscn_kernel<<<dim3(ceil_div(W, kTx), ceil_div(H, kTy), B), dim3(kTx, kTy), 0, (cudaStream_t)stream>>>(img, H, W, win, out);
  GRL_LAUNCH_CHECK("niqe_mscn_kernel");
  return GRL_OK;
}

int grl_niqe_half_f32(const float* img, int B, int H, int W, float* tmp, float* out, void* stream) {
  GRL_REQUIRE(img && tmp && out, "niqe_half: null argument");
  GRL_REQUIRE(B >= 0 && H >= 4 && W >= 4 && H % 2 == 0 && W % 2 == 0, "niqe_half: needs even sizes >= 4, got %d x %d", H, W);
  if (B == 0) return GRL_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  NiqeTaps taps;
  niqe_half_taps(taps.w);
  niqe_half_rows_kernel<<<dim3(grid_1d((long long)H / 2 * W), B), 256, 0, st>>>(img, H, W, taps, tmp);
  GRL_LAUNCH_CHECK("niqe_half_rows_kernel");
  niqe_half_cols_kernel<<<dim3(grid_1d((long long)H / 2 * W / 2), B), 256, 0, st>>>(tmp, H, W, taps, out);
  GRL_LAUNCH_CHECK("niqe_half_cols_kernel");
  return GRL_OK;
}

int grl_niqe_feat_f32(const float* mscn1, const float* mscn2, int B, int nbh, int nbw, const double* tables, double* feats,
                      void* stream) {
  GRL_REQUIRE(mscn1 && mscn2 && feats, "niqe_feat: null argument");
  GRL_REQUIRE(B >= 0 && nbh >= 1 && nbw >= 1 && (long long)nbh * nbw <= 0x7fffffffLL && tables,
              "niqe_feat: bad arguments B=%d blocks %d x %d", B, nbh, nbw);
  if (B == 0) return GRL_OK;
  niqe_feat_kernel<<<dim3(nbh * nbw, 2, B), kFeatThreads, 0, (cudaStream_t)stream>>>(mscn1, mscn2, nbh, nbw, tables, feats);
  GRL_LAUNCH_CHECK("niqe_feat_kernel");
  return GRL_OK;
}

size_t grl_niqe_workspace(int B, int H, int W, int border) {
  if (B <= 0 || H - 2 * border < 96 || W - 2 * border < 96) return 0;
  const size_t Hc = (H - 2 * border) / 96 * 96, Wc = (W - 2 * border) / 96 * 96;
  const size_t full = align256(sizeof(float) * B * Hc * Wc), half = align256(sizeof(float) * B * (Hc / 2) * (Wc / 2));
  return 2 * full + align256(sizeof(float) * B * (Hc / 2) * Wc) + 2 * half;
}

int grl_niqe_features_f32(const float* restored, int B, int C, int H, int W, int border, const double* window49,
                          const double* tables, void* workspace, size_t workspace_bytes, double* feats, void* stream) {
  return niqe_features_run(F32Planes{restored, (long long)H * W, C}, B, C, H, W, border, window49, tables, workspace,
                           workspace_bytes, feats, stream);
}

int grl_niqe_features_u8(const uint8_t* restored, int B, int H, int W, int C, int border, const double* window49,
                         const double* tables, void* workspace, size_t workspace_bytes, double* feats, void* stream) {
  return niqe_features_run(U8Pixels{restored, (long long)H * W, C}, B, C, H, W, border, window49, tables, workspace,
                           workspace_bytes, feats, stream);
}

}  // extern "C"
