// metric.cu -- the validation step's PSNR on the device in one pass (engines/base.py:255-268, utils/utils_image.py:8-11
// shave, :30-33 tensor_round, :43-80 rgb2ycbcr; utils/metrics/psnr.py:44-48).
//
// restored / target are (B, C, H, W) fp32 planes.  Both are rounded to the 8-bit grid (clamp to [0, 1], x255, round half
// to even like torch.round), `border` pixels are shaved on every side, and the squared error is accumulated EXACTLY as an
// integer (a rounded pixel is k/255; (k1 - k2)^2 <= 65025): the per-image sums are 64-bit integer atomics, so the result
// is independent of the block schedule.  C == 3 additionally accumulates the error of the luma of MATLAB's rgb2ycbcr
// (coefficients 65.481, 128.553, 24.966, offset 16, rounded to 8 bit).  HBM-bound: 2 x 4 bytes read per element.
#include <algorithm>

#include "grl_common.cuh"
#include "ops_f32.h"

namespace grl {

__device__ __forceinline__ float round8(float v) {
  v = fminf(fmaxf(v, 0.f), 1.f);
  return rintf(v * 255.0f);  // round half to even == torch.round
}

// y = round(65.481/255 * R + 128.553/255 * G + 24.966/255 * B + 16) with R, G, B on the 0..255 grid
// (metrics.rgb_to_y: (img * 255) @ (coeff / 255) + 16, rounded)
__device__ __forceinline__ float luma8(float r, float g, float b) {
  float acc = r * (65.481f / 255.0f);
  acc = fmaf(g, 128.553f / 255.0f, acc);
  acc = fmaf(b, 24.966f / 255.0f, acc);
  return rintf(acc + 16.0f);
}

__global__ void psnr_sse_kernel(const float* __restrict__ a, const float* __restrict__ b, int C, int H, int W, int border,
                                unsigned long long* __restrict__ sse /* (B, 2): rgb, y */) {
  const int img = blockIdx.y;
  const int h = H - 2 * border, w = W - 2 * border;
  const long long n = (long long)h * w;
  const long long plane = (long long)H * W;
  const float* pa = a + (long long)img * C * plane;
  const float* pb = b + (long long)img * C * plane;
  unsigned long long s_rgb = 0, s_y = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / w), x = (int)(i - (long long)y * w);
    const long long off = (long long)(y + border) * W + (x + border);
    float ra[3], rb[3];
    for (int c = 0; c < C; ++c) {
      const float va = round8(pa[c * plane + off]), vb = round8(pb[c * plane + off]);
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

int launch_psnr(const float* restored, const float* target, int B, int C, int H, int W, int border,
                unsigned long long* workspace, float* psnr_rgb, float* psnr_y, cudaStream_t st) {
  GRL_REQUIRE(B >= 0 && C >= 1 && C <= 4 && H > 2 * border && W > 2 * border && border >= 0, "psnr: bad shape (%d,%d,%d,%d) border %d",
              B, C, H, W, border);
  if (B == 0) return GRL_OK;
  GRL_CUDA(cudaMemsetAsync(workspace, 0, sizeof(unsigned long long) * 2 * (size_t)B, st));
  const long long n = (long long)(H - 2 * border) * (W - 2 * border);
  const int threads = 256;
  const int bx = (int)std::min<long long>((n + threads * 4 - 1) / (threads * 4), 592);  // ~4 CTAs per SM per image at most
  psnr_sse_kernel<<<dim3((unsigned)std::max(bx, 1), (unsigned)B), threads, 0, st>>>(restored, target, C, H, W, border, workspace);
  GRL_LAUNCH_CHECK("psnr_sse_kernel");
  psnr_finalize_kernel<<<(B + 127) / 128, 128, 0, st>>>(workspace, B, C, n, psnr_rgb, psnr_y);
  GRL_LAUNCH_CHECK("psnr_finalize_kernel");
  return GRL_OK;
}

// ---- PSNR-B (utils/metrics/psnrb.py:22-115) -------------------------------------------------------------------------
// Per image and per channel (the C channels, then the luma of luma8 for C == 3), five exact integer sums of squared 8-bit
// differences: the error against the target, and on the RESTORED image alone the differences of horizontal neighbours
// (x, x + 1) at block boundaries x = 7, 15, ... < W - 1 and elsewhere, and the same for vertical neighbours.
constexpr int kPsnrbSets = 4, kPsnrbSums = 5;  // sse, horizontal boundary, horizontal other, vertical boundary, vertical other

__global__ void psnrb_sums_kernel(const float* __restrict__ a, const float* __restrict__ b, int C, int H, int W,
                                  unsigned long long* __restrict__ sums /* (B, 4, 5) */) {
  const int img = blockIdx.y;
  const long long plane = (long long)H * W, n = plane;
  const float* pa = a + (long long)img * C * plane;
  const float* pb = b + (long long)img * C * plane;
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
        const float* p = pa + c * plane + i;
        va[c] = round8(p[0]), vb[c] = round8(pb[c * plane + i]);
        if (right) vr[c] = round8(p[1]);
        if (down) vd[c] = round8(p[W]);
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

int launch_psnrb(const float* restored, const float* target, int B, int C, int H, int W, unsigned long long* workspace,
                 double* psnrb_rgb, double* psnrb_y, cudaStream_t st) {
  GRL_REQUIRE(B >= 0 && (C == 1 || C == 3), "psnrb: needs C == 1 or 3, got %d", C);
  GRL_REQUIRE(H >= 16 && W >= 16, "psnrb: needs at least 16 x 16 pixels (the blocking-effect factor divides 0 by 0 below), got %d x %d",
              H, W);
  if (B == 0) return GRL_OK;
  GRL_CUDA(cudaMemsetAsync(workspace, 0, psnrb_workspace(B), st));
  const long long n = (long long)H * W;
  const int threads = 256;
  const int bx = (int)std::min<long long>((n + threads * 4 - 1) / (threads * 4), 592);
  psnrb_sums_kernel<<<dim3((unsigned)std::max(bx, 1), (unsigned)B), threads, 0, st>>>(restored, target, C, H, W, workspace);
  GRL_LAUNCH_CHECK("psnrb_sums_kernel");
  psnrb_finalize_kernel<<<(B + 127) / 128, 128, 0, st>>>(workspace, B, C, H, W, psnrb_rgb, psnrb_y);
  GRL_LAUNCH_CHECK("psnrb_finalize_kernel");
  return GRL_OK;
}

size_t psnrb_workspace(int B) { return sizeof(unsigned long long) * kPsnrbSets * kPsnrbSums * (size_t)(B > 0 ? B : 0); }

}  // namespace grl
