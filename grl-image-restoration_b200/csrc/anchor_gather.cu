// anchor_gather.cu -- the patch gather in front of the convolutional anchor projections (AnchorProjection with proj_type
// "conv2d" or "patchmerging", mixed_attn_block.py:679-711,:739-785).  A k x k, stride s, zero-padded convolution of a
// channels-last image is a GEMM of its patch rows with the (Cout, tap * C + c) weight, and PatchMerging is the same GEMM
// with a 2 x 2, stride 2 patch taken in its own tap order.  Anchors are L / df^2 rows, so the gather writes those rows
// once and the existing fp32 and tensor-core GEMMs do the projection:
//   y[(b, yo, xo), tap * C + c] = x[b, yo * s - pad + ky, xo * s - pad + kx, c]   (0 outside the image)
//   y[(b, yo, xo), k] = 0 for taps * C <= k < ldy   (the GEMM's K padding)
// tap = ky * k + kx (row_major, nn.Conv2d's weight order) or kx * k + ky (PatchMerging: x0 [0::2, 0::2], x1 [1::2, 0::2],
// x2 [0::2, 1::2], x3 [1::2, 1::2]).  The values are copied, so one kernel per element width serves fp32 and both 16-bit
// operand formats.
#include "grl_common.cuh"

namespace grl {

namespace {

template <class T>
__global__ void anchor_gather_kernel(const T* __restrict__ x, long long ldx, int B, int H, int W, int C, int ksize,
                                     int stride, int pad, int row_major, int Ho, int Wo, T* __restrict__ y, int ldy) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long rows = (long long)B * Ho * Wo;
  if (i >= rows * ldy) return;
  const long long m = i / ldy;
  const int k = (int)(i - m * ldy);
  T v = T(0);
  if (k < ksize * ksize * C) {
    const int tap = k / C, c = k - tap * C;
    const int ky = row_major ? tap / ksize : tap % ksize, kx = row_major ? tap % ksize : tap / ksize;
    const int xo = (int)(m % Wo);
    const long long t = m / Wo;
    const int yo = (int)(t % Ho), b = (int)(t / Ho);
    const int yy = yo * stride - pad + ky, xx = xo * stride - pad + kx;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = x[(((long long)b * H + yy) * W + xx) * ldx + c];
  }
  y[i] = v;
}

template <class T>
int launch_gather(const T* x, int64_t ldx, int B, int H, int W, int C, int ksize, int stride, int pad, int row_major, T* y,
                  int ldy, cudaStream_t st) {
  GRL_REQUIRE(x && y, "anchor_gather: null argument");
  GRL_REQUIRE(B >= 0 && H > 0 && W > 0 && C > 0 && ldx >= C && ksize >= 1 && stride >= 1 && pad >= 0 && pad < ksize,
              "anchor_gather: bad shape (%dx%dx%d, pitch %lld, k %d, stride %d, pad %d)", H, W, C, (long long)ldx, ksize,
              stride, pad);
  GRL_REQUIRE(H + 2 * pad >= ksize && W + 2 * pad >= ksize, "anchor_gather: %dx%d image smaller than the %d x %d patch", H,
              W, ksize, ksize);
  GRL_REQUIRE(ldy >= ksize * ksize * C, "anchor_gather: output pitch %d < %d taps x %d channels", ldy, ksize * ksize, C);
  const int Ho = (H + 2 * pad - ksize) / stride + 1, Wo = (W + 2 * pad - ksize) / stride + 1;
  const long long total = (long long)B * Ho * Wo * ldy;
  if (total == 0) return GRL_OK;
  anchor_gather_kernel<T><<<ceil_div(total, 256), 256, 0, st>>>(x, ldx, B, H, W, C, ksize, stride, pad, row_major, Ho, Wo,
                                                                 y, ldy);
  GRL_LAUNCH_CHECK("anchor_gather_kernel");
  return GRL_OK;
}

}  // namespace

}  // namespace grl

extern "C" {

int grl_anchor_gather_f32(const float* x, int64_t ldx, int B, int H, int W, int C, int ksize, int stride, int pad,
                          int row_major, float* y, int ldy, void* stream) {
  return grl::launch_gather<float>(x, ldx, B, H, W, C, ksize, stride, pad, row_major, y, ldy, (cudaStream_t)stream);
}

int grl_tc_anchor_gather16(const void* x, int64_t ldx, int B, int H, int W, int C, int ksize, int stride, int pad,
                           int row_major, void* y, int ldy, void* stream) {
  return grl::launch_gather<uint16_t>((const uint16_t*)x, ldx, B, H, W, C, ksize, stride, pad, row_major, (uint16_t*)y,
                                      ldy, (cudaStream_t)stream);
}

}  // extern "C"
