// grl_image_u8.h -- the 8-bit grid at both ends of the pipeline, as closed forms shared by the host expansions
// (grl_u8_to_f32_host, grl_f32_to_u8_host), the conversion kernels (image_u8.cu) and the metric kernels (metric.cu,
// niqe.cu).
//
// In:  every dataset turns an 8-bit HWC array into k / 255 fp32 CHW (transforms.functional.to_tensor:
//      img.float().div(255) on the CPU, an IEEE division).  u8_unit is that division, grl_hd.h's fdiv_rn: the
//      correctly rounded intrinsic on the device, the plain IEEE division on the host.
// Out: tensor_round (utils/utils_image.py:30-33) then x255 is round8: clamp to [0, 1], x255 in fp32, round half to even
//      like torch.round.  NaN, where torch leaves the byte undefined, is defined here as 0: fmaxf returns its non-NaN
//      operand, so the clamp already maps NaN to 0.  -0 -> 0, +inf -> 255, -inf -> 0.
// round8(u8_unit(k)) == k for all 256 k (tests/test_image_u8.py), which is why a metric read from the bytes equals the
// metric read from u8_unit of them bit for bit.
#pragma once

#include <math.h>
#include <stdint.h>

#include "grl_hd.h"

namespace grl {

// k / 255 in fp32, correctly rounded (whatever the build's -prec-div / fast-math flags).
GRL_HD float u8_unit(int k) { return fdiv_rn((float)k, 255.0f); }

// The 8-bit integer (as a float) of tensor_round(v) * 255; NaN -> 0.
GRL_HD float round8(float v) {
  v = fminf(fmaxf(v, 0.f), 1.f);
  return rintf(v * 255.0f);  // round half to even == torch.round
}

// The metric kernels' pixel readers.  img(b) selects image b; the result's (c, off) is the 8-bit integer k (as a float) of
// channel c at pixel off = y * W + x.
// (B, C, H, W) fp32 planes, tensor_round'ed on the fly.
struct F32Planes {
  const float* p;
  long long plane;  // H * W
  int C;
  GRL_HD F32Planes img(int b) const { return {p + (long long)b * C * plane, plane, C}; }
  GRL_HD float operator()(int c, long long off) const { return round8(p[c * plane + off]); }
};
// (B, H, W, C) uint8 pixels: the byte itself.
struct U8Pixels {
  const uint8_t* p;
  long long plane;  // H * W
  int C;
  GRL_HD U8Pixels img(int b) const { return {p + (long long)b * C * plane, plane, C}; }
  GRL_HD float operator()(int c, long long off) const { return (float)p[off * C + c]; }
};

}  // namespace grl
