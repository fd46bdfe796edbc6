// grl_ssim.h -- the SSIM of the validation step (utils/metrics/ssim.py:17-85 as called by
// StructuralSimilarityIndexMeasure.update, ssim.py:167-193), as a closed form shared by the host computation
// (grl_ssim_host) and the kernel (ssim_tile_kernel in metric.cu).
//
// Both images are tensor_round'ed, so every plane holds 8-bit integers k (the value is k / 255).  The arithmetic is float64
// on the integers themselves: the SSIM map is unchanged when both images are scaled by 255 and C1, C2 by 255^2, and k, k^2
// and k1 * k2 are exact in float64.  A windowed sum is separable: 11 taps along the row, then 11 taps down the column, each
// an fma chain from tap 0 to tap 10 starting at 0; positions outside the image hold 0 (zero padding, windows at the border
// are not renormalised), and fma(t, 0, acc) == acc, so skipping them or not gives the same bits.  The reference convolves
// with the 2-D window float32(t t^T) and sums in fp32; the two windows differ by at most 6e-8 relative per weight.
#pragma once

#include "grl_hd.h"

namespace grl {

constexpr int kSsimTaps = 11, kSsimHalo = 5;
// round(exp(-(i - 5)^2 / 4.5), 6) over their sum, in float64 (gaussian(11, 1.5), ssim.py:17-24)
GRL_HD double ssim_tap(int i) {
  // the sum as the reference takes it, left to right: 3.7592320000000004
  constexpr double s = 0.003866 + 0.028566 + 0.135335 + 0.411112 + 0.800737 + 1.0 + 0.800737 + 0.411112 + 0.135335 + 0.028566 + 0.003866;
  constexpr double t[kSsimTaps] = {0.003866 / s, 0.028566 / s, 0.135335 / s, 0.411112 / s, 0.800737 / s, 1.0 / s,
                                   0.800737 / s, 0.411112 / s, 0.135335 / s, 0.028566 / s, 0.003866 / s};
  return t[i];
}

// C1 = 0.01^2 and C2 = 0.03^2 (ssim.py:57-58) for data in [0, 1], times 255^2 for data in [0, 255]
constexpr double kSsimC1 = 1e-4 * 65025.0, kSsimC2 = 9e-4 * 65025.0;

// One value of the SSIM map (ssim.py:42-62) from the five windowed sums of a, b, a^2, b^2 and a * b on the 0..255 scale.
GRL_HD double ssim_map_value(double sa, double sb, double saa, double sbb, double sab) {
  const double mu_aa = dmul_rn(sa, sa), mu_bb = dmul_rn(sb, sb), mu_ab = dmul_rn(sa, sb);
  const double var_a = dsub_rn(saa, mu_aa), var_b = dsub_rn(sbb, mu_bb), cov = dsub_rn(sab, mu_ab);
  const double num = dmul_rn(dfma_rn(2.0, mu_ab, kSsimC1), dfma_rn(2.0, cov, kSsimC2));
  const double den = dmul_rn(dadd_rn(dadd_rn(mu_aa, mu_bb), kSsimC1), dadd_rn(dadd_rn(var_a, var_b), kSsimC2));
  return ddiv_rn(num, den);
}

}  // namespace grl
