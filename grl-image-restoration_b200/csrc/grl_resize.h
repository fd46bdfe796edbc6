// grl_resize.h -- MATLAB's bicubic imresize with antialiasing for the integer downscales 1/2, 1/3 and 1/4, as closed forms
// shared by the host copy (grl_imresize_f32_host, grl_imresize_taps_host) and the kernel (resize.cu).
//
// The reference: utils/matlab_functions.py:20-88 (calculate_weights_indices) and :92-188 (imresize), the LR image of the
// SR dataset's online branch (data/datasets/restoration_sr.py:127-141).  For scale 1/s, output sample x = 1 .. out
// (MATLAB's 1-based numbering) sits at u = s x + (1 - s) / 2; the 4s + 2 candidate inputs j = floor(u - 2s) + m,
// m = 0 .. 4s + 1, weigh (1/s) cubic((u - j) / s), normalised by their sum.  u - floor(u - 2s) = 2s + frac(u) does not
// depend on x, so every output has the same weight row.  Candidate 0 always has weight 0 (cubic(2.25), cubic(2),
// cubic(2.125)), and the reference then drops the first and the last candidate, which leaves T = 4s taps m = 1 .. 4s; for
// s = 3 three of them (cubic(+-1) and cubic(-2)) are exactly 0 and stay.  In 0-based indices output o reads inputs
// s o + c + k, k = 0 .. T - 1, with c = floor((1 - 3s) / 2): -3, -4, -6 for s = 2, 3, 4.
//
// Here each weight is computed in double and rounded once to float32.  A pass is t = float32(sum_k w_k v_k) in
// increasing k with a float64 accumulator: w_k and v_k are floats, so each product is exact in double and dfma_rn rounds
// the sum only.  The H pass runs first and its float32 result feeds the W pass, as the reference's out_1 does.
// Indices past an edge mirror with the edge sample repeated (-1 -> 0, -2 -> 1, n -> n - 1), which is the reference's
// symmetric copy while its pad lengths pad_s = -c and pad_e = s (out - 1) + c + T - n are at most n.  Past that its copy
// fails, except for n = 1, where it broadcasts the one sample to every pad; resize_fits refuses exactly the failing
// lengths (2 .. 3, 2 .. 5 and 2 .. 6 for s = 2, 3, 4).
#pragma once

#include "grl_hd.h"

namespace grl {

constexpr int kResizeMaxTaps = 16;  // T = 4s for s = 4

GRL_HD constexpr int resize_taps_of(int s) { return 4 * s; }
// floor((1 - 3s) / 2): the 0-based first input of output 0
GRL_HD constexpr int resize_offset(int s) { return (1 - 3 * s) % 2 == 0 ? (1 - 3 * s) / 2 : (1 - 3 * s - 1) / 2; }

struct ResizeGeom {
  int T, c, out, pad_s, pad_e;  // taps, first input of output 0, ceil(n / s), the reference's sym_len_s and sym_len_e
};

GRL_HD ResizeGeom resize_geom(int n, int s) {
  const int T = resize_taps_of(s), c = resize_offset(s), out = (n + s - 1) / s;
  return {T, c, out, -c, s * (out - 1) + c + T - n};
}

// The reference's symmetric copy exists for this length: both pads inside the side, or a single sample.
GRL_HD bool resize_fits(int n, int s) {
  const ResizeGeom g = resize_geom(n, s);
  return n == 1 || (n >= 1 && g.pad_s <= n && g.pad_e <= n);
}

// The kernel of calculate_weights_indices (utils/matlab_functions.py:10-17) in double.
GRL_HD double resize_cubic(double x) {
  const double a = fabs(x), a2 = dmul_rn(a, a), a3 = dmul_rn(a2, a);
  if (a <= 1.0) return dadd_rn(dsub_rn(dmul_rn(1.5, a3), dmul_rn(2.5, a2)), 1.0);
  if (a <= 2.0) return dadd_rn(dsub_rn(dadd_rn(dmul_rn(-0.5, a3), dmul_rn(2.5, a2)), dmul_rn(4.0, a)), 2.0);
  return 0.0;
}

// The T = 4s float32 taps of scale 1/s, s in {2, 3, 4}, into w[0 .. T - 1]; returns T.
GRL_HD int resize_taps(int s, float* w) {
  const int P = 4 * s + 2;
  const double f = (s % 2 == 0) ? 0.5 : 0.0;  // frac(u); candidate m is at distance 2s + f - m from u
  double raw[4 * 4 + 2], sum = 0.0;
  for (int m = 0; m < P; ++m) {
    raw[m] = ddiv_rn(resize_cubic(ddiv_rn(dsub_rn(dadd_rn((double)(2 * s), f), (double)m), (double)s)), (double)s);
    sum = dadd_rn(sum, raw[m]);
  }
  const int T = resize_taps_of(s);
  for (int k = 0; k < T; ++k) w[k] = (float)ddiv_rn(raw[k + 1], sum);  // candidates 0 and P - 1 dropped
  return T;
}

// The reference's symmetric padding for -n <= i < 2n.
GRL_HD int resize_mirror(int i, int n) { return i < 0 ? -1 - i : (i >= n ? 2 * n - 1 - i : i); }
// The input sample that index i of a side of length n (resize_fits) reads.
GRL_HD int resize_index(int i, int n) { return n == 1 ? 0 : resize_mirror(i, n); }

// One output sample of a pass: float32(sum_k w[k] v[k]), k = 0 .. T - 1 in order, float64 accumulator.
GRL_HD float resize_dot(const float* w, const float* v, int T) {
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < T; ++k) acc = dfma_rn((double)w[k], (double)v[k], acc);
  return (float)acc;
}

}  // namespace grl
