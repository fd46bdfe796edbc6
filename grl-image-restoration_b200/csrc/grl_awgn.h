// grl_awgn.h -- the denoising test command's noisy input (DnDataset.__getitem__, validation branch,
// data/datasets/restoration_dn.py:134-143) as closed forms shared by the host entries of awgn.cu and its kernel.
//
// The reference seeds np.random.RandomState with the 8 little-endian uint32 words of sha256(name) and draws
// normal(0, sigma / 255, (C, H, W)), then adds the noise, rounded to float32, to the k / 255 image:
//   - RandomState(key array): MT19937 init_genrand(19650218) then init_by_array over the key; has_gauss = 0, pos = 624,
//     so the first draw twists.
//   - legacy_double: (tempered word >> 5) * 2^26 + (next >> 6), over 2^53 -- exact.
//   - legacy_gauss (Marsaglia polar): x1 = 2u - 1, x2 = 2u' - 1, r2 = x1 x1 + x2 x2, rejected while r2 >= 1 or r2 == 0;
//     f = sqrt(-2 log(r2) / r2); returns f x2, caches f x1 for the next call.  A candidate takes 4 words, so a twist of
//     624 words holds exactly 156 candidates and no candidate straddles two twists.
//   - legacy_normal: loc + scale * gauss, loc = 0; samples fill the tensor in C order.
//   - torch.from_numpy(noise).float(), then img_gt + noise in float32.
// Every double operation goes through the rounded operations of grl_hd.h: nvcc contracts x1 * x1 + x2 * x2 into an FMA
// by default, and that changes r2.  On the host they are plain IEEE operations and the build turns contraction off
// (-ffp-contract=off), so the host evaluates the operations numpy's C code writes, on any host ISA.
//
// The one step that is not exact is log.  The host calls libm's log, as numpy does.  The device evaluates awgn_log_cr,
// a double-double log accurate to about 2^-100 relative, rounded once: the correctly rounded log(r2) except where log(r2)
// lies within that distance of a rounding midpoint.  So the device agrees with numpy wherever libm's log(r2) is
// correctly rounded; elsewhere f may differ by 1 ulp in float64, which reaches the float32 noise only when the product
// falls on a float32 rounding boundary (about 2^-29 per such sample).
#pragma once

#include <math.h>
#include <stdint.h>

#include "grl_hd.h"
#include "grl_image_u8.h"

namespace grl {

constexpr int kMtN = 624, kMtM = 397;
constexpr int kAwgnPairsPerTwist = kMtN / 4;  // 156 polar candidates of 4 words each

// ---- MT19937 (numpy's randomkit) -------------------------------------------------------------------------------------
// init_by_array(key, 8) after init_genrand(19650218).
GRL_HD void awgn_mt_seed(uint32_t* mt, const uint32_t* key) {
  uint32_t s = 19650218u;
  for (int p = 0; p < kMtN; ++p) {
    mt[p] = s;
    s = 1812433253u * (s ^ (s >> 30)) + (uint32_t)(p + 1);
  }
  int i = 1, j = 0;
  for (int k = kMtN; k; --k) {
    mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1664525u)) + key[j] + (uint32_t)j;
    if (++i >= kMtN) {
      mt[0] = mt[kMtN - 1];
      i = 1;
    }
    if (++j >= 8) j = 0;
  }
  for (int k = kMtN - 1; k; --k) {
    mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1566083941u)) - (uint32_t)i;
    if (++i >= kMtN) {
      mt[0] = mt[kMtN - 1];
      i = 1;
    }
  }
  mt[0] = 0x80000000u;
}

// One word of the twist: new[i] = far ^ twist(old[i], next), far = the word kMtM ahead (mod kMtN), next = word i + 1.
GRL_HD uint32_t awgn_twist_word(uint32_t cur, uint32_t next, uint32_t far) {
  const uint32_t y = (cur & 0x80000000u) | (next & 0x7fffffffu);
  return far ^ (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
}

// The whole twist in place, in order (host).  The kernel runs it as three parallel passes (awgn.cu).
GRL_HD void awgn_mt_twist(uint32_t* mt) {
  for (int i = 0; i < kMtN; ++i) mt[i] = awgn_twist_word(mt[i], mt[(i + 1) % kMtN], mt[(i + kMtM) % kMtN]);
}

GRL_HD uint32_t awgn_temper(uint32_t y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  return y ^ (y >> 18);
}

// ---- the polar method ------------------------------------------------------------------------------------------------
// 2 * legacy_double - 1 from two tempered words (every step exact).
GRL_HD double awgn_signed_unit(uint32_t w0, uint32_t w1) {
  const double u = ddiv_rn(dadd_rn(dmul_rn((double)(w0 >> 5), 67108864.0), (double)(w1 >> 6)), 9007199254740992.0);
  return dadd_rn(dmul_rn(2.0, u), -1.0);
}

// r2 = x1 * x1 + x2 * x2, each product rounded.
GRL_HD double awgn_r2(double x1, double x2) { return dadd_rn(dmul_rn(x1, x1), dmul_rn(x2, x2)); }

GRL_HD bool awgn_accept(double r2) { return !(r2 >= 1.0 || r2 == 0.0); }

// ---- log: double-double, rounded once ---------------------------------------------------------------------------------
struct AwgnDD {
  double hi, lo;
};

GRL_HD AwgnDD awgn_two_sum(double a, double b) {
  const double s = dadd_rn(a, b), bb = dadd_rn(s, -a);
  return {s, dadd_rn(dadd_rn(a, -dadd_rn(s, -bb)), dadd_rn(b, -bb))};
}
GRL_HD AwgnDD awgn_fast_two_sum(double a, double b) {  // |a| >= |b|
  const double s = dadd_rn(a, b);
  return {s, dadd_rn(b, -dadd_rn(s, -a))};
}
GRL_HD AwgnDD awgn_dd_add(AwgnDD x, AwgnDD y) {
  AwgnDD s = awgn_two_sum(x.hi, y.hi);
  const AwgnDD t = awgn_two_sum(x.lo, y.lo);
  s = awgn_fast_two_sum(s.hi, dadd_rn(s.lo, t.hi));
  return awgn_fast_two_sum(s.hi, dadd_rn(s.lo, t.lo));
}
GRL_HD AwgnDD awgn_dd_mul(AwgnDD x, AwgnDD y) {
  const double p = dmul_rn(x.hi, y.hi);
  double e = dfma_rn(x.hi, y.hi, -p);
  e = dadd_rn(e, dadd_rn(dmul_rn(x.hi, y.lo), dmul_rn(x.lo, y.hi)));
  return awgn_fast_two_sum(p, e);
}
// 1 / d as a double-double.
GRL_HD AwgnDD awgn_dd_recip(double d) {
  const double q = ddiv_rn(1.0, d);
  return {q, ddiv_rn(dfma_rn(-q, d, 1.0), d)};
}

// log(x) for a positive normal x, accurate to about 2^-100 relative before the final rounding:
//   x = 2^e m, m in [sqrt(1/2), sqrt(2));  log m = 2 atanh(s) = 2 s (1 + t P(t)), s = (m - 1) / (m + 1), t = s^2 <= 0.0295,
//   P(t) = sum_k t^k / (2k + 3): k < 9 in double-double, k = 9..19 in double (below 2^-50 of P), the rest below 2^-101.
GRL_HD double awgn_log_cr(double x) {
  int e;
  double m = frexp(x, &e);
  if (m < 0.70710678118654752440) {
    m = dmul_rn(m, 2.0);
    --e;
  }
  const double num = dadd_rn(m, -1.0);  // exact (Sterbenz)
  const AwgnDD den = awgn_two_sum(m, 1.0);
  // s = num / den
  const double q1 = ddiv_rn(num, den.hi);
  const double r = dadd_rn(dfma_rn(-q1, den.hi, num), -dmul_rn(q1, den.lo));  // the fma is the exact remainder
  const AwgnDD s = awgn_fast_two_sum(q1, ddiv_rn(r, den.hi));
  const AwgnDD t = awgn_dd_mul(s, s);
  double tail = ddiv_rn(1.0, 41.0);
  for (int k = 18; k >= 9; --k) tail = dfma_rn(tail, t.hi, ddiv_rn(1.0, (double)(2 * k + 3)));
  AwgnDD p = {tail, 0.0};
  for (int k = 8; k >= 0; --k) p = awgn_dd_add(awgn_dd_mul(p, t), awgn_dd_recip((double)(2 * k + 3)));
  AwgnDD lm = awgn_dd_mul(s, awgn_dd_add({1.0, 0.0}, awgn_dd_mul(t, p)));
  lm = {dmul_rn(lm.hi, 2.0), dmul_rn(lm.lo, 2.0)};
  const double ln2_hi = 0x1.62e42fefa39efp-1, ln2_lo = 0x1.abc9e3b39803fp-56;  // ln 2 to 2^-106
  const double ed = (double)e, eh = dmul_rn(ed, ln2_hi);
  const AwgnDD el = awgn_fast_two_sum(eh, dadd_rn(dfma_rn(ed, ln2_hi, -eh), dmul_rn(ed, ln2_lo)));
  const AwgnDD sum = awgn_dd_add(el, lm);
  return dadd_rn(sum.hi, sum.lo);
}

GRL_HD double awgn_log(double x) {
#if defined(__CUDA_ARCH__)
  return awgn_log_cr(x);
#else
  return log(x);
#endif
}

// f of an accepted candidate: sqrt(-2 log(r2) / r2).
GRL_HD double awgn_polar_f(double r2) { return dsqrt_rn(ddiv_rn(dmul_rn(-2.0, awgn_log(r2)), r2)); }

// legacy_normal(0, scale) of a gauss g, in float64.
GRL_HD double awgn_normal(double scale, double g) { return dadd_rn(0.0, dmul_rn(scale, g)); }

// img_gt + torch.from_numpy(noise).float(): k / 255 plus the float32-rounded noise, a float32 add.
GRL_HD float awgn_pixel(int k, double noise) { return fadd_rn(u8_unit(k), (float)noise); }

}  // namespace grl
