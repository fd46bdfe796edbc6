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
// Every double operation is written rounded (awgn_add / awgn_mul / awgn_div / awgn_sqrt): nvcc contracts
// x1 * x1 + x2 * x2 into an FMA by default, and that changes r2.  The host evaluates plain IEEE operations, as numpy's
// C code does on x86-64 (no FMA contraction without -mfma).
//
// The one step that is not exact is log.  The host calls libm's log, as numpy does.  The device evaluates awgn_log_cr,
// a double-double log accurate to about 2^-100 relative, rounded once: the correctly rounded log(r2) except where log(r2)
// lies within that distance of a rounding midpoint.  So the device agrees with numpy wherever libm's log(r2) is
// correctly rounded; elsewhere f may differ by 1 ulp in float64, which reaches the float32 noise only when the product
// falls on a float32 rounding boundary (about 2^-29 per such sample).
#pragma once

#include <math.h>
#include <stdint.h>

#include "grl_image_u8.h"

#if defined(__CUDACC__)
#define GRL_AWGN_HD __host__ __device__ __forceinline__
#else
#define GRL_AWGN_HD inline
#endif

namespace grl {

constexpr int kMtN = 624, kMtM = 397;
constexpr int kAwgnPairsPerTwist = kMtN / 4;  // 156 polar candidates of 4 words each

// ---- rounded double arithmetic (no contraction on the device) -------------------------------------------------------
GRL_AWGN_HD double awgn_add(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
GRL_AWGN_HD double awgn_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
GRL_AWGN_HD double awgn_div(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
GRL_AWGN_HD double awgn_sqrt(double a) {
#if defined(__CUDA_ARCH__)
  return __dsqrt_rn(a);
#else
  return sqrt(a);
#endif
}
GRL_AWGN_HD double awgn_fma(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
  return __fma_rn(a, b, c);
#else
  return fma(a, b, c);
#endif
}

// ---- MT19937 (numpy's randomkit) -------------------------------------------------------------------------------------
// init_by_array(key, 8) after init_genrand(19650218).
GRL_AWGN_HD void awgn_mt_seed(uint32_t* mt, const uint32_t* key) {
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
GRL_AWGN_HD uint32_t awgn_twist_word(uint32_t cur, uint32_t next, uint32_t far) {
  const uint32_t y = (cur & 0x80000000u) | (next & 0x7fffffffu);
  return far ^ (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
}

// The whole twist in place, in order (host).  The kernel runs it as three parallel passes (awgn.cu).
GRL_AWGN_HD void awgn_mt_twist(uint32_t* mt) {
  for (int i = 0; i < kMtN; ++i) mt[i] = awgn_twist_word(mt[i], mt[(i + 1) % kMtN], mt[(i + kMtM) % kMtN]);
}

GRL_AWGN_HD uint32_t awgn_temper(uint32_t y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  return y ^ (y >> 18);
}

// ---- the polar method ------------------------------------------------------------------------------------------------
// 2 * legacy_double - 1 from two tempered words (every step exact).
GRL_AWGN_HD double awgn_signed_unit(uint32_t w0, uint32_t w1) {
  const double u = awgn_div(awgn_add(awgn_mul((double)(w0 >> 5), 67108864.0), (double)(w1 >> 6)), 9007199254740992.0);
  return awgn_add(awgn_mul(2.0, u), -1.0);
}

// r2 = x1 * x1 + x2 * x2, each product rounded.
GRL_AWGN_HD double awgn_r2(double x1, double x2) { return awgn_add(awgn_mul(x1, x1), awgn_mul(x2, x2)); }

GRL_AWGN_HD bool awgn_accept(double r2) { return !(r2 >= 1.0 || r2 == 0.0); }

// ---- log: double-double, rounded once ---------------------------------------------------------------------------------
struct AwgnDD {
  double hi, lo;
};

GRL_AWGN_HD AwgnDD awgn_two_sum(double a, double b) {
  const double s = awgn_add(a, b), bb = awgn_add(s, -a);
  return {s, awgn_add(awgn_add(a, -awgn_add(s, -bb)), awgn_add(b, -bb))};
}
GRL_AWGN_HD AwgnDD awgn_fast_two_sum(double a, double b) {  // |a| >= |b|
  const double s = awgn_add(a, b);
  return {s, awgn_add(b, -awgn_add(s, -a))};
}
GRL_AWGN_HD AwgnDD awgn_dd_add(AwgnDD x, AwgnDD y) {
  AwgnDD s = awgn_two_sum(x.hi, y.hi);
  const AwgnDD t = awgn_two_sum(x.lo, y.lo);
  s = awgn_fast_two_sum(s.hi, awgn_add(s.lo, t.hi));
  return awgn_fast_two_sum(s.hi, awgn_add(s.lo, t.lo));
}
GRL_AWGN_HD AwgnDD awgn_dd_mul(AwgnDD x, AwgnDD y) {
  const double p = awgn_mul(x.hi, y.hi);
  double e = awgn_fma(x.hi, y.hi, -p);
  e = awgn_add(e, awgn_add(awgn_mul(x.hi, y.lo), awgn_mul(x.lo, y.hi)));
  return awgn_fast_two_sum(p, e);
}
// 1 / d as a double-double.
GRL_AWGN_HD AwgnDD awgn_dd_recip(double d) {
  const double q = awgn_div(1.0, d);
  return {q, awgn_div(awgn_fma(-q, d, 1.0), d)};
}

// log(x) for a positive normal x, accurate to about 2^-100 relative before the final rounding:
//   x = 2^e m, m in [sqrt(1/2), sqrt(2));  log m = 2 atanh(s) = 2 s (1 + t P(t)), s = (m - 1) / (m + 1), t = s^2 <= 0.0295,
//   P(t) = sum_k t^k / (2k + 3): k < 9 in double-double, k = 9..19 in double (below 2^-50 of P), the rest below 2^-101.
GRL_AWGN_HD double awgn_log_cr(double x) {
  int e;
  double m = frexp(x, &e);
  if (m < 0.70710678118654752440) {
    m = awgn_mul(m, 2.0);
    --e;
  }
  const double num = awgn_add(m, -1.0);  // exact (Sterbenz)
  const AwgnDD den = awgn_two_sum(m, 1.0);
  // s = num / den
  const double q1 = awgn_div(num, den.hi);
  const double r = awgn_add(awgn_fma(-q1, den.hi, num), -awgn_mul(q1, den.lo));  // the fma is the exact remainder
  const AwgnDD s = awgn_fast_two_sum(q1, awgn_div(r, den.hi));
  const AwgnDD t = awgn_dd_mul(s, s);
  double tail = awgn_div(1.0, 41.0);
  for (int k = 18; k >= 9; --k) tail = awgn_fma(tail, t.hi, awgn_div(1.0, (double)(2 * k + 3)));
  AwgnDD p = {tail, 0.0};
  for (int k = 8; k >= 0; --k) p = awgn_dd_add(awgn_dd_mul(p, t), awgn_dd_recip((double)(2 * k + 3)));
  AwgnDD lm = awgn_dd_mul(s, awgn_dd_add({1.0, 0.0}, awgn_dd_mul(t, p)));
  lm = {awgn_mul(lm.hi, 2.0), awgn_mul(lm.lo, 2.0)};
  const double ln2_hi = 0x1.62e42fefa39efp-1, ln2_lo = 0x1.abc9e3b39803fp-56;  // ln 2 to 2^-106
  const double ed = (double)e, eh = awgn_mul(ed, ln2_hi);
  const AwgnDD el = awgn_fast_two_sum(eh, awgn_add(awgn_fma(ed, ln2_hi, -eh), awgn_mul(ed, ln2_lo)));
  const AwgnDD sum = awgn_dd_add(el, lm);
  return awgn_add(sum.hi, sum.lo);
}

GRL_AWGN_HD double awgn_log(double x) {
#if defined(__CUDA_ARCH__)
  return awgn_log_cr(x);
#else
  return log(x);
#endif
}

// f of an accepted candidate: sqrt(-2 log(r2) / r2).
GRL_AWGN_HD double awgn_polar_f(double r2) { return awgn_sqrt(awgn_div(awgn_mul(-2.0, awgn_log(r2)), r2)); }

// legacy_normal(0, scale) of a gauss g, in float64.
GRL_AWGN_HD double awgn_normal(double scale, double g) { return awgn_add(0.0, awgn_mul(scale, g)); }

// img_gt + torch.from_numpy(noise).float(): k / 255 plus the float32-rounded noise, a float32 add.
GRL_AWGN_HD float awgn_pixel(int k, double noise) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(u8_unit(k), __double2float_rn(noise));
#else
  return u8_unit(k) + (float)noise;
#endif
}

}  // namespace grl
