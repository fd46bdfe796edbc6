// grl_demosaic.h -- the MATLAB-style demosaic of packed RGGB Bayer planes (dm_matlab, utils/utils_mosaic.py:36-111) as a
// closed form shared by the host expansion (grl_demosaic_host), the standalone kernel (demosaic.cu) and the fused
// tensor-core head (misc_tc.cu).
//
// cfa4 (4, h, w) holds the mosaic of a (2h, 2w) image: cfa[2i, 2j] = R = cfa4[0], cfa[2i, 2j+1] = G = cfa4[1],
// cfa[2i+1, 2j] = G = cfa4[2], cfa[2i+1, 2j+1] = B = cfa4[3] (utils_mosaic.py:87-91).  The mosaic is reflect-padded by 2
// and correlated with four 5 x 5 filters (utils_mosaic.py:44-85, every weight k / 8 is exact in fp32).  Channel c at
// pixel (y, x) is the raw mosaic value at its native sites and one filter's response at the others (the fill table
// utils_mosaic.py:97-109):
//   G: (even, even) and (odd, odd) <- kgrb
//   R: (even, odd) <- krbg0, (odd, even) <- krbg1 = krbg0^T, (odd, odd) <- krbbr
//   B: (even, odd) <- krbg1, (odd, even) <- krbg0,          (even, even) <- krbbr
// A response is accumulated over the filter's nonzero taps in row-major order (dy, then dx), starting from the first
// product, with the rounded multiplies and adds of grl_hd.h, never contracted into FMAs, so every user of this code
// (host, standalone kernel, fused head) gives the same bits.
#pragma once

#include "grl_hd.h"

namespace grl {

enum { kDmRaw = -1, kDmGRB = 0, kDmRBG0 = 1, kDmRBG1 = 2, kDmRBBR = 3 };

// Which filter fills channel c (0 R, 1 G, 2 B) at a pixel of row parity py and column parity px (kDmRaw: the raw value).
GRL_HD int dm_filter(int c, int py, int px) {
  if (c == 1) return py == px ? kDmGRB : kDmRaw;
  const int f = (py == 0) ? (px == 0 ? kDmRBBR : kDmRBG0) : (px == 0 ? kDmRBG1 : kDmRBBR);
  if (c == 0) return (py == 0 && px == 0) ? kDmRaw : f;
  if (py == 1 && px == 1) return kDmRaw;  // c == 2: B is native at (odd, odd)
  return f == kDmRBG0 ? kDmRBG1 : f == kDmRBG1 ? kDmRBG0 : f;
}

// F.pad(..., "reflect") by at most 2 on an axis of n >= 3 samples: -1 -> 1, -2 -> 2, n -> n - 2, n + 1 -> n - 3.  Even n
// (always the case here) keeps the Bayer phase of every index.
GRL_HD int dm_reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

// Response of filter f at the pixel m is centred on; m(dy, dx) returns the (reflect-padded) mosaic value at offset (dy, dx).
template <class M>
GRL_HD float dm_response(int f, const M& m) {
  float a;
  switch (f) {
    case kDmGRB:  // [0 0 -1 0 0; 0 0 2 0 0; -1 2 4 2 -1; 0 0 2 0 0; 0 0 -1 0 0] / 8
      a = fmul_rn(-0.125f, m(-2, 0));
      a = fadd_rn(a, fmul_rn(0.25f, m(-1, 0)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(0, -2)));
      a = fadd_rn(a, fmul_rn(0.25f, m(0, -1)));
      a = fadd_rn(a, fmul_rn(0.5f, m(0, 0)));
      a = fadd_rn(a, fmul_rn(0.25f, m(0, 1)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(0, 2)));
      a = fadd_rn(a, fmul_rn(0.25f, m(1, 0)));
      return fadd_rn(a, fmul_rn(-0.125f, m(2, 0)));
    case kDmRBG0:  // [0 0 1/2 0 0; 0 -1 0 -1 0; -1 4 5 4 -1; 0 -1 0 -1 0; 0 0 1/2 0 0] / 8
      a = fmul_rn(0.0625f, m(-2, 0));
      a = fadd_rn(a, fmul_rn(-0.125f, m(-1, -1)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(-1, 1)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(0, -2)));
      a = fadd_rn(a, fmul_rn(0.5f, m(0, -1)));
      a = fadd_rn(a, fmul_rn(0.625f, m(0, 0)));
      a = fadd_rn(a, fmul_rn(0.5f, m(0, 1)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(0, 2)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(1, -1)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(1, 1)));
      return fadd_rn(a, fmul_rn(0.0625f, m(2, 0)));
    case kDmRBG1:  // krbg0 transposed
      a = fmul_rn(-0.125f, m(-2, 0));
      a = fadd_rn(a, fmul_rn(-0.125f, m(-1, -1)));
      a = fadd_rn(a, fmul_rn(0.5f, m(-1, 0)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(-1, 1)));
      a = fadd_rn(a, fmul_rn(0.0625f, m(0, -2)));
      a = fadd_rn(a, fmul_rn(0.625f, m(0, 0)));
      a = fadd_rn(a, fmul_rn(0.0625f, m(0, 2)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(1, -1)));
      a = fadd_rn(a, fmul_rn(0.5f, m(1, 0)));
      a = fadd_rn(a, fmul_rn(-0.125f, m(1, 1)));
      return fadd_rn(a, fmul_rn(-0.125f, m(2, 0)));
    default:  // kDmRBBR: [0 0 -3/2 0 0; 0 2 0 2 0; -3/2 0 6 0 -3/2; 0 2 0 2 0; 0 0 -3/2 0 0] / 8
      a = fmul_rn(-0.1875f, m(-2, 0));
      a = fadd_rn(a, fmul_rn(0.25f, m(-1, -1)));
      a = fadd_rn(a, fmul_rn(0.25f, m(-1, 1)));
      a = fadd_rn(a, fmul_rn(-0.1875f, m(0, -2)));
      a = fadd_rn(a, fmul_rn(0.75f, m(0, 0)));
      a = fadd_rn(a, fmul_rn(-0.1875f, m(0, 2)));
      a = fadd_rn(a, fmul_rn(0.25f, m(1, -1)));
      a = fadd_rn(a, fmul_rn(0.25f, m(1, 1)));
      return fadd_rn(a, fmul_rn(-0.1875f, m(2, 0)));
  }
}

// Channel c of the demosaiced image at a pixel of phase (py, px); m is centred on that pixel.
template <class M>
GRL_HD float dm_value(int c, int py, int px, const M& m) {
  const int f = dm_filter(c, py, px);
  return f == kDmRaw ? m(0, 0) : dm_response(f, m);
}

// Reads the reflect-padded mosaic of one image straight from its packed planes p (4, h, w), centred on (y, x).
struct DmPlanes {
  const float* p;
  int h, w, y, x;
  GRL_HD float operator()(int dy, int dx) const {
    const int Y = dm_reflect(y + dy, 2 * h), X = dm_reflect(x + dx, 2 * w);
    return p[((long long)((Y & 1) * 2 + (X & 1)) * h + (Y >> 1)) * w + (X >> 1)];
  }
};

// dm_matlab at full-resolution pixel (y, x) of the image whose packed planes are p (4, h, w); h, w >= 2.
GRL_HD float dm_pixel(const float* p, int h, int w, int c, int y, int x) {
  return dm_value(c, y & 1, x & 1, DmPlanes{p, h, w, y, x});
}

}  // namespace grl
