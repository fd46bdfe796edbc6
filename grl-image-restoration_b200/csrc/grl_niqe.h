// grl_niqe.h -- the luma NIQE is computed on (utils/metrics/niqe.py:143-156, :75-111, :529-542, :566-576), as a closed
// form shared by the host expansion (grl_niqe_luma_host) and the luma kernel (niqe.cu).
//
// The evaluator receives tensor_round(model(x)) (engines/base_gan.py:152), so every channel is k / 255 in fp32 with k an
// 8-bit integer.  Its chain is: p * 255 in fp32; / 255 in fp32; a float64 dot with (24.966, 128.553, 65.481) + 16 --
// bgr2ycbcr's BGR weights applied to an RGB array, so R takes 24.966 and B 65.481, the reverse of MATLAB's rgb2ycbcr and
// of metric.cu's luma8; / 255 in float64; a cast to fp32; * 255 in fp32; round half to even.  The dot is summed R, G, B
// in that order without FMA, which reproduces NumPy on all 256^3 triples (tests/test_niqe.py).
#pragma once

#include <math.h>

#include "grl_hd.h"

namespace grl {

// fp32 value of one channel after p * 255 and / 255 (p = k / 255 from tensor_round).
GRL_HD float niqe_chan(int k) {
  const float p = fdiv_rn((float)k, 255.0f);
  return fdiv_rn(fmul_rn(p, 255.0f), 255.0f);
}

// Rounded luma (a float holding an integer in [16, 235]) of the 8-bit RGB triple (r, g, b).
GRL_HD float niqe_luma(int r, int g, int b) {
  double d = dmul_rn((double)niqe_chan(r), 24.966);
  d = dadd_rn(d, dmul_rn((double)niqe_chan(g), 128.553));
  d = dadd_rn(d, dmul_rn((double)niqe_chan(b), 65.481));
  d = dadd_rn(d, 16.0);
  const float f = (float)ddiv_rn(d, 255.0);
  return rintf(fmul_rn(f, 255.0f));
}

}  // namespace grl
