// grl_dataset_u8.h -- two test inputs the datasets build from a clean 8-bit RGB image, as closed forms shared by the host
// entries of dataset_u8.cu and its kernels.
//
// Bayer mosaic (DemosaicDataset.__getitem__, data/datasets/restoration_dm.py:33-37): mosaic_CFA_Bayer(img)[1]
// (utils/utils_mosaic.py:124-147) keeps R at (2y, 2x), G at (2y, 2x + 1), G at (2y + 1, 2x) and B at (2y + 1, 2x + 1) of
// every 2 x 2 quad, as (H / 2, W / 2, 4) uint8; to_tensor makes it (4, H / 2, W / 2) float32 of k / 255.  The reference
// raises on an odd H or W, which its datasets never pass (they crop to multiples of 8); here the odd last row or column
// is dropped, the mosaic of the even crop.  Values are the u8_unit of grl_image_u8.h.  Byte selection and one correctly rounded division:
// exact on both sides.
//
// MATLAB luma (rgb2ycbcr_np(img, y_only=True), utils/utils_image.py:143-190, the clean image of the gray JPEG command on
// LIVE1 / BSDS500 / Urban100, data/datasets/base_image.py:233-241): x = float32(k) / 255 in float32, widened to float64,
// np.dot(x, [65.481, 128.553, 24.966]) + 16.0, np.round (ties to even), cast to uint8.  numpy's dot of a length-3 row is
// BLAS ddot, whose order of operations depends on the BLAS build; luma_y evaluates the FMA chain
// fma(b, 24.966, fma(g, 128.553, r * 65.481)) through grl_hd.h.  What the result depends on is only the byte: for all
// 2^24 RGB triples it equals numpy's (tests/test_dataset_u8.py), because no triple lies close enough to a rounding
// midpoint for the order of the three products and two sums to decide it.  The float64 value before rounding is not
// claimed to equal numpy's.
#pragma once

#include <math.h>
#include <stdint.h>

#include "grl_hd.h"
#include "grl_image_u8.h"

namespace grl {

// Packed RGGB plane p (0 R, 1 G of the even rows, 2 G of the odd rows, 3 B) at quad (y, x) of an (H, W, 3) uint8 image:
// the byte mosaic_CFA_Bayer keeps there.
GRL_HD int mosaic_byte(const uint8_t* img, int W, int p, int y, int x) {
  const int dy = p >> 1, dx = p & 1, c = (p + 1) >> 1;  // R: c 0, both G: c 1, B: c 2
  return img[((long long)(2 * y + dy) * W + 2 * x + dx) * 3 + c];
}

// to_tensor of that byte.
GRL_HD float mosaic_value(const uint8_t* img, int W, int p, int y, int x) { return u8_unit(mosaic_byte(img, W, p, y, x)); }

// rgb2ycbcr_np(., y_only=True) of one RGB pixel, as a byte.
GRL_HD uint8_t luma_y(int r, int g, int b) {
  const double xr = (double)u8_unit(r), xg = (double)u8_unit(g), xb = (double)u8_unit(b);
  const double dot = dfma_rn(xb, 24.966, dfma_rn(xg, 128.553, dmul_rn(xr, 65.481)));
  return (uint8_t)rint(dadd_rn(dot, 16.0));  // in [16, 235]: the cast needs no clamp
}

}  // namespace grl
