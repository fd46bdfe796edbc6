// grl_jpeg.h -- the pixels of a baseline JPEG round trip (the JPEG test command's jpeg_compress,
// data/datasets/restoration_jpeg.py:62-79: cv2.imencode at quality q, then cv2.imdecode) as closed forms shared by the
// host expansion grl_jpeg_roundtrip_host and the kernels of jpeg.cu.
//
// Entropy coding is lossless, so the decoded pixels are a function of integer arithmetic only: libjpeg's default
// compressor (4:2:0 for colour, islow forward DCT, jpeg_set_quality tables) and default decompressor (islow inverse DCT,
// "fancy" h2v2 upsampling).  Every step below works on one 8 x 8 block or one 2 x 2 neighbourhood, in integers, so the
// kernels and the host agree bit for bit; tests/test_jpeg.py pins the host expansion to the codec's bytes.
//
// An image is uint8 (H, W, C), C = 1 (one component, coded as is) or 3 (RGB -> YCbCr, Cb / Cr downsampled 2 x 2).
// Edges, as the codec pads them: columns past W - 1 replicate the last column (up to the MCU width); rows past H - 1
// replicate the last row up to an even height, and below that each component replicates its own last row -- for the
// chroma that is the last DOWNSAMPLED row, which differs from downsampling replicated image rows when H is even.
#pragma once

#include <stdint.h>

#include "grl_hd.h"

namespace grl {

typedef long long jpeg_long;  // libjpeg's JLONG: the DCT products and the colour sums

// ITU T.81 Annex K tables K.1 (luminance) and K.2 (chrominance), natural order.
GRL_HD int jpeg_std_table(int chroma, int k) {
  const int r = k >> 3, c = k & 7;
  if (chroma) {
    const uint8_t t[4][4] = {{17, 18, 24, 47}, {18, 21, 26, 66}, {24, 26, 56, 99}, {47, 66, 99, 99}};
    return r < 4 && c < 4 ? t[r][c] : 99;
  }
  const uint8_t t[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40, 57,
                         69, 56, 14, 17, 22,  29,  51,  87,  80, 62, 18, 22, 37,  56,  68,  109, 103, 77, 24, 35, 55, 64,
                         81, 104, 113, 92, 49, 64, 78,  87,  103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
  return t[k];
}

// jpeg_set_quality(q, force_baseline = TRUE): entry k (natural order) of the luma (chroma = 0) or chroma table.
GRL_HD int jpeg_quant(int quality, int chroma, int k) {
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  const int v = (jpeg_std_table(chroma, k) * scale + 50) / 100;
  return v < 1 ? 1 : (v > 255 ? 255 : v);
}

// ---- colour, 16-bit fixed point: FIX(x) = (int)(x * 65536 + 0.5) ------------------------------------------------------
constexpr int kJpegScale = 16;
constexpr jpeg_long kJpegHalf = (jpeg_long)1 << (kJpegScale - 1);

GRL_HD int jpeg_y(int r, int g, int b) { return (int)((19595LL * r + 38470LL * g + 7471LL * b + kJpegHalf) >> 16); }
// Cb (comp 1) or Cr (comp 2); the rounding is 0.5 - epsilon, so the result stays <= 255 without a clamp.
GRL_HD int jpeg_chroma(int comp, int r, int g, int b) {
  const jpeg_long off = ((jpeg_long)128 << kJpegScale) + kJpegHalf - 1;
  return comp == 1 ? (int)((-11059LL * r - 21709LL * g + 32768LL * b + off) >> 16)
                   : (int)((32768LL * r - 27439LL * g - 5329LL * b + off) >> 16);
}
GRL_HD int jpeg_clamp255(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }
// YCbCr -> one of R (c = 0), G, B, range-limited to 0..255.
GRL_HD int jpeg_rgb(int c, int y, int cb, int cr) {
  cb -= 128;
  cr -= 128;
  int v;
  if (c == 0)
    v = y + (int)((91881LL * cr + kJpegHalf) >> 16);
  else if (c == 1)
    v = y + (int)((-22554LL * cb - 46802LL * cr + kJpegHalf) >> 16);
  else
    v = y + (int)((116130LL * cb + kJpegHalf) >> 16);
  return jpeg_clamp255(v);
}

// ---- the islow DCT (CONST_BITS 13, PASS1_BITS 2) ----------------------------------------------------------------------
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr jpeg_long F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                    F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

// Rounded right shift of a product sum; every result of the two passes fits an int.
GRL_HD int jpeg_descale(jpeg_long x, int n) { return (int)((x + ((jpeg_long)1 << (n - 1))) >> n); }

// One forward pass over 8 values d[0], d[s], ..., d[7 s]; pass 1 (rows) keeps PASS1_BITS of extra precision.
GRL_HD void jpeg_fdct_1d(int* d, int s, bool pass1) {
  const jpeg_long tmp0 = d[0] + d[7 * s], tmp7 = d[0] - d[7 * s], tmp1 = d[s] + d[6 * s], tmp6 = d[s] - d[6 * s];
  const jpeg_long tmp2 = d[2 * s] + d[5 * s], tmp5 = d[2 * s] - d[5 * s], tmp3 = d[3 * s] + d[4 * s],
                  tmp4 = d[3 * s] - d[4 * s];
  const jpeg_long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  const int n = pass1 ? kConstBits - kPass1Bits : kConstBits + kPass1Bits;
  d[0] = pass1 ? (int)(tmp10 + tmp11) * (1 << kPass1Bits) : jpeg_descale(tmp10 + tmp11, kPass1Bits);
  d[4 * s] = pass1 ? (int)(tmp10 - tmp11) * (1 << kPass1Bits) : jpeg_descale(tmp10 - tmp11, kPass1Bits);
  const jpeg_long e = (tmp12 + tmp13) * F0541;
  d[2 * s] = jpeg_descale(e + tmp13 * F0765, n);
  d[6 * s] = jpeg_descale(e - tmp12 * F1847, n);
  const jpeg_long z5 = (tmp4 + tmp6 + tmp5 + tmp7) * F1175;
  const jpeg_long z1 = -(tmp4 + tmp7) * F0899, z2 = -(tmp5 + tmp6) * F2562;
  const jpeg_long z3 = -(tmp4 + tmp6) * F1961 + z5, z4 = -(tmp5 + tmp7) * F0390 + z5;
  d[7 * s] = jpeg_descale(tmp4 * F0298 + z1 + z3, n);
  d[5 * s] = jpeg_descale(tmp5 * F2053 + z2 + z4, n);
  d[3 * s] = jpeg_descale(tmp6 * F3072 + z2 + z3, n);
  d[s] = jpeg_descale(tmp7 * F1501 + z1 + z4, n);
}

// One inverse pass over 8 values; pass 1 (columns of dequantised coefficients) keeps PASS1_BITS, pass 2 (rows) also
// removes the DCT's factor of 8.
GRL_HD void jpeg_idct_1d(int* z, int s, bool pass1) {
  const jpeg_long e = ((jpeg_long)z[2 * s] + z[6 * s]) * F0541;
  const jpeg_long tmp2 = e - z[6 * s] * F1847, tmp3 = e + z[2 * s] * F0765;
  const jpeg_long tmp0 = ((jpeg_long)z[0] + z[4 * s]) * (1 << kConstBits);
  const jpeg_long tmp1 = ((jpeg_long)z[0] - z[4 * s]) * (1 << kConstBits);
  const jpeg_long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  jpeg_long t0 = z[7 * s], t1 = z[5 * s], t2 = z[3 * s], t3 = z[s];
  const jpeg_long z5 = (t0 + t2 + t1 + t3) * F1175;
  const jpeg_long z1 = -(t0 + t3) * F0899, z2 = -(t1 + t2) * F2562;
  const jpeg_long z3 = -(t0 + t2) * F1961 + z5, z4 = -(t1 + t3) * F0390 + z5;
  t0 = t0 * F0298 + z1 + z3;
  t1 = t1 * F2053 + z2 + z4;
  t2 = t2 * F3072 + z2 + z3;
  t3 = t3 * F1501 + z1 + z4;
  const int n = pass1 ? kConstBits - kPass1Bits : kConstBits + kPass1Bits + 3;
  z[0] = jpeg_descale(tmp10 + t3, n);
  z[7 * s] = jpeg_descale(tmp10 - t3, n);
  z[s] = jpeg_descale(tmp11 + t2, n);
  z[6 * s] = jpeg_descale(tmp11 - t2, n);
  z[2 * s] = jpeg_descale(tmp12 + t1, n);
  z[5 * s] = jpeg_descale(tmp12 - t1, n);
  z[3 * s] = jpeg_descale(tmp13 + t0, n);
  z[4 * s] = jpeg_descale(tmp13 - t0, n);
}

// The coefficient the decoder sees: the FDCT output (8 x the DCT) divided by 8 qv, rounded half away from zero, times qv.
GRL_HD int jpeg_requant(int c, int qv) {
  const int div = 8 * qv, a = c < 0 ? -c : c, q = (a + (div >> 1)) / div;
  return (c < 0 ? -q : q) * qv;
}

// One block through the codec: b (64 samples 0..255, row-major) -> FDCT -> quantise -> dequantise -> IDCT -> b, the
// decoder's samples (the IDCT's + 128, clamped to 0..255).  qt: the component's 64 quantisation values, natural order.
GRL_HD void jpeg_block_roundtrip(int* b, const uint8_t* qt) {
#pragma unroll
  for (int i = 0; i < 64; ++i) b[i] -= 128;
#pragma unroll
  for (int r = 0; r < 8; ++r) jpeg_fdct_1d(b + 8 * r, 1, true);
#pragma unroll
  for (int c = 0; c < 8; ++c) jpeg_fdct_1d(b + c, 8, false);
#pragma unroll
  for (int i = 0; i < 64; ++i) b[i] = jpeg_requant(b[i], qt[i]);
#pragma unroll
  for (int c = 0; c < 8; ++c) jpeg_idct_1d(b + c, 8, true);
#pragma unroll
  for (int r = 0; r < 8; ++r) jpeg_idct_1d(b + 8 * r, 1, false);
#pragma unroll
  for (int i = 0; i < 64; ++i) b[i] = jpeg_clamp255(b[i] + 128);
}

// ---- whole blocks of an image ------------------------------------------------------------------------------------------
struct JpegImage {
  const uint8_t* src;  // (H, W, C) uint8
  int H, W, C;
  GRL_HD int h2() const { return (H + 1) >> 1; }  // the chroma components' real size
  GRL_HD int w2() const { return (W + 1) >> 1; }
  GRL_HD int px(int y, int x, int c) const {      // clamp-to-edge
    y = y < H ? y : H - 1;
    x = x < W ? x : W - 1;
    return src[((long long)y * W + x) * C + c];
  }
  GRL_HD int luma(int y, int x) const {
    return C == 1 ? px(y, x, 0) : jpeg_y(px(y, x, 0), px(y, x, 1), px(y, x, 2));
  }
  // Downsampled chroma sample (cy, cx) of component comp (1 = Cb, 2 = Cr): the 2 x 2 sum plus a bias of 1, 2, 1, 2, ...
  // along the row, >> 2.  Rows below the component's last real row repeat it.
  GRL_HD int chroma(int comp, int cy, int cx) const {
    cy = cy < h2() ? cy : h2() - 1;
    int s = 1 + (cx & 1);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int y = 2 * cy + dy, x = 2 * cx + dx;
        s += jpeg_chroma(comp, px(y, x, 0), px(y, x, 1), px(y, x, 2));
      }
    return s >> 2;
  }
};

// Coded blocks of component comp (0 = Y or gray, 1 = Cb, 2 = Cr): rows x cols.
GRL_HD int jpeg_blocks_y(const JpegImage& im, int comp) { return ((comp ? im.h2() : im.H) + 7) >> 3; }
GRL_HD int jpeg_blocks_x(const JpegImage& im, int comp) { return ((comp ? im.w2() : im.W) + 7) >> 3; }

// Block (by, bx) of component comp through the codec; the decoded samples inside the component's real area go to
// out (row pitch ld): the image's size for Y, (h2, w2) for chroma.
GRL_HD void jpeg_component_block(const JpegImage& im, int comp, int by, int bx, const uint8_t* qt, uint8_t* out,
                                 int ld) {
  int b[64];
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c)
      b[8 * r + c] = comp ? im.chroma(comp, 8 * by + r, 8 * bx + c) : im.luma(8 * by + r, 8 * bx + c);
  jpeg_block_roundtrip(b, qt);
  const int h = comp ? im.h2() : im.H, w = comp ? im.w2() : im.W;
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int y = 8 * by + r, x = 8 * bx + c;
      if (y < h && x < w) out[(long long)y * ld + x] = (uint8_t)b[8 * r + c];
    }
}

// The decoder's chroma at image pixel (y, x) from the decoded (h2, w2) plane p: "fancy" (triangle) upsampling, the
// nearer chroma row and column weighted 3 against 1 and edge samples replicated: 3 near + far vertically, then
// (3 this + neighbour + 8) >> 4 on even columns, + 7 on odd ones.  A component at most 2 samples wide is upsampled by
// plain replication instead (libjpeg's h2v2_upsample).
GRL_HD int jpeg_upsample(const uint8_t* p, int h2, int w2, int y, int x) {
  const int cy = y >> 1, cx = x >> 1;
  if (w2 <= 2) return p[(long long)cy * w2 + cx];
  int ny = (y & 1) ? cy + 1 : cy - 1;
  ny = ny < 0 ? 0 : (ny >= h2 ? h2 - 1 : ny);
  int nx = (x & 1) ? cx + 1 : cx - 1;
  nx = nx < 0 ? 0 : (nx >= w2 ? w2 - 1 : nx);
  const uint8_t* r0 = p + (long long)cy * w2;
  const uint8_t* r1 = p + (long long)ny * w2;
  const int here = 3 * r0[cx] + r1[cx], next = 3 * r0[nx] + r1[nx];
  return (3 * here + next + 8 - (x & 1)) >> 4;
}

// Decoded RGB at pixel (y, x) from the decoded planes: Y (H, W), Cb and Cr (h2, w2).
GRL_HD void jpeg_decode_pixel(const uint8_t* Y, const uint8_t* cb, const uint8_t* cr, int H, int W, int y, int x,
                              uint8_t* rgb) {
  const int h2 = (H + 1) >> 1, w2 = (W + 1) >> 1;
  const int l = Y[(long long)y * W + x], u = jpeg_upsample(cb, h2, w2, y, x), v = jpeg_upsample(cr, h2, w2, y, x);
#pragma unroll
  for (int c = 0; c < 3; ++c) rgb[c] = (uint8_t)jpeg_rgb(c, l, u, v);
}

}  // namespace grl
