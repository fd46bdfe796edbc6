"""Integer restatement of the baseline JPEG round trip  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The JPEG test command degrades every clean test image with JPEGDataset.jpeg_compress
(data/datasets/restoration_jpeg.py:62-79): cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q]) then cv2.imdecode, i.e.
libjpeg's default baseline encoder (4:2:0 for colour, islow DCT) and its default decoder (islow IDCT, "fancy" h2v2
upsampling).  Entropy coding is lossless, so the pixels are a function of the integer arithmetic below, restated in numpy
from ITU T.81 and libjpeg's documented integer algorithms.  oracle/make_golden_jpeg.py checks both halves of it against
the codec (tables and coefficients parsed from the codec's bitstream by oracle/jpeg_bitstream.py, pixels from cv2) and
writes tests/golden/jpeg_*.  Only tests/ and oracle/ import this file.

Images are uint8 (H, W, C), C = 1 (one gray component) or 3 (RGB, converted to YCbCr, chroma subsampled 2 x 2).
"""
import numpy as np

# ITU T.81 Annex K.1, tables K.1 (luminance) and K.2 (chrominance), natural (row-major) order
STD_LUMA = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], dtype=np.int64)
STD_CHROMA = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32, dtype=np.int64)

# zigzag position k -> natural index (ITU T.81 figure A.6)
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
    47, 55, 62, 63], dtype=np.int64)

CONST_BITS, PASS1_BITS = 13, 2
SCALEBITS = 16
ONE_HALF = 1 << (SCALEBITS - 1)


def FIX(x, bits=SCALEBITS):
    return int(x * (1 << bits) + 0.5)


# islow constants, FIX(x) at CONST_BITS = 13
F_0_298, F_0_390, F_0_541, F_0_765 = 2446, 3196, 4433, 6270
F_0_899, F_1_175, F_1_501, F_1_847 = 7373, 9633, 12299, 15137
F_1_961, F_2_053, F_2_562, F_3_072 = 16069, 16819, 20995, 25172


def quant_tables(q):
    """(luma, chroma) int64 (64,) natural order: jpeg_set_quality(q, force_baseline=TRUE)."""
    if not 1 <= int(q) <= 100:
        raise ValueError(f"quality must be in 1..100, got {q}")
    q = int(q)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return tuple(np.clip((t * scale + 50) // 100, 1, 255) for t in (STD_LUMA, STD_CHROMA))


def rgb_to_ycc(rgb):
    """(H, W, 3) -> three int64 planes, 16-bit fixed point (rounding 0.5 - epsilon on Cb / Cr)."""
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    y = (FIX(0.299) * r + FIX(0.587) * g + FIX(0.114) * b + ONE_HALF) >> SCALEBITS
    cb = (-FIX(0.16874) * r - FIX(0.33126) * g + FIX(0.5) * b + (128 << SCALEBITS) + ONE_HALF - 1) >> SCALEBITS
    cr = (FIX(0.5) * r - FIX(0.41869) * g - FIX(0.08131) * b + (128 << SCALEBITS) + ONE_HALF - 1) >> SCALEBITS
    return y, cb, cr


def ycc_to_rgb(y, cb, cr):
    """Three int64 planes -> (H, W, 3) uint8."""
    cb, cr = cb - 128, cr - 128
    r = y + ((FIX(1.402) * cr + ONE_HALF) >> SCALEBITS)
    g = y + ((-FIX(0.34414) * cb - FIX(0.71414) * cr + ONE_HALF) >> SCALEBITS)
    b = y + ((FIX(1.772) * cb + ONE_HALF) >> SCALEBITS)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def downsample_h2v2(p):
    """(2h, 2w) -> (h, w): the 2 x 2 sum plus a bias of 1, 2, 1, 2, ... along each output row, >> 2."""
    s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
    bias = 1 + (np.arange(s.shape[1]) & 1)
    return (s + bias[None, :]) >> 2


def upsample_h2v2(c, H, W):
    """Decoder chroma (h2, w2) real samples -> (H, W).  Fancy (triangle) upsampling with the component's edge samples
    replicated, except for components at most 2 samples wide, which libjpeg upsamples by plain replication."""
    h2, w2 = c.shape
    if w2 <= 2:
        return np.repeat(np.repeat(c, 2, 0), 2, 1)[:H, :W]
    up = np.concatenate([c[:1], c[:-1]], 0)
    dn = np.concatenate([c[1:], c[-1:]], 0)
    rows = np.empty((2 * h2, w2), np.int64)
    rows[0::2] = 3 * c + up
    rows[1::2] = 3 * c + dn
    left = np.concatenate([rows[:, :1], rows[:, :-1]], 1)
    right = np.concatenate([rows[:, 1:], rows[:, -1:]], 1)
    out = np.empty((2 * h2, 2 * w2), np.int64)
    out[:, 0::2] = (3 * rows + left + 8) >> 4
    out[:, 1::2] = (3 * rows + right + 7) >> 4
    return out[:H, :W]


def _fdct_1d(d, first):
    """One islow pass along the last axis; first = the row pass (output scaled up by PASS1_BITS)."""
    d = [d[..., i] for i in range(8)]
    tmp0, tmp7 = d[0] + d[7], d[0] - d[7]
    tmp1, tmp6 = d[1] + d[6], d[1] - d[6]
    tmp2, tmp5 = d[2] + d[5], d[2] - d[5]
    tmp3, tmp4 = d[3] + d[4], d[3] - d[4]
    tmp10, tmp13 = tmp0 + tmp3, tmp0 - tmp3
    tmp11, tmp12 = tmp1 + tmp2, tmp1 - tmp2
    sh = CONST_BITS - PASS1_BITS if first else CONST_BITS + PASS1_BITS

    def ds(x, n):
        return (x + (1 << (n - 1))) >> n

    out = [None] * 8
    if first:
        out[0], out[4] = (tmp10 + tmp11) << PASS1_BITS, (tmp10 - tmp11) << PASS1_BITS
    else:
        out[0], out[4] = ds(tmp10 + tmp11, PASS1_BITS), ds(tmp10 - tmp11, PASS1_BITS)
    z1 = (tmp12 + tmp13) * F_0_541
    out[2] = ds(z1 + tmp13 * F_0_765, sh)
    out[6] = ds(z1 - tmp12 * F_1_847, sh)
    z1, z2, z3, z4 = tmp4 + tmp7, tmp5 + tmp6, tmp4 + tmp6, tmp5 + tmp7
    z5 = (z3 + z4) * F_1_175
    tmp4, tmp5, tmp6, tmp7 = tmp4 * F_0_298, tmp5 * F_2_053, tmp6 * F_3_072, tmp7 * F_1_501
    z1, z2, z3, z4 = -z1 * F_0_899, -z2 * F_2_562, -z3 * F_1_961 + z5, -z4 * F_0_390 + z5
    out[7] = ds(tmp4 + z1 + z3, sh)
    out[5] = ds(tmp5 + z2 + z4, sh)
    out[3] = ds(tmp6 + z2 + z3, sh)
    out[1] = ds(tmp7 + z1 + z4, sh)
    return np.stack(out, -1)


def fdct(blocks):
    """(..., 8, 8) samples 0..255 -> 8 x the 2-D DCT of (sample - 128), islow integer arithmetic: rows, then columns."""
    d = blocks.astype(np.int64) - 128
    d = _fdct_1d(d, True)
    return np.swapaxes(_fdct_1d(np.swapaxes(d, -1, -2), False), -1, -2)


def quantize(coef, qv):
    """coef (..., 8, 8) from fdct, qv (64,) natural order: coef / (8 qv) rounded half away from zero."""
    div = (8 * qv).reshape(8, 8)
    a = np.abs(coef)
    return np.sign(coef) * ((a + (div >> 1)) // div)


def _idct_1d(z, first):
    """One islow pass along the last axis; first = the column pass on dequantised coefficients."""
    z = [z[..., i] for i in range(8)]
    a1 = (z[2] + z[6]) * F_0_541
    tmp2 = a1 - z[6] * F_1_847
    tmp3 = a1 + z[2] * F_0_765
    tmp0 = (z[0] + z[4]) << CONST_BITS
    tmp1 = (z[0] - z[4]) << CONST_BITS
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = z[7], z[5], z[3], z[1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F_1_175
    t0, t1, t2, t3 = t0 * F_0_298, t1 * F_2_053, t2 * F_3_072, t3 * F_1_501
    z1, z2, z3, z4 = -z1 * F_0_899, -z2 * F_2_562, -z3 * F_1_961 + z5, -z4 * F_0_390 + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    n = CONST_BITS - PASS1_BITS if first else CONST_BITS + PASS1_BITS + 3
    r = 1 << (n - 1)
    out = [tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0, tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3]
    return np.stack([(v + r) >> n for v in out], -1)


def idct(qcoef, qv):
    """(..., 8, 8) quantised coefficients, qv (64,) -> samples: dequantise, islow columns then rows, + 128 clamped to
    0..255."""
    z = qcoef.astype(np.int64) * qv.reshape(8, 8)
    w = np.swapaxes(_idct_1d(np.swapaxes(z, -1, -2), True), -1, -2)
    return np.clip(_idct_1d(w, False) + 128, 0, 255)


def _blocks(p):
    h, w = p.shape
    return p.reshape(h // 8, 8, w // 8, 8).swapaxes(1, 2)


def _unblocks(b):
    nh, nw = b.shape[:2]
    return b.swapaxes(1, 2).reshape(nh * 8, nw * 8)


def _ceil(a, b):
    return -(-a // b)


def component_blocks(H, W, C):
    """[(rows, cols) of coded blocks] per component, without the MCU's dummy blocks."""
    if C == 1:
        return [(_ceil(H, 8), _ceil(W, 8))]
    hc, wc = _ceil(H, 2), _ceil(W, 2)
    return [(_ceil(H, 8), _ceil(W, 8))] + [(_ceil(hc, 8), _ceil(wc, 8))] * 2


def encode(img, q):
    """uint8 (H, W, C) -> [quantised coefficients (rows, cols, 8, 8) int64 per component] (coded blocks only)."""
    H, W, C = img.shape
    lq, cq = quant_tables(q)
    m = 8 if C == 1 else 16
    Hp, Wp = _ceil(H, m) * m, _ceil(W, m) * m
    # The codec replicates the last column up to the MCU width and the last row up to an even height before it
    # downsamples; below that it replicates the last row of each component, i.e. the last DOWNSAMPLED chroma row (which
    # differs from downsampling replicated full-resolution rows when H is even).
    H2 = _ceil(H, 2) * 2 if C == 3 else H
    pad = np.pad(img, ((0, H2 - H), (0, Wp - W), (0, 0)), mode="edge")
    if C == 1:
        planes, tables = [pad[..., 0].astype(np.int64)], [lq]
    else:
        y, cb, cr = rgb_to_ycc(pad)
        planes, tables = [y, downsample_h2v2(cb), downsample_h2v2(cr)], [lq, cq, cq]
    planes = [np.pad(p, ((0, Hp * len(p) // H2 - len(p)), (0, 0)), mode="edge") for p in planes]
    out = []
    for p, qv, (nh, nw) in zip(planes, tables, component_blocks(H, W, C)):
        out.append(quantize(fdct(_blocks(p)), qv)[:nh, :nw])
    return out


def decode(coefs, tables, H, W):
    """[quantised coefficients per component], [qv (64,) per component] -> uint8 (H, W, C)."""
    planes = [_unblocks(idct(c, qv)) for c, qv in zip(coefs, tables)]
    if len(planes) == 1:
        return planes[0][:H, :W, None].astype(np.uint8)
    hc, wc = _ceil(H, 2), _ceil(W, 2)
    cb, cr = (upsample_h2v2(p[:hc, :wc], H, W) for p in planes[1:])
    return ycc_to_rgb(planes[0][:H, :W], cb, cr)


CONTENTS = ("random", "ramp", "edges", "saturated")


def synth_image(content, H, W, C, seed):
    """Seeded uint8 (H, W, C) test content: uniform noise; smooth ramps; hard-edged flat cells; or 0 / 255 regions
    with a little noise (the range limits of both colour conversions and of the IDCT)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    if content == "random":
        return rng.integers(0, 256, (H, W, C), dtype=np.uint8)
    if content == "ramp":
        a, b = rng.uniform(-6, 6, (2, C))
        off = rng.uniform(0, 255, C)
        return np.clip(off + a * yy[..., None] + b * xx[..., None], 0, 255).astype(np.uint8)
    if content == "edges":
        cell = int(rng.integers(3, 7))
        colours = rng.integers(0, 256, (H // cell + 1, W // cell + 1, C), dtype=np.uint8)
        return colours[yy // cell, xx // cell]
    if content == "saturated":
        lo = rng.integers(0, 256, C) < 128
        mask = (yy * rng.uniform(-1, 1) + xx * rng.uniform(-1, 1) + rng.uniform(-4, 4)) > 0
        img = np.where(mask[..., None], np.where(lo, 0, 255), np.where(lo, 255, 0)).astype(np.int64)
        img += rng.integers(-3, 4, (H, W, C)) * (rng.random((H, W, 1)) < 0.1)
        return np.clip(img, 0, 255).astype(np.uint8)
    raise ValueError(f"unknown content {content!r}")


def roundtrip(img, q):
    """jpeg_compress of one uint8 (H, W, C) image, C in {1, 3}."""
    H, W, C = img.shape
    lq, cq = quant_tables(q)
    return decode(encode(img, q), [lq] if C == 1 else [lq, cq, cq], H, W)
