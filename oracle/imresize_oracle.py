"""TEST INFRASTRUCTURE.  A float64 numpy restatement of the reference's MATLAB bicubic imresize with antialiasing
(utils/matlab_functions.py:20-188) for the integer downscales 1/2, 1/3 and 1/4: exact rational weights (fractions),
rounded once to float64, symmetric padding, the H pass then the W pass with no rounding in between.  It is the reference
point of tests/test_imresize.py and tests/test_gpu_imresize.py and of the fixture check in make_golden_imresize.py.

The keyword arguments of weights() and resize() restate plausible mistakes (the mutation controls of the tests); their
defaults are the reference's algorithm.

Bounds (derived in tests/test_imresize.py's docstring).  With u = 2^-24, P = the resize of |v| with the taps |w|
(abs_resize), T the tap count:
    host copy (float32 taps, float64 sums, one float32 rounding per pass):  ((1 + u)^4 (1 + g)^4 - 1) P,
        g = gamma_{2T+2} in float64;
    reference (its own float32 taps w_r, float32 sums of unknown order):    ((1 + gamma_T)^2 (1 + g)^2 - 1) P_r + E,
        P_r the resize of |v| with |w_r|, gamma_T = T u / (1 - T u), E = the resize of |v| with the tap pairs
        (|w_r| (x) eps + eps (x) |w|), eps = |w_r - w|.
"""
import math
from fractions import Fraction

import numpy as np

SCALES = (2, 3, 4)
U32 = 2.0 ** -24


def _cubic(x):
    a = abs(x)
    if a <= 1:
        return Fraction(3, 2) * a ** 3 - Fraction(5, 2) * a ** 2 + 1
    if a <= 2:
        return -Fraction(1, 2) * a ** 3 + Fraction(5, 2) * a ** 2 - 4 * a + 2
    return Fraction(0)


def weights(s, antialias=True, centre=True, normalise=True, prefactor=True):
    """(taps float64 (T,), c): the one weight row of calculate_weights_indices(n, ceil(n / s), 1 / s, "cubic", 4, True)
    and the 0-based first input of output 0 (output o reads inputs s o + c + k).  Exact in rationals, rounded once.

    antialias=False: kernel width 4 at stride s (the reference's antialiasing=False); centre=False: u = s x without the
    (1 - s) / 2 term; prefactor=False: cubic((u - j) / s) without the 1 / s factor; normalise=False: no division by the
    row sum (with the 1 / s factor the integer-downscale rows already sum to exactly 1)."""
    x = 1  # every output has the same row: take MATLAB's first output
    u = s * x + (Fraction(1 - s, 2) if centre else 0)
    kw = 4 * s if antialias else 4
    left = math.floor(u - Fraction(kw, 2))
    p = kw + 2
    w = []
    for m in range(p):
        d = u - (left + m)
        w.append(((Fraction(1, s) if prefactor else 1) * _cubic(d / s)) if antialias else _cubic(d))
    if normalise:
        total = sum(w)
        w = [v / total for v in w]
    first = 0
    if w[0] == 0:  # the reference narrows (1, p - 2): drops the first AND the last candidate
        w, first = w[1:-1], 1
    elif w[-1] == 0:  # narrow(0, p - 2): drops the last two
        w = w[:-2]
    return np.array([float(v) for v in w]), left + first - 1


def out_size(n, s):
    return -(-n // s)


def pads(n, s, antialias=True, centre=True):
    """The reference's (sym_len_s, sym_len_e) for a side of length n.  Its imresize fails where one exceeds n > 1."""
    w, c = weights(s, antialias, centre)
    return -c, s * (out_size(n, s) - 1) + c + len(w) - n


def _index(n, s, T, c, pad):
    i = s * np.arange(out_size(n, s))[:, None] + c + np.arange(T)[None, :]
    if pad == "edge" or n == 1:  # the reference's copy broadcasts a single sample to every pad
        return np.clip(i, 0, n - 1)
    i = np.mod(i, 2 * n)  # the symmetric copy for -n <= i < 2n, extended periodically for the mutated geometries
    return np.where(i >= n, 2 * n - 1 - i, i)


def apply(v, s, taps_h, taps_w, c, pad="symmetric"):
    """v (C, H, W) float64 -> (C, ceil(H / s), ceil(W / s)): the H pass with taps_h, then the W pass with taps_w, both
    reading inputs s o + c + k; float64 throughout."""
    v = np.asarray(v, dtype=np.float64)
    _, H, W = v.shape
    ih = _index(H, s, len(taps_h), c, pad)
    iw = _index(W, s, len(taps_w), c, pad)
    t = np.einsum("chkw,k->chw", v[:, ih, :], np.asarray(taps_h, np.float64))
    return np.einsum("chwk,k->chw", t[:, :, iw], np.asarray(taps_w, np.float64))


def resize(v, s, antialias=True, centre=True, normalise=True, prefactor=True, shift=0, pad="symmetric"):
    """imresize(v, 1 / s) of v (C, H, W) in float64.  shift: the taps applied `shift` inputs to the left; pad "edge":
    edge replication instead of the symmetric copy."""
    w, c = weights(s, antialias, centre, normalise, prefactor)
    return apply(v, s, w, w, c - shift, pad)


def abs_resize(v, s, taps_h=None, taps_w=None):
    """P: the resize of |v| with |taps| (the reference's taps by default)."""
    w, c = weights(s)
    th = np.abs(w if taps_h is None else taps_h)
    tw = np.abs(w if taps_w is None else taps_w)
    return apply(np.abs(v), s, th, tw, c)


def _gamma(n, unit):
    return n * unit / (1 - n * unit)


def host_bound(v, s):
    T = len(weights(s)[0])
    g = _gamma(2 * T + 2, 2.0 ** -53)
    return ((1 + U32) ** 4 * (1 + g) ** 4 - 1) * abs_resize(v, s)


def reference_bound(v, s, ref_taps):
    w, _ = weights(s)
    T = len(w)
    ref_taps = np.asarray(ref_taps, np.float64)
    eps = np.abs(ref_taps - w)
    g = _gamma(2 * T + 2, 2.0 ** -53)
    main = ((1 + _gamma(T, U32)) ** 2 * (1 + g) ** 2 - 1) * abs_resize(v, s, ref_taps, ref_taps)
    taps_err = abs_resize(v, s, ref_taps, eps) + abs_resize(v, s, eps, w)
    return main + taps_err * (1 + g) ** 2
