"""TEST INFRASTRUCTURE ONLY. The validation step's SSIM (utils/metrics/ssim.py:17-85) restated in NumPy float64, on planes
that already are what the metric receives (tensor_round'ed, shaved, luma taken): (B, C, h, w) values k / 255.

window="2d" is the reference's window, float32(t t^T), with float64 sums; window="separable" is the kernel's form, a pass
along the rows then one down the columns.  The remaining arguments each switch on one deliberate deviation, for the
mutation controls of tests/test_ssim.py.
"""
import math

import numpy as np


def taps(rounded=True):
    t = [math.exp(-((i - 5) ** 2) / 4.5) for i in range(11)]
    t = [round(v, 6) for v in t] if rounded else t
    total = 0.0
    for v in t:  # plain left-to-right additions, as the reference's gauss.sum() comes out (sum() compensates)
        total += v
    return np.asarray(t, np.float64) / total


def _blur(x, t, window, pad):
    h, w = x.shape[-2:]
    xp = np.pad(x, [(0, 0)] * (x.ndim - 2) + [(5, 5), (5, 5)], mode="reflect" if pad == "reflect" else "constant")
    if window == "2d":
        win = np.outer(t, t).astype(np.float32).astype(np.float64)
        return sum(win[i, j] * xp[..., i:i + h, j:j + w] for i in range(11) for j in range(11))
    rows = sum(t[j] * xp[..., :, j:j + w] for j in range(11))
    return sum(t[i] * rows[..., i:i + h, :] for i in range(11))


def ssim_map(a, b, window="separable", pad="zero", renormalise=False, rounded_taps=True, c_scale=1.0):
    a, b, t = np.asarray(a, np.float64), np.asarray(b, np.float64), taps(rounded_taps)
    mass = _blur(np.ones_like(a), t, window, pad) if renormalise else 1.0
    mu_a, mu_b = _blur(a, t, window, pad) / mass, _blur(b, t, window, pad) / mass
    var_a = _blur(a * a, t, window, pad) / mass - mu_a**2
    var_b = _blur(b * b, t, window, pad) / mass - mu_b**2
    cov = _blur(a * b, t, window, pad) / mass - mu_a * mu_b
    c1, c2 = 0.01**2 * c_scale, 0.03**2 * c_scale
    return ((2 * mu_a * mu_b + c1) * (2 * cov + c2)) / ((mu_a**2 + mu_b**2 + c1) * (var_a + var_b + c2))


def ssim(a, b, valid_only=False, **kw):
    """Per-image mean of the map, (B,) float64; valid_only: over the pixels whose window lies inside the image."""
    m = ssim_map(a, b, **kw)
    if valid_only:
        m = m[..., 5:-5, 5:-5]
    return m.mean((-3, -2, -1))
