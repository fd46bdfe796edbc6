"""TEST INFRASTRUCTURE ONLY. A vectorised NumPy restatement of the reference's NIQE (utils/metrics/niqe.py:341-546) with
its fp32 storage points, used to pin the device kernels stage by stage.

Storage points follow the reference: the luma chain of csrc/grl_niqe.h; the 7 x 7 "nearest" convolutions accumulated in
float64 over the flipped window in row-major order (scipy.ndimage.convolve's footprint order) and stored to fp32; mu^2,
the difference, abs, sqrt and the MSCN quotient in fp32; the x0.5 resize of img / 255 (fp32) with float64 accumulation
stored to fp32 per pass, times 255 in fp32; the products of the np.roll-shifted block in fp32.  The AGGD moments are
float64 (the reference takes fp32 means, so the two differ by about 1e-7 relative), and every fit also reports its
margin: how far rhatnorm lies from the nearest decision midpoint of the r_gam table, which bounds how large a moment
error the chosen alpha survives.
"""
import numpy as np

GAM_N = 9801
SHIFTS = ((0, 1), (1, 0), (1, 1), (1, -1))


def tables():
    """(gam, r_gam, sqrt(G(1/a)/G(3/a)), G(2/a)/G(1/a)) as the product builds them (metrics.niqe_tables)."""
    import math

    start = 0.2
    delta = (start + 0.001) - start
    gam = np.array([start] + [start + i * delta for i in range(1, GAM_N)])
    g = math.gamma
    r_gam = np.array([g(2 * (1.0 / a)) ** 2 / (g(1.0 / a) * g(3 * (1.0 / a))) for a in gam])
    bfac = np.array([math.sqrt(g(1 / a) / g(3 / a)) for a in gam])
    mfac = np.array([g(2 / a) / g(1 / a) for a in gam])
    return gam, r_gam, bfac, mfac


def luma(rgb8):
    """(..., 3) uint8 RGB -> fp32 rounded luma, the chain of calculate_niqe on tensor_round'ed data (BGR weights)."""
    p = rgb8.astype(np.float32) / np.float32(255.0)
    u = (p * np.float32(255.0)) / np.float32(255.0)
    u = u.astype(np.float64)
    d = u[..., 0] * 24.966 + u[..., 1] * 128.553
    d = d + u[..., 2] * 65.481
    d = d + 16.0
    return np.round((d / 255.0).astype(np.float32) * np.float32(255.0))


def crop(y, border):
    if border:
        y = y[border:-border, border:-border]
    h, w = y.shape
    return y[: h // 96 * 96, : w // 96 * 96]


def conv7(img, win):
    """scipy.ndimage.convolve(img, win, mode="nearest") for fp32 img: float64 sum over the flipped window, row-major."""
    h, w = img.shape
    pad = np.pad(img, 3, mode="edge").astype(np.float64)
    wf = win[::-1, ::-1]
    acc = np.zeros((h, w))
    for i in range(7):
        for j in range(7):
            acc = acc + pad[i:i + h, j:j + w] * wf[i, j]
    return acc.astype(np.float32)


def mscn(img, win):
    mu = conv7(img, win)
    sigma = np.sqrt(np.abs(conv7(np.square(img), win) - np.square(mu)))
    return (img - mu) / (sigma + np.float32(1))


HALF_TAPS = np.array([-0.01171875, -0.03515625, 0.11328125, 0.43359375, 0.43359375, 0.11328125, -0.03515625, -0.01171875],
                     np.float32)


def _sym(i, n):
    return np.where(i < 0, -1 - i, np.where(i >= n, 2 * n - 1 - i, i))


def half(img):
    """255 * imresize(img / 255, 0.5): rows then columns, 8 taps, symmetric padding, float64 sums stored to fp32."""
    t = img / np.float32(255.0)
    h, w = t.shape
    taps = HALF_TAPS.astype(np.float64)
    rows = _sym(2 * np.arange(h // 2)[:, None] - 3 + np.arange(8)[None, :], h)  # (h/2, 8)
    a = np.zeros((h // 2, w))
    for k in range(8):
        a = a + taps[k] * t[rows[:, k], :].astype(np.float64)
    a = a.astype(np.float32)
    cols = _sym(2 * np.arange(w // 2)[:, None] - 3 + np.arange(8)[None, :], w)
    b = np.zeros((h // 2, w // 2))
    for k in range(8):
        b = b + taps[k] * a[:, cols[:, k]].astype(np.float64)
    return b.astype(np.float32) * np.float32(255.0)


def blocks(m, bs):
    """(nbw * nbh, bs, bs): block iw * nbh + ih (niqe.py:458-465)."""
    h, w = m.shape
    nbh, nbw = h // bs, w // bs
    return m.reshape(nbh, bs, nbw, bs).transpose(2, 0, 1, 3).reshape(nbw * nbh, bs, bs)


def aggd(x, tab):
    """Vectorised estimate_aggd_param over rows of x (n, N) fp32 -> (idx, left_std, right_std, margin)."""
    _, r_gam, _, _ = tab
    d = x.astype(np.float64)
    neg, pos = d < 0, d > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        lstd = np.sqrt((d * d * neg).sum(1) / neg.sum(1))
        rstd = np.sqrt((d * d * pos).sum(1) / pos.sum(1))
        g = lstd / rstd
        n = d.shape[1]
        rhat = (np.abs(d).sum(1) / n) ** 2 / ((d * d).sum(1) / n)
        rn = rhat * (g ** 3 + 1) * (g + 1) / ((g ** 2 + 1) ** 2)
        idx = np.argmin((r_gam[None, :] - rn[:, None]) ** 2, axis=1)  # all-NaN rows -> 0, like the reference
        mids = (r_gam[1:] + r_gam[:-1]) / 2
        lo = np.where(idx > 0, np.abs(rn - mids[np.maximum(idx - 1, 0)]), np.inf)
        hi = np.where(idx < GAM_N - 1, np.abs(rn - mids[np.minimum(idx, GAM_N - 2)]), np.inf)
        margin = np.where(np.isnan(rn), np.inf, np.minimum(lo, hi))
    return idx, lstd, rstd, margin


def features(m, bs, tab):
    """(n, 18) features of every block of the MSCN image m and the (n, 5) fit margins (compute_feature, niqe.py:373-397)."""
    gam, _, bfac, mfac = tab
    blk = blocks(m, bs)
    n = blk.shape[0]
    out = np.empty((n, 18))
    margins = np.empty((n, 5))
    idx, ls, rs, margins[:, 0] = aggd(blk.reshape(n, -1), tab)
    out[:, 0] = gam[idx]
    out[:, 1] = (ls * bfac[idx] + rs * bfac[idx]) / 2
    for s, sh in enumerate(SHIFTS):
        prod = blk * np.roll(blk, sh, axis=(1, 2))
        idx, ls, rs, margins[:, 1 + s] = aggd(prod.reshape(n, -1), tab)
        bl, br = ls * bfac[idx], rs * bfac[idx]
        out[:, 2 + 4 * s], out[:, 3 + 4 * s], out[:, 4 + 4 * s], out[:, 5 + 4 * s] = gam[idx], (br - bl) * mfac[idx], bl, br
    return out, margins


def distance(feats, mu_pris, cov_pris):
    """niqe.py:475-490 on one image's (n, 36) features."""
    mu = np.nanmean(feats, axis=0)
    ok = feats[~np.isnan(feats).any(axis=1)]
    cov = np.cov(ok, rowvar=False)
    inv = np.linalg.pinv((cov_pris + cov) / 2)
    d = mu_pris - mu
    return float(np.sqrt(np.squeeze(d @ inv @ d.T)))


def niqe(rgb8, params, border=0, tab=None):
    """Every stage of one image's NIQE: rgb8 (3, H, W) uint8 -> dict(y, mscn1, half, mscn2, feats, margins, score)."""
    tab = tab or tables()
    win = params["gaussian_window"]
    y = crop(luma(np.moveaxis(rgb8, 0, -1)), border)
    m1 = mscn(y, win)
    y2 = half(y)
    m2 = mscn(y2, win)
    f1, g1 = features(m1, 96, tab)
    f2, g2 = features(m2, 48, tab)
    feats = np.concatenate([f1, f2], axis=1)
    return dict(y=y, mscn1=m1, half=y2, mscn2=m2, feats=feats, margins=np.concatenate([g1, g2], axis=1),
                score=distance(feats, params["mu_pris_param"], params["cov_pris_param"]))
