"""The image-quality numbers the reference's validation step reports, evaluated on the device the images live on.

Reference: engines/base.py:255-268 (round -> shave for SR -> metrics), utils/utils_image.py:8-11 (shave), :30-33
(tensor_round), :43-80 (rgb2ycbcr, MATLAB coefficients, rounded to 8 bit), utils/metrics/psnr.py:44-48 (psnr),
utils/metrics/ssim.py:17-82 (Gaussian-window SSIM, 11 taps, sigma 1.5, taps rounded to 6 decimals, zero padding).
psnr_fused() is the hand-written kernel (csrc/metric.cu, grl_psnr_f32) the benchmarked validation step uses for PSNR
(RGB and luma); the torch-op functions below define the same quantities on any device (SSIM stays torch ops) and are
what the CPU tests pin against the reference's own functions.
"""
import math

import torch
import torch.nn.functional as F


def tensor_round(img, data_range=1.0):
    img = img.clamp(0.0, 1.0 * data_range)
    return (img * 255.0 / data_range).round() * data_range / 255.0


def shave(img, border):
    return img[..., border:-border, border:-border] if border > 0 else img


def rgb_to_y(img, data_range=1.0):
    """Luma of MATLAB's rgb2ycbcr on (B, 3, H, W), rounded to the 8-bit grid, returned as (B, 1, H, W)."""
    scale = 255.0 if data_range == 1.0 else 1.0
    coeff = torch.tensor([65.481, 128.553, 24.966], device=img.device, dtype=img.dtype) / 255.0
    y = (img * scale).permute(0, 2, 3, 1) @ coeff + 16.0
    y = y.round().unsqueeze(1)
    return y / 255.0 if data_range == 1 else y


def psnr(restored, target, border=0, channel="rgb"):
    """Per-image PSNR (B,) of 8-bit-rounded tensors, `border` pixels shaved (SR: border = scale), RGB or luma."""
    a, b = shave(tensor_round(restored), border), shave(tensor_round(target), border)
    if channel == "y":
        a, b = rgb_to_y(a), rgb_to_y(b)
    return -10 * (a - b).pow(2).mean([-3, -2, -1]).log10()


def psnr_fused(restored, target, border=0):
    """(psnr_rgb, psnr_y), each (B,), from ONE fused kernel over CUDA fp32 (B, C, H, W) images: tensor_round + shave +
    exact integer squared-error reduction (csrc/metric.cu).  No torch math on the images."""
    from . import capi

    capi.require_device(restored)
    capi.require_device(target)
    if restored.shape != target.shape or restored.dim() != 4:
        raise RuntimeError(f"grl_b200: psnr_fused needs two (B, C, H, W) tensors of one shape, got {tuple(restored.shape)} / {tuple(target.shape)}")
    a = restored if (restored.dtype == torch.float32 and restored.is_contiguous()) else restored.float().contiguous()
    b = target if (target.dtype == torch.float32 and target.is_contiguous()) else target.float().contiguous()
    B, C, H, W = a.shape
    ws = torch.empty(2 * max(B, 1), device=a.device, dtype=torch.int64)
    out = torch.empty(2, B, device=a.device, dtype=torch.float32)
    capi.check(capi.lib().grl_psnr_f32(capi.ptr(a), capi.ptr(b), B, C, H, W, int(border), capi.ptr(ws), ws.numel() * 8,
                                       capi.ptr(out[0]), capi.ptr(out[1]), capi.stream()))
    return out[0], out[1]


def _gaussian_window(channels, size, sigma, like):
    taps = torch.tensor([round(math.exp(-((i - size // 2) ** 2) / (2.0 * sigma**2)), 6) for i in range(size)],
                        dtype=torch.float64)
    taps = taps / taps.sum()
    win = torch.outer(taps, taps).float()
    return win.expand(channels, 1, size, size).contiguous().to(device=like.device, dtype=like.dtype)


def ssim(restored, target, border=0, channel="rgb", window_size=11, sigma=1.5):
    """Per-image SSIM (B,): mean of the SSIM map over channels and pixels (zero-padded Gaussian local statistics)."""
    a, b = shave(tensor_round(restored), border), shave(tensor_round(target), border)
    if channel == "y":
        a, b = rgb_to_y(a), rgb_to_y(b)
    c = a.shape[1]
    win = _gaussian_window(c, window_size, sigma, a)

    def blur(t):
        return F.conv2d(t, win, padding=window_size // 2, groups=c)

    mu_a, mu_b = blur(a), blur(b)
    var_a, var_b, cov = blur(a * a) - mu_a.pow(2), blur(b * b) - mu_b.pow(2), blur(a * b) - mu_a * mu_b
    c1, c2 = 0.01**2, 0.03**2
    ssim_map = ((2 * mu_a * mu_b + c1) * (2 * cov + c2)) / ((mu_a.pow(2) + mu_b.pow(2) + c1) * (var_a + var_b + c2))
    return ssim_map.mean([-3, -2, -1])


def _grid8(img):
    """(B, C, H, W) image on the 8-bit grid (k / 255) -> the integers k as float64."""
    return (img * 255.0).round().double()


def _blocking_effect_factor(k):
    """bef of one channel (B, H, W) of 8-bit integers, in units of 1 / 255^2 (utils/metrics/psnrb.py:22-101).  The
    normalisers are the reference's formulas, H * (W // 8 - 1) and the rest of H * (W - 1), not the number of positions
    the sums run over (arange(7, W - 1, 8) holds one column more when W % 8 > 0)."""
    H, W = k.shape[-2:]
    dh = (k[..., :, :-1] - k[..., :, 1:]).pow(2)  # pair (x, x + 1) at column x
    dv = (k[..., :-1, :] - k[..., 1:, :]).pow(2)
    bh = torch.arange(W - 1, device=k.device) % 8 == 7
    bv = torch.arange(H - 1, device=k.device) % 8 == 7
    n_bh, n_bv = H * (W // 8 - 1), W * (H // 8 - 1)
    n_nh, n_nv = H * (W - 1) - n_bh, W * (H - 1) - n_bv
    boundary = (dh[..., bh].sum((-2, -1)) + dv[..., bv, :].sum((-2, -1))) / (n_bh + n_bv)
    other = (dh[..., ~bh].sum((-2, -1)) + dv[..., ~bv, :].sum((-2, -1))) / (n_nh + n_nv)
    scaler = math.log2(8) / math.log2(min(H, W))
    return torch.where(boundary <= other, torch.zeros_like(boundary), scaler * (boundary - other))


def psnrb(restored, target, channel="rgb"):
    """Per-image PSNR-B (B,) float64 of the JPEG test commands (PeakSignalNoiseRatioBlock.update, psnrb.py:104-163) on
    tensor_round'ed images: per channel 10 log10(1 / (mse + bef)) with the blocking-effect factor of the RESTORED image
    only, averaged in dB over the channels.  channel="y": on the luma of rgb_to_y.  Sums are taken on the 8-bit integers,
    exactly as the fused kernel takes them."""
    if restored.shape != target.shape or restored.dim() != 4:
        raise RuntimeError(f"grl_b200: psnrb needs two (B, C, H, W) tensors of one shape, got {tuple(restored.shape)} / {tuple(target.shape)}")
    if min(restored.shape[-2:]) < 16:
        raise RuntimeError(f"grl_b200: psnrb needs at least 16 x 16 pixels, got {tuple(restored.shape[-2:])}")
    a, b = tensor_round(restored), tensor_round(target)
    if channel == "y":
        if a.shape[1] != 3:
            raise RuntimeError("grl_b200: psnrb(channel='y') needs RGB images")
        a, b = rgb_to_y(a), rgb_to_y(b)
    ka, kb = _grid8(a), _grid8(b)
    mse = (ka - kb).pow(2).mean((-2, -1))  # (B, C), units of 1 / 255^2
    bef = _blocking_effect_factor(ka)
    return (10 * torch.log10(65025.0 / (mse + bef))).mean(1)


def psnrb_fused(restored, target):
    """(psnrb_rgb, psnrb_y), each (B,) float64, from one fused kernel over CUDA fp32 (B, C, H, W) images, C = 1 or 3
    (csrc/metric.cu, grl_psnrb_f32); psnrb_y is a copy of psnrb_rgb for C = 1."""
    from . import capi

    capi.require_device(restored)
    capi.require_device(target)
    if restored.shape != target.shape or restored.dim() != 4:
        raise RuntimeError(f"grl_b200: psnrb_fused needs two (B, C, H, W) tensors of one shape, got {tuple(restored.shape)} / {tuple(target.shape)}")
    a = restored if (restored.dtype == torch.float32 and restored.is_contiguous()) else restored.float().contiguous()
    b = target if (target.dtype == torch.float32 and target.is_contiguous()) else target.float().contiguous()
    B, C, H, W = a.shape
    nbytes = capi.lib().grl_psnrb_workspace(B)
    ws = torch.empty(max(nbytes // 8, 1), device=a.device, dtype=torch.int64)
    out = torch.empty(2, B, device=a.device, dtype=torch.float64)
    capi.check(capi.lib().grl_psnrb_f32(capi.ptr(a), capi.ptr(b), B, C, H, W, capi.ptr(ws), ws.numel() * 8,
                                        capi.ptr(out[0]), capi.ptr(out[1]), capi.stream()))
    return out[0], out[1]


NIQE_GAM = 9801  # gam = 0.2 : 0.001 : 10 (utils/metrics/niqe.py:352)


def niqe_gam():
    """np.arange(0.2, 10.001, 0.001) value for value: NumPy fills start + i * (second - first)."""
    start = 0.2
    delta = (start + 0.001) - start
    return [start] + [start + i * delta for i in range(1, NIQE_GAM)]


def niqe_tables():
    """(4, 9801) float64 host tensor: gam, r_gam (niqe.py:353-356, 1/g computed first), sqrt(G(1/a) / G(3/a)) (:368) and
    G(2/a) / G(1/a) (:395), built with math.gamma."""
    g = math.gamma
    rows = [[], [], [], []]
    for a in niqe_gam():
        r = 1.0 / a
        rows[0].append(a)
        rows[1].append(g(r * 2) ** 2 / (g(r) * g(r * 3)))
        rows[2].append(math.sqrt(g(1 / a) / g(3 / a)))
        rows[3].append(g(2 / a) / g(1 / a))
    return torch.tensor(rows, dtype=torch.float64)


_niqe_cache = {}


def _niqe_device_tables(device):
    key = ("tables", device)
    if key not in _niqe_cache:
        _niqe_cache[key] = niqe_tables().to(device)
    return _niqe_cache[key]


def niqe_params(params):
    """The pristine model: a path to the reference's niqe_pris_params.npz or a mapping with its three arrays ->
    (mu_pris (1, 36), cov_pris (36, 36), gaussian_window (7, 7)) float64 host tensors."""
    if isinstance(params, (str, bytes)) or hasattr(params, "__fspath__"):
        import numpy as np

        with np.load(params) as f:
            params = {k: f[k] for k in ("mu_pris_param", "cov_pris_param", "gaussian_window")}
    out = []
    for k, shape in (("mu_pris_param", (1, 36)), ("cov_pris_param", (36, 36)), ("gaussian_window", (7, 7))):
        t = torch.as_tensor(params[k], dtype=torch.float64).cpu()
        if tuple(t.shape) != shape:
            raise RuntimeError(f"grl_b200: niqe parameter {k} has shape {tuple(t.shape)}, expected {shape}")
        out.append(t.contiguous())
    return tuple(out)


def _niqe_check(restored, border):
    from . import capi

    capi.require_device(restored)
    if restored.dim() != 4 or restored.shape[1] != 3:
        raise RuntimeError(f"grl_b200: niqe needs (B, 3, H, W) RGB images, got {tuple(restored.shape)}")
    if min(restored.shape[-2:]) - 2 * border < 96:
        raise RuntimeError(f"grl_b200: niqe needs at least 96 x 96 pixels after cropping border {border}, got {tuple(restored.shape[-2:])}")
    return restored if (restored.dtype == torch.float32 and restored.is_contiguous()) else restored.float().contiguous()


def niqe_features(restored, params, border=0):
    """(B, nblocks, 36) float64 per-block features (niqe.py:445-473) from the device kernels (csrc/niqe.cu)."""
    import ctypes

    from . import capi

    _, _, win = niqe_params(params)
    x = _niqe_check(restored, border)
    B, C, H, W = x.shape
    nb = ((H - 2 * border) // 96) * ((W - 2 * border) // 96)
    nbytes = capi.lib().grl_niqe_workspace(B, H, W, int(border))
    ws = torch.empty(max(nbytes, 1), device=x.device, dtype=torch.uint8)
    feats = torch.empty(B, nb, 36, device=x.device, dtype=torch.float64)
    win_host = (ctypes.c_double * 49)(*win.flatten().tolist())
    capi.check(capi.lib().grl_niqe_features_f32(capi.ptr(x), B, C, H, W, int(border), win_host,
                                                capi.ptr(_niqe_device_tables(x.device)), capi.ptr(ws), ws.numel(),
                                                capi.ptr(feats), capi.stream()))
    return feats


def niqe_stages(restored, params, border=0):
    """The intermediate images of niqe_features, one stage entry point each (tests): dict of y (B, Hc, Wc), mscn1,
    half (B, Hc/2, Wc/2), mscn2 and feats."""
    import ctypes

    from . import capi

    _, _, win = niqe_params(params)
    x = _niqe_check(restored, border)
    B, C, H, W = x.shape
    Hc, Wc = (H - 2 * border) // 96 * 96, (W - 2 * border) // 96 * 96
    win_host = (ctypes.c_double * 49)(*win.flatten().tolist())
    f32 = dict(device=x.device, dtype=torch.float32)
    s = {"y": torch.empty(B, Hc, Wc, **f32), "mscn1": torch.empty(B, Hc, Wc, **f32), "tmp": torch.empty(B, Hc // 2, Wc, **f32),
         "half": torch.empty(B, Hc // 2, Wc // 2, **f32), "mscn2": torch.empty(B, Hc // 2, Wc // 2, **f32),
         "feats": torch.empty(B, (Hc // 96) * (Wc // 96), 36, device=x.device, dtype=torch.float64)}
    L, st = capi.lib(), capi.stream()
    capi.check(L.grl_niqe_luma_f32(capi.ptr(x), B, C, H, W, int(border), capi.ptr(s["y"]), st))
    capi.check(L.grl_niqe_mscn_f32(capi.ptr(s["y"]), B, Hc, Wc, win_host, capi.ptr(s["mscn1"]), st))
    capi.check(L.grl_niqe_half_f32(capi.ptr(s["y"]), B, Hc, Wc, capi.ptr(s["tmp"]), capi.ptr(s["half"]), st))
    capi.check(L.grl_niqe_mscn_f32(capi.ptr(s["half"]), B, Hc // 2, Wc // 2, win_host, capi.ptr(s["mscn2"]), st))
    capi.check(L.grl_niqe_feat_f32(capi.ptr(s["mscn1"]), capi.ptr(s["mscn2"]), B, Hc // 96, Wc // 96,
                                   capi.ptr(_niqe_device_tables(x.device)), capi.ptr(s["feats"]), st))
    del s["tmp"]
    return s


def niqe_distance(feats, mu_pris, cov_pris):
    """NIQE score (B,) float64 from per-block features (B, n, 36) (niqe.py:475-490): nanmean over blocks, the covariance
    (ddof 1) of the blocks without NaN, pinv of the mean of the two covariances with NumPy's cutoff (1e-15 times the largest
    singular value), the quadratic form, sqrt.  Batched over images, no host synchronisation.  An image with fewer than two
    NaN-free blocks has no covariance and scores NaN."""
    mu_pris = mu_pris.to(feats.device, torch.float64)
    cov_pris = cov_pris.to(feats.device, torch.float64)
    mu = torch.nanmean(feats, dim=1)
    ok = ~torch.isnan(feats).any(dim=2, keepdim=True)
    m = ok.sum(1, keepdim=True).double()
    zero = torch.zeros((), dtype=feats.dtype, device=feats.device)
    mean = torch.where(ok, feats, zero).sum(1, keepdim=True) / m
    xc = torch.where(ok, feats - mean, zero)
    enough = (m > 1).reshape(-1)
    cov = xc.transpose(1, 2) @ xc / (m - 1).clamp_min(1)
    inv = torch.linalg.pinv((cov_pris + cov) / 2, rtol=1e-15)
    d = (mu_pris - mu).unsqueeze(1)
    q = (d @ inv @ d.transpose(1, 2)).reshape(-1)
    return torch.where(enough, q.sqrt(), torch.full_like(q, float("nan")))


def niqe(restored, params, border=0):
    """Per-image NIQE (B,) float64 of the blind-SR test command (NaturalImageQualityEvaluator.update, niqe.py:566-576):
    restored (B, 3, H, W) CUDA fp32, the model's output (tensor_round is applied inside).  params: a path to the
    reference's niqe_pris_params.npz (utils/metrics/ in a reference checkout) or a mapping with its three arrays; nothing
    of it ships with this package.  `border` pixels are cropped on every side first.  The luma is the reference's:
    bgr2ycbcr weights on RGB data (grl_niqe.h)."""
    mu_pris, cov_pris, _ = niqe_params(params)
    return niqe_distance(niqe_features(restored, params, border), mu_pris, cov_pris)


def validation_metrics(restored, target, scale=1, is_sr=False):
    """dict of per-image (B,) tensors: psnr, psnr_y, ssim, ssim_y, as validation_step + the metric collection yield them."""
    border = scale if is_sr else 0
    return {
        "psnr": psnr(restored, target, border, "rgb"),
        "psnr_y": psnr(restored, target, border, "y"),
        "ssim": ssim(restored, target, border, "rgb"),
        "ssim_y": ssim(restored, target, border, "y"),
    }
