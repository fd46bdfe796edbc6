"""What each pair of metric tests shares, the host test (test_<metric>.py) and the device test (test_gpu_<metric>.py):
the golden cases written from the reference's own metrics (oracle/make_golden_<metric>.py) and the score gates, whose
derivations are in the host tests' docstrings."""
import ctypes
import os

import numpy as np
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

SSIM_GOLDEN = os.path.join(GOLD, "ssim.npz")
SSIM_CASES = ["flat", "letterbox", "sr_b2", "gray", "tiny", "clamp"]
SSIM_SCORE_GATE = 2e-5

PSNRB_GOLDEN = os.path.join(GOLD, "psnrb.npz")
PSNRB_CASES = ["rgb_b2", "rgb_w20", "gray", "clamp"]

NIQE_CASES = ["smooth", "flat", "b2"]
NIQE_SCORE_GATE = 2e-3
ALPHA_COLS = [0, 2, 6, 10, 14, 18, 20, 24, 28, 32]  # the GGD / AGGD shape columns of a NIQE feature row


def golden_pair(g, name):
    """(restored, target) fp32 (B, C, H, W) of a golden case: the restoration as stored or as k / 255 of its bytes."""
    restored = (torch.from_numpy(g[f"{name}_restored"]) if f"{name}_restored" in g
                else torch.from_numpy(g[f"{name}_restored8"].astype(np.float32) / np.float32(255.0)))
    target = torch.from_numpy(g[f"{name}_target8"].astype(np.float32) / np.float32(255.0))
    return restored, target


def golden_scores(g, name):
    """(ssim, ssim_y) of the reference; ssim_y of a one-channel case is its ssim."""
    s = g[f"{name}_ssim"]
    return s, (g[f"{name}_ssim_y"] if f"{name}_ssim_y" in g else s)


def host_ssim(restored, target, border=0, maps=False):
    """grl_ssim_host on two fp32 (B, C, H, W) host tensors -> (ssim_rgb, ssim_y[, map_rgb, map_y]) as NumPy float64."""
    from grl_image_restoration_b200 import capi

    a, b = np.ascontiguousarray(restored.numpy(), np.float32), np.ascontiguousarray(target.numpy(), np.float32)
    B, C, H, W = a.shape
    h, w = max(H - 2 * border, 0), max(W - 2 * border, 0)
    s, sy = np.zeros(B), np.zeros(B)
    m, my = np.zeros((B, C, h, w)), np.zeros((B, 1, h, w))
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    capi.check(capi.lib().grl_ssim_host(p(a), p(b), B, C, H, W, border, p(s), p(sy), p(m) if maps else None,
                                        p(my) if maps and C == 3 else None))
    return (s, sy, m, my) if maps else (s, sy)


def niqe_params():
    """The reference's pristine NIQE model (mu_pris_param, cov_pris_param, gaussian_window)."""
    return dict(np.load(os.path.join(GOLD, "niqe_pris_params.npz")))
