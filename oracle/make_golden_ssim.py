"""TEST INFRASTRUCTURE ONLY. Writes tests/golden/ssim.npz from the UNMODIFIED reference SSIM (utils/metrics/ssim.py).

Needs the reference checkout; registers the torchmetrics stand-in of make_golden_metrics.py.  The recipe is the validation
step's (engines/base.py:255-268): both images tensor_round'ed, shaved by `border`, then
StructuralSimilarityIndexMeasure.update (ssim.py:167-193), i.e. ssim(p.unsqueeze(0), t.unsqueeze(0)) per image on the
channels and, for RGB cases, on rgb2ycbcr(., 1.0).  Inputs are stored as 8-bit values; the restored images of case
"clamp" are stored as fp32 because they leave [0, 1].  The cases:

  flat       157 x 203 RGB, no multiple of any tile: a smooth image with large flat areas and a saturated patch, the
             restored one with mild noise -- where E[x^2] - mu^2 cancels most in the reference's fp32 sums
  letterbox  black rows at the top and bottom of both images: windowed sums exactly 0, map exactly 1
  sr_b2      B = 2 with border = 4: the shave decides which pixels meet the zero padding
  gray       one channel
  tiny       7 x 9, smaller than the window
  clamp      restored values outside [0, 1]

    python oracle/make_golden_ssim.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from _ref_import import REF_ROOT, reference_available  # noqa: E402

CASES = {"flat": (1, 3, 157, 203, 0), "letterbox": (1, 3, 64, 80, 0), "sr_b2": (2, 3, 48, 56, 4), "gray": (1, 1, 40, 52, 0),
         "tiny": (1, 3, 7, 9, 0), "clamp": (1, 3, 33, 47, 0)}


def smooth(g, b, c, h, w):
    """A low-frequency image: a 5 x 6 random grid, bilinearly enlarged."""
    return torch.nn.functional.interpolate(torch.rand(b, c, 5, 6, generator=g), size=(h, w), mode="bilinear", align_corners=True)


def main():
    if not reference_available():
        raise SystemExit("reference not mounted: the SSIM golden can only be regenerated next to a reference checkout")
    if "torchmetrics" not in sys.modules:
        tm = types.ModuleType("torchmetrics")
        tm.Metric = type("Metric", (torch.nn.Module,), {})
        sys.modules["torchmetrics"] = tm
    sys.path.insert(0, REF_ROOT)
    from utils.metrics.ssim import gaussian, ssim as ref_ssim
    from utils.utils_image import rgb2ycbcr, shave, tensor_round

    g = torch.Generator().manual_seed(4242)
    out = {"taps": gaussian(11, 1.5).numpy()}
    for name, (b, c, h, w, border) in CASES.items():
        target = smooth(g, b, c, h, w)
        if name == "flat":
            target = (target * 6).floor() / 6 * 0.9 + 0.05  # plateaus
            target[..., 20:60, 30:90] = 1.0  # a saturated patch
            target[..., 100:140, 120:200] = 0.5
            restored = target + 0.01 * torch.randn(b, c, h, w, generator=g)
        elif name == "clamp":
            restored = (target + 0.1 * torch.randn(b, c, h, w, generator=g)) * 1.4 - 0.2
        else:
            restored = target + 0.05 * torch.randn(b, c, h, w, generator=g)
        if name == "letterbox":
            for t in (target, restored):
                t[..., :12, :] = 0.0
                t[..., -12:, :] = 0.0
        if name == "clamp":
            out[f"{name}_restored"] = restored.numpy()
        else:
            out[f"{name}_restored8"] = (tensor_round(restored.clone(), 1.0) * 255).round().to(torch.uint8).numpy()
            restored = torch.from_numpy(out[f"{name}_restored8"].astype(np.float32) / np.float32(255.0))
        out[f"{name}_target8"] = (tensor_round(target.clone(), 1.0) * 255).round().to(torch.uint8).numpy()
        target = torch.from_numpy(out[f"{name}_target8"].astype(np.float32) / np.float32(255.0))
        r, t = shave(tensor_round(restored.clone(), 1.0), border), shave(tensor_round(target.clone(), 1.0), border)
        out[f"{name}_border"] = np.array(border)
        out[f"{name}_ssim"] = np.array([ref_ssim(p.unsqueeze(0), q.unsqueeze(0)).item() for p, q in zip(r, t)], np.float64)
        if c == 3:
            ry, ty = rgb2ycbcr(r, 1.0), rgb2ycbcr(t, 1.0)
            out[f"{name}_ssim_y"] = np.array([ref_ssim(p.unsqueeze(0), q.unsqueeze(0)).item() for p, q in zip(ry, ty)], np.float64)
    path = os.path.join(HERE, "..", "tests", "golden", "ssim.npz")
    np.savez_compressed(path, **out)
    print("wrote", os.path.normpath(path), {k: v.tolist() for k, v in out.items() if "ssim" in k})


if __name__ == "__main__":
    main()
