"""TEST INFRASTRUCTURE ONLY. Writes tests/golden/psnrb.npz from the UNMODIFIED reference PSNR-B (utils/metrics/psnrb.py).

Needs the reference checkout; registers the torchmetrics stand-in of make_golden_metrics.py.  The recipe is the JPEG
test command's (config/metric/restorer_jpeg*.yaml): both images tensor_round'ed (engines/base.py:259-260), no shave,
then PeakSignalNoiseRatioBlock.update (psnrb.py:141-163), i.e. psnrb(target, restored) on RGB and, for RGB cases, on
rgb2ycbcr(., 1.0).  Inputs are stored as 8-bit values; the restored images of case "clamp" are stored as fp32 because
they leave [0, 1].

    python oracle/make_golden_psnrb.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from _ref_import import REF_ROOT, reference_available  # noqa: E402


def main():
    if not reference_available():
        raise SystemExit("reference not mounted: the PSNR-B golden can only be regenerated next to a reference checkout")
    if "torchmetrics" not in sys.modules:
        tm = types.ModuleType("torchmetrics")
        tm.Metric = type("Metric", (torch.nn.Module,), {})
        sys.modules["torchmetrics"] = tm
    sys.path.insert(0, REF_ROOT)
    from utils.metrics.psnrb import psnrb as ref_psnrb
    from utils.utils_image import rgb2ycbcr, tensor_round

    g = torch.Generator().manual_seed(77)

    def blocky(b, c, h, w):
        """8 x 8 block means plus noise: a JPEG-like image with real blocking."""
        base = torch.rand(b, c, (h + 7) // 8, (w + 7) // 8, generator=g).repeat_interleave(8, 2).repeat_interleave(8, 3)
        return base[..., :h, :w]

    out = {}
    for name, (b, c, h, w) in {"rgb_b2": (2, 3, 37, 53), "rgb_w20": (1, 3, 96, 20), "gray": (1, 1, 64, 96),
                               "clamp": (2, 3, 40, 48)}.items():
        target = torch.rand(b, c, h, w, generator=g)
        restored = 0.6 * blocky(b, c, h, w) + 0.4 * target + 0.05 * torch.randn(b, c, h, w, generator=g)
        if name == "clamp":
            restored = restored * 1.4 - 0.2  # leaves [0, 1]: exercises tensor_round's clamp
            out[f"{name}_restored"] = restored.numpy()
        else:
            restored = tensor_round(restored.clone(), 1.0)
            out[f"{name}_restored8"] = (restored * 255).round().to(torch.uint8).numpy()
            restored = out[f"{name}_restored8"]
            restored = torch.from_numpy(restored.astype(np.float32) / np.float32(255.0))
        target = tensor_round(target.clone(), 1.0)
        out[f"{name}_target8"] = (target * 255).round().to(torch.uint8).numpy()
        target = torch.from_numpy(out[f"{name}_target8"].astype(np.float32) / np.float32(255.0))
        r, t = tensor_round(restored.clone(), 1.0), tensor_round(target.clone(), 1.0)
        out[f"{name}_psnrb"] = ref_psnrb(t, r).numpy()
        if c == 3:
            out[f"{name}_psnrb_y"] = ref_psnrb(rgb2ycbcr(t, 1.0), rgb2ycbcr(r, 1.0)).numpy()
    path = os.path.join(HERE, "..", "tests", "golden", "psnrb.npz")
    np.savez_compressed(path, **out)
    print("wrote", os.path.normpath(path), {k: v.tolist() for k, v in out.items() if "psnrb" in k})


if __name__ == "__main__":
    main()
