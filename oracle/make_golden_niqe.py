"""TEST INFRASTRUCTURE ONLY. Writes tests/golden/niqe_*.npz from the UNMODIFIED reference NIQE (utils/metrics/niqe.py)
and copies its pristine-model parameters to tests/golden/niqe_pris_params.npz as a data fixture.

Needs the reference checkout.  The metric files import torchmetrics for their Metric base class only; the stand-in of
make_golden_metrics.py is registered.  Per case the golden holds the 8-bit input (B, 3, H, W), `border`, and from the
reference's own functions: the rounded luma after both crops (to_y_channel + crop + round, :529-542 and :439-443), its
x0.5 image (imresize, :470-471), the per-block feature matrix (convolve + compute_feature as niqe() calls them,
:446-473), the resize weights (calculate_weights_indices) and the score of calculate_niqe itself.  The feature matrix is
checked to give calculate_niqe's score before anything is written.

    python oracle/make_golden_niqe.py
"""
import os
import shutil
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from _ref_import import REF_ROOT, reference_available  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")


def smooth_noise(rng, h, w, sigma=12):
    yy, xx = np.mgrid[0:h, 0:w] / max(h, w)
    base = np.stack([np.sin(6 * xx + 2 * yy), np.cos(5 * yy - 3 * xx), np.sin(4 * (xx + yy))]) * 70 + 128
    return np.clip(base + rng.normal(0, sigma, (3, h, w)), 0, 255).round().astype(np.uint8)


def cases():
    rng = np.random.default_rng(2024)
    flat = smooth_noise(rng, 500, 700, sigma=4)
    flat[:, :110] = 0  # black letterbox rows: the first row of blocks is flat at both scales
    flat[:, 490:] = 0
    flat[:, 182:298, 182:394] = 255  # saturated patch: blocks (2, 2) and (2, 3) plus their halo are flat
    return {
        "smooth": (smooth_noise(rng, 288, 384)[None], 0),
        "flat": (flat[None], 0),
        "b2": (np.stack([smooth_noise(rng, 200, 200), smooth_noise(rng, 200, 200)]), 4),
    }


def main():
    if not reference_available():
        raise SystemExit("reference not mounted: the NIQE goldens can only be regenerated next to a reference checkout")
    if "torchmetrics" not in sys.modules:
        tm = types.ModuleType("torchmetrics")
        tm.Metric = type("Metric", (torch.nn.Module,), {})
        sys.modules["torchmetrics"] = tm
    sys.path.insert(0, REF_ROOT)
    warnings.simplefilter("ignore")
    from utils.metrics import niqe as ref
    from utils.utils_image import tensor_round

    params_path = os.path.join(REF_ROOT, "utils", "metrics", "niqe_pris_params.npz")
    shutil.copyfile(params_path, os.path.join(GOLD, "niqe_pris_params.npz"))
    prm = np.load(params_path)
    mu_p, cov_p, win = prm["mu_pris_param"], prm["cov_pris_param"], prm["gaussian_window"]
    for name, (rgb8, border) in cases().items():
        out = {"rgb8": rgb8, "border": np.array(border)}
        ys, halves, feats, scores = [], [], [], []
        for img8 in rgb8:
            p = tensor_round(torch.from_numpy(img8.astype(np.float32) / np.float32(255.0)), 1.0).numpy()
            score = ref.calculate_niqe(p * 255, crop_border=border, input_order="CHW")  # NaturalImageQualityEvaluator.update
            img = ref.to_y_channel(ref.reorder_image((p * 255).astype(np.float32), input_order="CHW"))
            img = np.squeeze(img)
            if border:
                img = img[border:-border, border:-border]
            img = img.round()
            h, w = img.shape
            nbh, nbw = h // 96, w // 96
            img = img[: nbh * 96, : nbw * 96]
            ys.append(img.astype(np.uint8))
            assert np.array_equal(ys[-1].astype(np.float32), img)
            dist = []
            cur = img
            for scale in (1, 2):
                mu = ref.convolve(cur, win, mode="nearest")
                sigma = np.sqrt(np.abs(ref.convolve(np.square(cur), win, mode="nearest") - np.square(mu)))
                m = (cur - mu) / (sigma + 1)
                bs = 96 // scale
                dist.append(np.array([ref.compute_feature(m[ih * bs:(ih + 1) * bs, iw * bs:(iw + 1) * bs])
                                      for iw in range(nbw) for ih in range(nbh)]))
                if scale == 1:
                    cur = ref.imresize(cur / 255.0, scale=0.5, antialiasing=True) * 255.0
                    halves.append(cur)
            f = np.concatenate(dist, axis=1)
            mu_d = np.nanmean(f, axis=0)
            cov_d = np.cov(f[~np.isnan(f).any(axis=1)], rowvar=False)
            inv = np.linalg.pinv((cov_p + cov_d) / 2)
            again = float(np.sqrt(np.squeeze((mu_p - mu_d) @ inv @ (mu_p - mu_d).T)))
            assert again == score, (name, again, score)
            feats.append(f)
            scores.append(score)
        wts, _, _, _ = ref.calculate_weights_indices(ys[0].shape[0], ys[0].shape[0] // 2, 0.5, "cubic", 4, True)
        out.update(y=np.stack(ys), half=np.stack(halves).astype(np.float32), feats=np.stack(feats),
                   weights=wts.numpy().astype(np.float32), score=np.array(scores))
        path = os.path.join(GOLD, f"niqe_{name}.npz")
        np.savez_compressed(path, **out)
        print("wrote", os.path.normpath(path), os.path.getsize(path), "bytes, score", scores)


if __name__ == "__main__":
    main()
