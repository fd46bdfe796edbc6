"""TEST INFRASTRUCTURE.  Writes the fixtures of the dataset-side inputs that evaluation.py builds on the device, from the
UNMODIFIED reference imported at generation time (as make_golden_dm.py does):

    python oracle/make_golden_eval.py            # validate + (re)write fixtures
    python oracle/make_golden_eval.py --check    # validate only

  mosaic: DemosaicDataset.__getitem__ (data/datasets/restoration_dm.py:26-44, validation branch: crop to multiples of 8,
          mosaic_CFA_Bayer(img)[1], to_tensor) on in-memory images, and mosaic_CFA_Bayer alone on images of even and odd
          sizes down to 2 x 2, 3 x 3 and one row, with saturated and random content.  The reference's mosaic_CFA_Bayer
          raises on an odd height or width (CFA4 has H // 2 rows, CFA[0::2] has ceil(H / 2)); the datasets never pass
          one, as they crop to multiples of 8 first.  The device mosaic drops the odd last row / column, so an odd case's
          fixture is mosaic_CFA_Bayer of the image's even crop, and this script checks that the reference raises on the
          odd image itself.
  luma:   rgb2ycbcr_np(img, y_only=True) (utils/utils_image.py:143-190) on a sampled subset of the RGB cube: the byte
          ramps, the saturated corners and seeded random triples.  No triple of the whole cube lies on a rounding tie
          decided by the evaluation order (tests/test_dataset_u8.py checks all 2^24 against numpy), so there are none to
          add.
  uint2single: utils/utils_bsr/utils_image.py:270-272 of all 256 bytes, the blind-SR dataset's reader.
  pipeline: one tiny end-to-end case per task row of evaluation.RECIPES on the micro architectures of tests/support.py
          (weights oracle.synth_state_dict(cfg, seed 0, "init")): seeded clean (and low-quality) 8-bit images, the model
          input the reference's dataset code makes from them (DnDataset / DemosaicDataset.__getitem__,
          JPEGDataset.jpeg_compress, rgb2ycbcr_np, modcrop, uint2single, to_tensor; dm_matlab for the dm network), the
          oracle network (tiled as engines/base.py:90-116 where the recipe tiles), tensor_round, and the per-image scores
          of the reference's metric functions (utils/metrics/psnr.py, ssim.py, psnrb.py, niqe.py, with the SR shave).

Fixtures: tests/golden/eval_cases.json (name -> how the case was made) and tests/golden/eval_inputs.npz (per case
<name>/img (H, W, 3) uint8 and <name>/mosaic (4, h, w) float32; luma/rgb (n, 3) uint8 and luma/y (n,) uint8;
uint2single (256,) float32); tests/golden/eval_pipeline.json (row -> checkpoint name, architecture, sizes, keys, dataset)
and tests/golden/eval_pipeline.npz (per row and image i: <row>/gt<i>, <row>/lq<i> (+ <row>/lqr<i>) uint8 files,
<row>/input<i> the dataset's model input (dn: float32; jpeg, dm: its bytes), <row>/out<i> the reference output's bytes (H, W, C) uint8, and per metric
<row>/<metric> (n,) float64 scores).
"""
import argparse
import importlib.util
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import make_golden_awgn  # noqa: E402
from _ref_import import REF_ROOT  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")

# name -> (H, W, content, seed, through the dataset).  The dataset crops to multiples of 8 first, so the odd sizes go
# through mosaic_CFA_Bayer directly.
MOSAIC = {
    "ds_45x61": (45, 61, "random", 1, True),
    "ds_64x40": (64, 40, "random", 2, True),
    "ds_17x23_saturated": (17, 23, "saturated", 3, True),
    "even_2x2": (2, 2, "random", 4, False),
    "odd_3x3": (3, 3, "random", 5, False),
    "one_row_1x9": (1, 9, "random", 6, False),
    "one_col_7x1": (7, 1, "random", 7, False),
    "odd_5x8": (5, 8, "saturated", 8, False),
    "odd_31x17": (31, 17, "random", 9, False),
    "even_24x36_saturated": (24, 36, "saturated", 10, False),
}


def load(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF_ROOT, *rel.split("/")))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def content(H, W, kind, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if kind == "saturated":
        img[: (H + 1) // 2] = 255
        img[(H + 1) // 2:, : W // 2] = 0
    return img


def demosaic_item(DemosaicDataset, img):
    ds = DemosaicDataset.__new__(DemosaicDataset)
    ds.stage = "val"
    ds.cfg = make_golden_awgn._Cfg(modulo=8)
    ds.num_train_samples = 0
    ds.img_info = [("<memory>", "<memory>")]
    ds._load_item = lambda index: img.copy()
    return ds[0]


def luma_triples():
    ramp = np.arange(256)
    rows = [np.stack([ramp, ramp, ramp], 1), np.stack([ramp, 0 * ramp, 0 * ramp], 1), np.stack([0 * ramp, ramp, 0 * ramp], 1),
            np.stack([0 * ramp, 0 * ramp, ramp], 1), np.stack([ramp, 255 - ramp, (7 * ramp) % 256], 1)]
    corners = np.array([[r, g, b] for r in (0, 255) for g in (0, 255) for b in (0, 255)])
    rng = np.random.default_rng(0)
    return np.concatenate(rows + [corners, rng.integers(0, 256, (4096, 3))]).astype(np.uint8)


# row -> (checkpoint name, micro architecture (tests/support.py MICRO), tile, overlap, scale, image sizes).  The tiles are
# the released ones, so on these small images the tile is min(tile, H, W) and the windows overlap as engines/base.py does.
PIPELINE = {
    "sr": ("sr_grl_tiny_c3x2.ckpt", "micro_cab_x2", 0, 0, 2, [(61, 75), (72, 56)]),
    "dn_c3": ("dn_grl_base_c3s15.ckpt", "micro_pad_dn", 256, 32, 1, [(61, 75), (72, 56)]),
    "dn_c1": ("dn_grl_small_c1s15.ckpt", "micro_gray", 0, 0, 1, [(61, 75), (72, 56)]),
    "jpeg_c3": ("jpeg_grl_small_c3q10.ckpt", "micro_pad_dn", 288, 36, 1, [(61, 75), (72, 56)]),
    "jpeg_c1": ("jpeg_grl_small_c1q10.ckpt", "micro_gray", 288, 36, 1, [(61, 75), (72, 56)]),
    "dm": ("dm_grl_small.ckpt", "micro_pad_dn", 0, 0, 1, [(61, 75), (72, 56)]),
    "bsr": ("bsr_grl_base.ckpt", "micro_pad_dn", 0, 0, 1, [(200, 104), (196, 196)]),
    "defocus": ("db_defocus_single_pixel_grl_base.ckpt", "micro_pad_dn", 480, 48, 1, [(61, 75), (72, 56)]),
    "defocus_dual": ("db_defocus_dual_pixel_grl_base.ckpt", "micro_dual", 480, 48, 1, [(61, 75), (72, 56)]),
    "motion": ("db_motion_grl_base_gopro.ckpt", "micro_pad_dn", 0, 0, 1, [(61, 75), (72, 56)]),
}


def pipeline(uimg, ubsr, mosaic, DemosaicDataset):
    """The reference pipeline of every PIPELINE row -> (table, arrays)."""
    import types

    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import engine_oracle
    import grl_oracle as orc
    from _pkgload import load_package
    from support import MICRO

    if "torchmetrics" not in sys.modules:
        tm = types.ModuleType("torchmetrics")
        tm.Metric = type("Metric", (torch.nn.Module,), {})
        sys.modules["torchmetrics"] = tm
    sys.path.insert(0, REF_ROOT)
    from utils.metrics import niqe as ref_niqe
    from utils.metrics.psnr import psnr as ref_psnr
    from utils.metrics.psnrb import psnrb as ref_psnrb
    from utils.metrics.ssim import ssim as ref_ssim
    from utils.utils_image import rgb2ycbcr, shave, tensor_round

    jpeg_mod = importlib.import_module("data.datasets.restoration_jpeg")
    DnDataset = make_golden_awgn._dn_dataset_class()
    configs = load_package().configs

    def to_tensor(a):
        return torch.from_numpy(np.ascontiguousarray(a)).permute(2, 0, 1).float().div(255)

    def jpeg(img, C):
        fake = types.SimpleNamespace(quality_factor=10, stage="val", quality_factor_range=[],
                                     cfg=make_golden_awgn._Cfg(num_channels=C))
        return jpeg_mod.JPEGDataset.jpeg_compress(fake, img)[0]

    table, arrays = {}, {}
    for row, (name, arch, tile, overlap, scale, sizes) in PIPELINE.items():
        cfg = configs.micro_config(**MICRO[arch])
        if arch == "micro_dual":
            cfg["out_channels"] = 3
        sd = orc.synth_state_dict(cfg, seed=0, style="init")
        rng = np.random.default_rng(1000 + list(PIPELINE).index(row))
        C = 1 if row == "dn_c1" else 3
        keys = [f"{'CBSD68' if C == 3 else 'Set12'}/{i:04d}.png" for i in range(len(sizes))] if row.startswith("dn") \
            else None
        dataset = "live1" if row == "jpeg_c1" else None
        scores = {}
        for i, (h, w) in enumerate(sizes):
            gt = rng.integers(0, 256, (h, w, C), dtype=np.uint8)
            arrays[f"{row}/gt{i}"] = gt
            if row == "sr":
                lq = rng.integers(0, 256, (h // 2, w // 2, 3), dtype=np.uint8)
                arrays[f"{row}/lq{i}"] = lq
                clean, x = uimg.modcrop(gt, scale), to_tensor(lq)  # base_image.py:404-405, restoration_sr.py:114
            elif row.startswith("dn"):
                item = make_golden_awgn.reference_item(DnDataset, gt, keys[i], 15)
                clean, x = np.ascontiguousarray(gt[: h // 8 * 8, : w // 8 * 8]), item["img_lq"]
                assert torch.equal(item["img_gt"], to_tensor(clean))
            elif row.startswith("jpeg"):
                clean = uimg.rgb2ycbcr_np(gt, y_only=True)[..., None] if row == "jpeg_c1" else gt
                x = to_tensor(jpeg(clean, clean.shape[2]))
            elif row == "dm":
                item = demosaic_item(DemosaicDataset, gt)
                clean, x = np.ascontiguousarray(gt[: h // 8 * 8, : w // 8 * 8]), item["img_lq"]
            elif row == "bsr":
                clean, x = None, ubsr.single2tensor3(ubsr.uint2single(gt))
            else:
                lq = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
                arrays[f"{row}/lq{i}"] = lq
                x = to_tensor(lq)
                if row == "defocus_dual":
                    lqr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
                    arrays[f"{row}/lqr{i}"] = lqr
                    x = torch.cat([x, to_tensor(lqr)], 0)  # engines/base.py:119-120
                clean = gt
            if row.startswith("dn"):
                arrays[f"{row}/input{i}"] = x.numpy()  # float32 (C, H, W): the noisy input
            elif row.startswith("jpeg") or row == "dm":  # k / 255 planes: their bytes (C, H, W)
                arrays[f"{row}/input{i}"] = (x * 255).round().to(torch.uint8).numpy()
                assert torch.equal(to_tensor(arrays[f"{row}/input{i}"].transpose(1, 2, 0)), x)
            net_in = mosaic.dm_matlab(x[None].clone()) if row == "dm" else x[None]  # engines/base.py:127-128
            with torch.no_grad():
                fn = lambda t: orc.grl_forward(sd, cfg, t)  # noqa: E731
                out = engine_oracle.forward_tile(fn, net_in, tile, overlap, scale) if tile else fn(net_in)
            pr = tensor_round(out.clone(), 1.0)
            arrays[f"{row}/out{i}"] = (pr[0] * 255).round().to(torch.uint8).permute(1, 2, 0).numpy()
            if row == "bsr":  # NaturalImageQualityEvaluator.update, niqe.py:566-576
                vals = {"val_niqe": ref_niqe.calculate_niqe(pr[0].numpy() * 255, crop_border=0, input_order="CHW")}
            else:
                t = tensor_round(to_tensor(clean)[None], 1.0)
                if row == "sr":  # engines/base.py:265-267
                    pr, t = shave(pr, scale), shave(t, scale)
                vals = {"val_psnr": ref_psnr(pr, t)[0], "val_ssim": ref_ssim(pr, t)}
                if t.shape[1] == 3:
                    py, ty = rgb2ycbcr(pr, 1.0), rgb2ycbcr(t, 1.0)
                    vals.update(val_psnr_y=ref_psnr(py, ty)[0], val_ssim_y=ref_ssim(py, ty))
                if row.startswith("jpeg"):
                    vals["val_psnrb"] = ref_psnrb(t, pr)[0]
                    if t.shape[1] == 3:
                        vals["val_psnrb_y"] = ref_psnrb(rgb2ycbcr(t, 1.0), rgb2ycbcr(pr, 1.0))[0]
            for k, v in vals.items():
                scores.setdefault(k, []).append(float(v))
        for k, v in scores.items():
            arrays[f"{row}/{k}"] = np.array(v, dtype=np.float64)
        table[row] = {"name": name, "arch": arch, "sizes": sizes, "keys": keys, "dataset": dataset,
                      "metrics": sorted(scores)}
        print(f"pipeline {row}: " + ", ".join(f"{k} {np.mean(v):.4f}" for k, v in scores.items()))
    return table, arrays


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    mosaic = load("utils/utils_mosaic.py", "ref_utils_mosaic")
    uimg = load("utils/utils_image.py", "ref_utils_image")
    ubsr = load("utils/utils_bsr/utils_image.py", "ref_utils_bsr_image")
    make_golden_awgn._dn_dataset_class()  # installs the stand-ins and package paths the dataset modules need
    DemosaicDataset = importlib.import_module("data.datasets.restoration_dm").DemosaicDataset

    table, arrays = {}, {}
    for name, (H, W, kind, seed, through_ds) in MOSAIC.items():
        img = content(H, W, kind, seed)
        even = img[: H // 2 * 2, : W // 2 * 2]
        if (H % 2, W % 2) != (0, 0) and (H > 1 or W % 2):
            try:  # the reference's CFA4 has H // 2 rows but CFA[0::2] has ceil(H / 2): it cannot mosaic an odd image
                mosaic.mosaic_CFA_Bayer(img)
                raise AssertionError(f"{name}: mosaic_CFA_Bayer accepted an odd image")
            except ValueError:
                pass
        direct = torch.from_numpy(np.ascontiguousarray(mosaic.mosaic_CFA_Bayer(even)[1])).permute(2, 0, 1).float().div(255)
        if through_ds:
            item = demosaic_item(DemosaicDataset, img)
            crop = img[: H // 8 * 8, : W // 8 * 8]
            want = torch.from_numpy(np.ascontiguousarray(mosaic.mosaic_CFA_Bayer(crop)[1])).permute(2, 0, 1).float().div(255)
            assert torch.equal(item["img_lq"], want), name
            assert torch.equal(item["img_gt"], torch.from_numpy(np.ascontiguousarray(crop)).permute(2, 0, 1).float().div(255))
            out, img = item["img_lq"], np.ascontiguousarray(crop)
        else:
            out = direct
        assert out.dtype == torch.float32 and tuple(out.shape) == (4, img.shape[0] // 2, img.shape[1] // 2), name
        print(f"mosaic {name}: {img.shape} -> {tuple(out.shape)}")
        table[name] = {"H": H, "W": W, "content": kind, "seed": seed, "dataset": through_ds}
        arrays[f"{name}/img"] = img
        arrays[f"{name}/mosaic"] = out.numpy()

    rgb = luma_triples()
    y = uimg.rgb2ycbcr_np(rgb[None], y_only=True)[0]
    assert y.dtype == np.uint8 and y.shape == (len(rgb),)
    arrays["luma/rgb"], arrays["luma/y"] = rgb, y
    table["luma"] = {"triples": len(rgb), "ties": []}
    print(f"luma: {len(rgb)} triples")

    u = ubsr.uint2single(np.arange(256, dtype=np.uint8))
    assert u.dtype == np.float32
    arrays["uint2single"] = u

    ptable, parrays = pipeline(uimg, ubsr, mosaic, DemosaicDataset)
    if args.check:
        print("check OK (fixtures not rewritten)")
        return
    with open(os.path.join(GOLD, "eval_cases.json"), "w") as f:
        json.dump(table, f, indent=1)
    np.savez_compressed(os.path.join(GOLD, "eval_inputs.npz"), **arrays)
    with open(os.path.join(GOLD, "eval_pipeline.json"), "w") as f:
        json.dump(ptable, f, indent=1)
    np.savez_compressed(os.path.join(GOLD, "eval_pipeline.npz"), **parrays)
    print("fixtures written to", GOLD)


if __name__ == "__main__":
    main()
