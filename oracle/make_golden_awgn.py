"""TEST INFRASTRUCTURE.  Writes the seeded-AWGN fixtures under tests/golden/ by running the reference's own
DnDataset.__getitem__ (data/datasets/restoration_dn.py:115-147, validation branch, with config/data_module/dn.yaml's
val settings: modulo 8, noise_level_map False) on in-memory 8-bit images:

    python oracle/make_golden_awgn.py            # validate + (re)write fixtures
    python oracle/make_golden_awgn.py --check    # validate only

The dataset is built with __new__ (its constructor reads the test-set file lists), `_load_item` is patched to return the
case's image, and omegaconf / h5py, which the dataset modules import but this path never uses, are stood in through
sys.modules as oracle/_ref_import.py does.  Every case is also recomputed directly -- top-left crop to multiples of 8,
x / 255, plus np.random.RandomState(np.frombuffer(sha256(name.split("_")[0]))).normal(0, sigma / 255, (C, H, W)) as
float32 -- and nothing is written on a mismatch.

The crop makes H and W multiples of 8, so no case has an odd C * H * W; a 1 x 1 image crops to an empty one.  Odd
counts are covered by tests/test_awgn.py against numpy directly.

Fixtures: tests/golden/awgn_cases.json (name -> channels, input H / W, key path, sigma, seed of the synthetic image) and
tests/golden/awgn.npz (per case: <name>/input (H, W, C) uint8, <name>/gt (C, H8, W8) float32, <name>/lq (C, H8, W8)
float32 = the dataset's img_gt and img_lq).
"""
import argparse
import hashlib
import importlib
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import _ref_import  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")

# name -> (C, H, W, key path, sigma, image seed).  Two Urban100 names that share the key "Urban100/img" (the second crop
# is smaller, so its noise is a prefix of the first's stream in C order), sigma in {15, 25, 50}, gray and RGB, an image
# already a multiple of 8, the smallest non-empty crop and 1 x 1 inputs.
CASES = {
    "c3_cbsd68_45x61_s15": (3, 45, 61, "CBSD68/0001.png", 15, 1),
    "c3_cbsd68_100x131_s50": (3, 100, 131, "CBSD68/0003.png", 50, 2),
    "c3_kodak_33x50_s25": (3, 33, 50, "Kodak24/kodim01.png", 25, 3),
    "c3_urban_30x41_s15": (3, 30, 41, "Urban100/img_004.png", 15, 4),
    "c3_urban_26x37_s15": (3, 26, 37, "Urban100/img_092.png", 15, 5),
    "c3_mcmaster_15x9_s50": (3, 15, 9, "McMaster/1.tif", 50, 6),
    "c3_1x1_s15": (3, 1, 1, "CBSD68/0002.png", 15, 7),
    "c1_set12_41x35_s15": (1, 41, 35, "Set12/01.png", 15, 8),
    "c1_bsd68_17x23_s25": (1, 17, 23, "BSD68/test001.png", 25, 9),
    "c1_urban_24x24_s50": (1, 24, 24, "Urban100/img_001.png", 50, 10),
    "c1_1x1_s50": (1, 1, 1, "Set12/02.png", 50, 11),
}


class _Cfg(dict):
    """The DictConfig surface the validation path reads: attribute access and .get."""

    __getattr__ = dict.__getitem__


def _dn_dataset_class():
    _ref_import._install_standins()
    sys.modules.setdefault("h5py", types.ModuleType("h5py"))
    oc = sys.modules["omegaconf"]
    if not hasattr(oc, "DictConfig"):
        oc.DictConfig = dict
    root = _ref_import.REF_ROOT
    if root not in sys.path:
        sys.path.insert(0, root)
    # data/__init__.py pulls in the training data module; the dataset files need only the package paths
    for pkg, path in (("data", "data"), ("data.datasets", os.path.join("data", "datasets"))):
        if pkg not in sys.modules:
            m = types.ModuleType(pkg)
            m.__path__ = [os.path.join(root, path)]
            sys.modules[pkg] = m
    return importlib.import_module("data.datasets.restoration_dn").DnDataset


def synth_image(H, W, C, seed):
    """Uniform bytes with saturated patches, so the noise also crosses 0 and 1."""
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (H, W, C), dtype=np.uint8)
    img[: H // 3, : W // 3] = 0
    img[H // 2:, W // 2:] = 255
    return img


def reference_item(DnDataset, img, key_path, sigma):
    C = img.shape[2]
    ds = DnDataset.__new__(DnDataset)
    ds.stage = "val"
    ds.cfg = _Cfg(noise_sigma=sigma, noise_level_map=False, modulo=8, num_channels=C)
    ds.noise_sigma = sigma
    ds.num_train_samples = 0
    ds.img_info = [(key_path, "<memory>")]
    ds._load_item = lambda index: img.copy()
    return ds[0]


def direct(img, key_path, sigma):
    H8, W8 = img.shape[0] // 8 * 8, img.shape[1] // 8 * 8
    gt = torch.from_numpy(np.ascontiguousarray(img[:H8, :W8]).transpose(2, 0, 1).copy()).float().div(255)
    key = np.frombuffer(hashlib.sha256(key_path.split("_")[0].encode("utf-8")).digest(), dtype="uint32")
    noise = np.random.RandomState(key).normal(0, sigma / 255, gt.shape)
    return gt, gt + torch.from_numpy(noise).float()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    DnDataset = _dn_dataset_class()
    table, arrays, bad = {}, {}, []
    for name, (C, H, W, key_path, sigma, seed) in CASES.items():
        img = synth_image(H, W, C, seed)
        item = reference_item(DnDataset, img, key_path, sigma)
        gt, lq = direct(img, key_path, sigma)
        ok = (item["img_gt"].dtype == torch.float32 and item["img_lq"].dtype == torch.float32
              and torch.equal(item["img_gt"], gt) and torch.equal(item["img_lq"], lq))
        print(f"{name}: {tuple(item['img_lq'].shape)} {'exact' if ok else 'MISMATCH'}")
        if not ok:
            bad.append(name)
        table[name] = {"channels": C, "H": H, "W": W, "key": key_path, "sigma": sigma, "seed": seed}
        arrays[f"{name}/input"] = img
        arrays[f"{name}/gt"] = item["img_gt"].numpy()
        arrays[f"{name}/lq"] = item["img_lq"].numpy()
    if bad:
        sys.exit(f"{len(bad)} mismatches: {bad}")
    if args.check:
        return
    with open(os.path.join(GOLD, "awgn_cases.json"), "w") as f:
        json.dump(table, f, indent=1)
    np.savez_compressed(os.path.join(GOLD, "awgn.npz"), **arrays)
    print(f"wrote {len(table)} cases to {GOLD}")


if __name__ == "__main__":
    main()
