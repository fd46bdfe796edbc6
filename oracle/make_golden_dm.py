"""TEST INFRASTRUCTURE.  Writes the demosaicking fixtures under tests/golden/ from the UNMODIFIED reference: its mosaic
helpers (utils/utils_mosaic.py: mosaic_CFA_Bayer and dm_matlab, imported from the reference checkout at generation time)
and its network (models/networks/grl.py).  Runs only where the reference exists (the build container):

    python oracle/make_golden_dm.py            # validate + (re)write fixtures
    python oracle/make_golden_dm.py --check    # validate only

For every case, the dm data path of the reference (data/datasets/restoration_dm.py:33-37, engines/base.py:127-128):
a seeded uint8 RGB image -> mosaic_CFA_Bayer(img)[1] (the packed RGGB planes, uint8) -> / 255 (to_tensor) = cfa4
(B, 4, h, w) -> dm_matlab(cfa4) = rgb (B, 3, 2h, 2w) -> GRL(**grl_config("small", "dm")) with "init" weights = output.

Fixtures: tests/golden/dm_cases.json (the case descriptions) and tests/golden/dm_<name>.npz with cfa4, rgb and output.
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
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import dm_oracle  # noqa: E402
import grl_oracle as orc  # noqa: E402
from _pkgload import load_package  # noqa: E402
from _ref_import import REF_ROOT, import_reference  # noqa: E402
from make_golden import build_reference  # noqa: E402

configs = load_package().configs
GOLD = os.path.join(ROOT, "tests", "golden")

CASES = {
    # name: (batch, (2h, 2w), seed).  The dm config pads to a multiple of 32: 40 x 56 reflects into 64 x 64; 4 x 4 needs a
    # pad of 28 > 4, so check_image_size falls back to zeros; 18 x 26 has odd h and w (9 x 13 Bayer quads).
    "b2_40x56": (2, (40, 56), 11),
    "zero_pad_4x4": (1, (4, 4), 12),
    "odd_18x26": (1, (18, 26), 13),
}
CFG = configs.grl_config("small", "dm", img_size=64)


def load_mosaic():
    path = os.path.join(REF_ROOT, "utils", "utils_mosaic.py")
    spec = importlib.util.spec_from_file_location("ref_utils_mosaic", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def seeded_images(batch, hw, seed):
    """uint8 (H, W, 3) images: a smooth colour ramp plus seeded noise, so the filters see both edges and gradients."""
    g = torch.Generator().manual_seed(seed)
    H, W = hw
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    ramp = torch.stack([yy, xx, 1 - 0.5 * (yy + xx)], -1)
    out = []
    for _ in range(batch):
        img = 0.6 * ramp + 0.4 * torch.rand(H, W, 3, generator=g)
        out.append((img * 255).round().clamp(0, 255).to(torch.uint8).numpy())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    grl_mod, _, _, _ = import_reference()
    mosaic = load_mosaic()
    torch.set_num_threads(os.cpu_count())
    sd = orc.synth_state_dict(CFG, seed=0, style="init")
    ref_net = build_reference(grl_mod, CFG, sd)
    files = {}
    for name, (batch, hw, seed) in CASES.items():
        planes = [mosaic.mosaic_CFA_Bayer(img)[1] for img in seeded_images(batch, hw, seed)]  # (h, w, 4) uint8
        cfa4 = torch.stack([torch.from_numpy(np.ascontiguousarray(p)).permute(2, 0, 1).float().div(255) for p in planes])
        rgb = mosaic.dm_matlab(cfa4.clone())
        mine = dm_oracle.dm_matlab(cfa4)
        assert torch.equal(rgb, mine), (name, (rgb - mine).abs().max().item())
        with torch.no_grad():
            out = ref_net(rgb.clone())
            out_orc = orc.grl_forward(sd, CFG, rgb.clone())
        err = (out - out_orc).abs().max().item()
        assert err <= 2e-6 * max(1.0, out.abs().max().item()), (name, err)
        print(f"[{name}] cfa4 {tuple(cfa4.shape)} -> rgb {tuple(rgb.shape)} -> out {tuple(out.shape)}; "
              f"oracle dm_matlab bit-exact, |oracle-ref| network max = {err:.3e}")
        files[name] = {"cfa4": cfa4.numpy(), "rgb": rgb.numpy(), "output": out.contiguous().numpy()}
    if args.check:
        print("check OK (fixtures not rewritten)")
        return
    for name, arrs in files.items():
        path = os.path.join(GOLD, f"dm_{name}.npz")
        np.savez_compressed(path, **arrs)
        size = os.path.getsize(path)
        assert size < 1 << 20, (path, size)
        print(f"{path}: {size} bytes")
    with open(os.path.join(GOLD, "dm_cases.json"), "w") as f:
        json.dump({"cfg": CFG, "style": "init", "seed": 0,
                   "cases": {k: dict(batch=b, hw=list(hw), image_seed=s) for k, (b, hw, s) in CASES.items()},
                   "arrays": {"cfa4": "(B, 4, h, w) float32: mosaic_CFA_Bayer(img)[1] / 255, img = seeded uint8 (2h, 2w, 3)",
                              "rgb": "(B, 3, 2h, 2w) float32: the reference's dm_matlab(cfa4)",
                              "output": "(B, 3, 2h, 2w) float32: the reference GRL (cfg, init weights) on rgb"}},
                  f, indent=1)
    print("fixtures written to", GOLD)


if __name__ == "__main__":
    main()
