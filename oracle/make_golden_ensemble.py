"""TEST INFRASTRUCTURE.  Writes the x8 self-ensemble fixtures under tests/golden/ from the UNMODIFIED reference: its
network (models/networks/grl.py) and its dihedral augmentation augment_img_tensor4 (utils/utils_bsr/utils_image.py:444-460,
imported from the reference checkout at generation time; that module needs cv2 and torchvision).  Runs only where the
reference exists (the build container):

    python oracle/make_golden_ensemble.py            # validate + (re)write fixtures
    python oracle/make_golden_ensemble.py --check    # validate only

For every case: y = 0.125 * (V_0 + ... + V_7) summed in mode order in fp32, V_m = inv_m(GRL(augment_img_tensor4(x, m))),
inv_m = augment_img_tensor4(., 8 - m) for m in {3, 5} and augment_img_tensor4(., m) otherwise.  Weights come from
oracle.synth_state_dict(style="init"), inputs from oracle.synth_input.

Fixtures: tests/golden/ensemble_cases.json (the case descriptions) and tests/golden/ensemble_<name>.npz with
  input (B, Cin, H, W); view<m>/input = augment_img_tensor4(input, m); view<m>/output = the reference network's output
  on that view (in the view's orientation); merged = the self-ensemble output (B, Cout, H s, W s).
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

import grl_oracle as orc  # noqa: E402
from _pkgload import load_package  # noqa: E402
from _ref_import import REF_ROOT, import_reference  # noqa: E402
from make_golden import build_reference  # noqa: E402

configs = load_package().configs
GOLD = os.path.join(ROOT, "tests", "golden")

CASES = {
    # name: (cfg, batch, (H, W), noise_sigma).  28 x 44 is non-square and not a multiple of the pad size 16, so both view
    # groups (28 x 44 and 44 x 28) are padded, differently; the denoiser (no upsampler, in == out channels) adds the
    # input back and runs two images per view.
    "micro_cab_x2": (configs.micro_config(), 1, (28, 44), 0.0),
    "micro_dn": (configs.micro_config(embed_dim=36, stripe=(8, 16), df=2, upsampler="", upscale=1, img_size=32),
                 2, (20, 36), 25.0),
}
INVERSE = {3: 5, 5: 3}


def load_augment():
    path = os.path.join(REF_ROOT, "utils", "utils_bsr", "utils_image.py")
    spec = importlib.util.spec_from_file_location("ref_utils_bsr_image", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.augment_img_tensor4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    grl_mod, _, _, _ = import_reference()
    augment = load_augment()
    torch.set_num_threads(os.cpu_count())
    files = {}
    for name, (cfg, batch, hw, sigma) in CASES.items():
        sd = orc.synth_state_dict(cfg, seed=0, style="init")
        ref = build_reference(grl_mod, cfg, sd)
        x = orc.synth_input((batch, cfg["in_channels"], *hw), seed=1234, noise_sigma=sigma)
        arrs = {"input": x.numpy()}
        acc = None
        for m in range(8):
            v = augment(x.clone(), m).contiguous()
            with torch.no_grad():
                out = ref(v.clone())
                out_orc = orc.grl_forward(sd, cfg, v.clone())
            err = (out - out_orc).abs().max().item()
            assert err <= 2e-6 * max(1.0, out.abs().max().item()), (name, m, err)
            back = augment(out, INVERSE.get(m, m))
            acc = back.clone() if acc is None else acc + back
            arrs[f"view{m}/input"] = v.numpy()
            arrs[f"view{m}/output"] = out.contiguous().numpy()
            print(f"[{name}] view {m}: in {tuple(v.shape)} out {tuple(out.shape)} |oracle-ref|max = {err:.3e}")
        arrs["merged"] = (acc * 0.125).contiguous().numpy()
        files[name] = arrs
    if args.check:
        print("check OK (fixtures not rewritten)")
        return
    for name, arrs in files.items():
        path = os.path.join(GOLD, f"ensemble_{name}.npz")
        np.savez_compressed(path, **arrs)
        print(f"{path}: {os.path.getsize(path)} bytes")
    with open(os.path.join(GOLD, "ensemble_cases.json"), "w") as f:
        json.dump({k: dict(cfg=v[0], batch=v[1], hw=list(v[2]), sigma=v[3], style="init", seed=0, input_seed=1234)
                   for k, v in CASES.items()}, f, indent=1)
    print("fixtures written to", GOLD)


if __name__ == "__main__":
    main()
