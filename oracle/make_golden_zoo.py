"""TEST INFRASTRUCTURE.  Golden outputs of the UNMODIFIED reference network (models/networks/grl.py, with the stand-ins of
_ref_import.py) for the released checkpoints configs.grl_config gained last: blind x4 SR (nearest+conv head), single-
and dual-pixel defocus deblurring (6 input channels, 3 output channels) and grayscale denoising (1 channel).  Runs only
where the reference exists (the build container):

    python oracle/make_golden_zoo.py            # validate + (re)write fixtures
    python oracle/make_golden_zoo.py --check    # validate only

Each case builds the reference GRL from the config's kwargs, loads oracle.synth_state_dict(cfg, seed 0, style) and runs
it (fp32, CPU) on oracle.synth_input((B, in_channels, H, W), seed).  H, W are not multiples of the config's pad size, so
check_image_size pads (reflect) every case.  The oracle restatement must reproduce each output bit for bit.

Fixtures: tests/golden/zoo_cases.json (kwargs, the reference's parameters as param_summary records them, case
descriptions) and tests/golden/zoo_<name>.npz:
  x       (B, Cin, H, W) float32 input
  sub     output[..., ::stride, ::stride] float32 (stride 1: the whole output)
  stride  the sub-sampling step, chosen so each file stays below 1 MB
  shape   the full output shape
  sha256  digest of the full float32 output
"""
import argparse
import hashlib
import json
import os
import re
import sys
from math import prod

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import grl_oracle as orc  # noqa: E402
from _pkgload import load_package  # noqa: E402
from _ref_import import import_reference  # noqa: E402
from make_golden import build_reference  # noqa: E402

configs = load_package().configs
GOLD = os.path.join(ROOT, "tests", "golden")

# name: (grl_config args, batch, (H, W), input seed, noise sigma, weight style, output stride)
CASES = {
    # pad 64: 40 x 56 -> 64 x 64, output (2, 3, 160, 224) sampled every 3rd pixel (the whole output is 0.8 MB)
    "bsr_b2_40x56": (dict(variant="base", task="bsr", upscale=4, img_size=64), 2, (40, 56), 21, 0.0, "init", 3),
    # pad 96: 100 x 120 -> 192 x 192 (non-square, reflect in both dimensions)
    "defocus_100x120": (dict(variant="base", task="defocus", upscale=1, img_size=96), 1, (100, 120), 22, 0.0, "init", 1),
    # 6 channels in (left | right view), 3 out, zero mean; pad 96: 48 x 80 -> 96 x 96
    "defocus_dual_b2_48x80": (dict(variant="base", task="defocus_dual", upscale=1, img_size=96), 2, (48, 80), 23, 0.0,
                              "init", 1),
    # grayscale: 1 channel in and out, zero mean, input residual; pad 128: 100 x 72 -> 128 x 128
    "dn_small_c1_b2_100x72": (dict(variant="small", task="dn", upscale=1, img_size=128, in_channels=1), 2, (100, 72), 24,
                              25.0, "init", 1),
}


def param_summary(shapes):
    """{parameter name: shape} -> what zoo_cases.json records of a network's parameters: their count and total size,
    the sha256 of the sorted "name shape" listing (all names and shapes), and the names and shapes outside the
    transformer blocks, where these configs differ (heads, tails, stage convs)."""
    listing = "\n".join(f"{k} {list(v)}" for k, v in sorted(shapes.items()))
    return dict(count=len(shapes), numel=sum(prod(v) for v in shapes.values()),
                sha256=hashlib.sha256(listing.encode()).hexdigest(),
                outside_blocks={k: list(v) for k, v in sorted(shapes.items()) if ".blocks." not in k})


def case_config(args):
    a = dict(args)
    return configs.grl_config(a.pop("variant"), a.pop("task"), a.pop("upscale"), a.pop("img_size"), **a)


def case_input(cfg, batch, hw, seed, sigma):
    return orc.synth_input((batch, cfg["in_channels"], *hw), seed=seed, noise_sigma=sigma)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    grl_mod, _, _, _ = import_reference()
    torch.set_num_threads(os.cpu_count())
    files, meta = {}, {}
    for name, (cargs, batch, hw, seed, sigma, style, stride) in CASES.items():
        cfg = case_config(cargs)
        sd = orc.synth_state_dict(cfg, seed=0, style=style)
        ref_net = build_reference(grl_mod, cfg, sd)
        params = {k: list(v.shape) for k, v in ref_net.state_dict().items()
                  if k.split("_")[0] not in ("table", "index", "mask")}
        assert params == {k: list(v) for k, v in orc.param_shapes(cfg).items()}, name
        params = param_summary(params)
        x = case_input(cfg, batch, hw, seed, sigma)
        with torch.no_grad():
            y = ref_net(x.clone())
            yo = orc.grl_forward(sd, cfg, x.clone())
        del ref_net
        err = (y - yo).abs().max().item()
        assert err == 0.0, (name, err)
        print(f"[{name}] x {tuple(x.shape)} -> out {tuple(y.shape)}; |oracle - reference| max = {err}", flush=True)
        y = y.contiguous()
        files[name] = dict(x=x.numpy(), sub=y[..., ::stride, ::stride].contiguous().numpy(), stride=np.int64(stride),
                           shape=np.array(y.shape, dtype=np.int64),
                           sha256=np.array(hashlib.sha256(y.numpy().tobytes()).hexdigest()))
        meta[name] = dict(kwargs=cfg, grl_config=cargs, batch=batch, hw=list(hw), input_seed=seed, noise_sigma=sigma,
                          style=style, weight_seed=0, stride=stride, out_shape=list(y.shape), params=params)
    if args.check:
        print("check OK (fixtures not rewritten)")
        return
    for name, arrs in files.items():
        path = os.path.join(GOLD, f"zoo_{name}.npz")
        np.savez_compressed(path, **arrs)
        size = os.path.getsize(path)
        assert size < 1 << 20, (path, size)
        print(f"{path}: {size} bytes")
    text = json.dumps({"cases": meta,
                       "params": "param_summary of the reference network's state_dict (index / mask / table buffers "
                                 "excluded)",
                       "arrays": {"x": "(B, in_channels, H, W) float32: oracle.synth_input(shape, input_seed, noise_sigma)",
                                  "sub": "output[..., ::stride, ::stride] float32 of the reference GRL(**kwargs) with "
                                         "oracle.synth_state_dict(kwargs, weight_seed, style)",
                                  "sha256": "sha256 of the full float32 output (C order)"}}, indent=1)
    # lists of scalars (shapes, depths) on one line
    text = re.sub(r"\[\s+([^\[\]{}]*?)\s+\]", lambda m: "[" + " ".join(m.group(1).split()) + "]", text)
    with open(os.path.join(GOLD, "zoo_cases.json"), "w") as f:
        f.write(text + "\n")
    print("fixtures written to", GOLD)


if __name__ == "__main__":
    main()
