"""Golden outputs of the UNMODIFIED reference network for the anchor_proj_type / anchor_one_stage / conv_type switches
(mixed_attn_block.py:679-785, swin_v1_block.py:457-485).  Runs only where the reference exists:

    python oracle/make_golden_switches.py            # validate + (re)write fixtures
    python oracle/make_golden_switches.py --check    # validate only

Each case builds the reference GRL from configs.micro_config (4 blocks: both stripe personalities, shifted and not)
with the switches, loads switch_cases.synth_state_dict ("routed" weights: every Linear bias non-zero) and runs it (fp32, CPU) on a 27 x 21 input (reflect padding).
A case the reference cannot build or run is recorded with its exception.  The restatement switch_cases.grl_forward
must reproduce each output bit for bit.

Fixtures: tests/golden/switches_cases.json (kwargs, the reference's parameter names and shapes as param_summary records
them, or the failure) and tests/golden/switches_<name>.npz (x, y: input and full output, float32).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import grl_oracle as orc  # noqa: E402
import switch_cases as sw  # noqa: E402
from _pkgload import load_package  # noqa: E402
from _ref_import import import_reference  # noqa: E402
from make_golden_zoo import param_summary  # noqa: E402

configs = load_package().configs
HW = (27, 21)

# name: (anchor_proj_type, anchor_one_stage, df, conv_type)
CASES = {
    "maxpool_df2": ("maxpool", True, 2, "1conv"),
    "maxpool_df4": ("maxpool", True, 4, "1conv"),
    "conv2d_df2": ("conv2d", True, 2, "1conv"),
    "conv2d_df4": ("conv2d", True, 4, "1conv"),
    "patchmerging_df2": ("patchmerging", True, 2, "1conv"),
    "conv2d_ms_df2": ("conv2d", False, 2, "1conv"),
    "conv2d_ms_df4": ("conv2d", False, 4, "1conv"),
    "patchmerging_ms_df2": ("patchmerging", False, 2, "1conv"),
    "patchmerging_ms_df4": ("patchmerging", False, 4, "1conv"),
    "3conv": ("avgpool", True, 2, "3conv"),
    "1conv1x1": ("avgpool", True, 2, "1conv1x1"),
    "linear": ("avgpool", True, 2, "linear"),
    "conv2d_ms_df4_3conv": ("conv2d", False, 4, "3conv"),
    # expected to fail in the reference
    "conv2d_df1": ("conv2d", True, 1, "1conv"),
    "conv2d_df3": ("conv2d", True, 3, "1conv"),
    "patchmerging_df4": ("patchmerging", True, 4, "1conv"),
    "patchmerging_df1": ("patchmerging", True, 1, "1conv"),
    "avgpool_ms_df2": ("avgpool", False, 2, "1conv"),
    "maxpool_ms_df4": ("maxpool", False, 4, "1conv"),
    "conv2d_ms_df1": ("conv2d", False, 1, "1conv"),
    "patchmerging_ms_df1": ("patchmerging", False, 1, "1conv"),
    "conv2d_ms_df3": ("conv2d", False, 3, "1conv"),
}


def case_config(proj, one_stage, df, conv_type):
    # df 3 needs stripes divisible by 3: (12, 24) stripes, 48 x 48 img_size
    kw = dict(stripe=(12, 24), img_size=48) if df == 3 else {}
    cfg = configs.micro_config(df=df, **kw)
    cfg.update(anchor_proj_type=proj, anchor_one_stage=one_stage, conv_type=conv_type)
    return cfg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    grl_mod, _, _, _ = import_reference()
    torch.set_num_threads(os.cpu_count())
    files, meta = {}, {}
    for seed, (name, sw_args) in enumerate(CASES.items()):
        cfg = case_config(*sw_args)
        rec = dict(kwargs=cfg, switches=dict(zip(("anchor_proj_type", "anchor_one_stage", "df", "conv_type"), sw_args)))
        x = orc.synth_input((1, 3, *HW), seed=100 + seed)
        try:
            torch.manual_seed(0)
            ref_net = grl_mod.GRL(**cfg).eval()
            shapes = {k: list(v.shape) for k, v in ref_net.state_dict().items()
                      if k.split("_")[0] not in ("table", "index", "mask")}
            sd = sw.synth_state_dict(orc, cfg, shapes)
            missing, unexpected = ref_net.load_state_dict(sd, strict=False)
            assert not unexpected and all(k.split("_")[0] in ("table", "index", "mask") for k in missing)
            with torch.no_grad():
                y = ref_net(x.clone())
        except Exception as e:  # the reference cannot run this combination
            rec.update(valid=False, error=f"{type(e).__name__}: {e}"[:300])
            print(f"[{name}] reference fails: {rec['error']}", flush=True)
            meta[name] = rec
            continue
        with torch.no_grad():
            yo = sw.grl_forward(orc, sd, cfg, x.clone())
        err = (y - yo).abs().max().item()
        assert err == 0.0, (name, err)
        print(f"[{name}] x {tuple(x.shape)} -> {tuple(y.shape)}; |restatement - reference| max = {err}", flush=True)
        rec.update(valid=True, input_seed=100 + seed, weight_seed=0, style="routed", params=param_summary(shapes),
                   param_shapes={k: v for k, v in sorted(shapes.items())
                                 if ".anchor." in k or ".conv." in k and ".blocks." not in k or "conv_after_body" in k})
        files[name] = dict(x=x.numpy(), y=y.contiguous().numpy())
        meta[name] = rec
    if args.check:
        print("check OK (fixtures not rewritten)")
        return
    for name, arrs in files.items():
        np.savez_compressed(os.path.join(sw.GOLD, f"switches_{name}.npz"), **arrs)
    with open(os.path.join(sw.GOLD, "switches_cases.json"), "w") as f:
        json.dump({"cases": meta, "hw": list(HW)}, f, indent=1)
        f.write("\n")
    print("fixtures written to", sw.GOLD)


if __name__ == "__main__":
    main()
