"""Dev tool: one forward of GRL-Base x4 SR on 256^2 inputs for each anchor projection and stage-conv type, against the
released avgpool / 1conv model, on cuda:0 (CUDA events).

Every variant is built and warmed up first (its packed weights, attention constants and every launch shape), then the
variants are timed in turns, one forward of each per round, so that clock and co-tenant drift spread over all of them.
Reports the median over the rounds, the card and its power limit.  The anchor variants change only the anchor
projection of each block; the conv variants change only the stage convs and conv_after_body.

    python tools/time_switches.py [--precision fp16] [--batch 1] [--rounds 20]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from _pkgload import load_package  # noqa: E402

# name: (anchor_proj_type, anchor_one_stage, conv_type); df is the released 2 except where a type needs another
VARIANTS = {
    "released avgpool/1conv": ("avgpool", True, "1conv"),
    "anchor maxpool": ("maxpool", True, "1conv"),
    "anchor conv2d": ("conv2d", True, "1conv"),
    "anchor patchmerging": ("patchmerging", True, "1conv"),
    "anchor conv2d two-stage": ("conv2d", False, "1conv"),
    "anchor patchmerging two-stage": ("patchmerging", False, "1conv"),
    "conv 3conv": ("avgpool", True, "3conv"),
    "conv 1conv1x1": ("avgpool", True, "1conv1x1"),
    "conv linear": ("avgpool", True, "linear"),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="fp16", choices=("fp32", "fp16", "bf16"))
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_switches: no CUDA device")
    pkg = load_package()
    import grl_oracle as orc
    import switch_cases as sw

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card or torch.cuda.get_device_name(0)}; precision {a.precision}; B={a.batch}, {a.size}^2 input")
    x = torch.rand(a.batch, 3, a.size, a.size, generator=torch.Generator().manual_seed(0)).cuda()
    models = {}
    for name, (proj, one, conv) in VARIANTS.items():
        cfg = pkg.configs.grl_config("base", "sr", 4, a.size)
        cfg.update(anchor_proj_type=proj, anchor_one_stage=one, conv_type=conv)
        m = pkg.GRL(**cfg)
        shapes = {k: list(v.shape) for k, v in m.state_dict().items() if k.split("_")[0] not in ("table", "index", "mask")}
        m.load_state_dict(sw.synth_state_dict(orc, cfg, shapes), strict=False)
        m = m.cuda().eval()
        m.set_precision(a.precision)
        for _ in range(a.warmup):
            m(x)
        models[name] = m
    torch.cuda.synchronize()
    times = {n: [] for n in models}
    with torch.no_grad():
        for _ in range(a.rounds):
            for name, m in models.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                m(x)
                e1.record()
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1))
    base = sorted(times["released avgpool/1conv"])[a.rounds // 2]
    for name, ts in times.items():
        ts = sorted(ts)
        med = ts[len(ts) // 2]
        print(f"{name:32s} median {med:8.2f} ms/forward  (min {ts[0]:.2f}, max {ts[-1]:.2f})  x{med / base:.3f} of released")


if __name__ == "__main__":
    main()
