"""CUDA-event time per image of the device metrics: metrics.niqe (features kernels + batched float64 distance) and
metrics.psnrb_fused, at B = 1 and 16, at 1024 x 1024 and 1356 x 2040 RGB.  Prints the card's name and power limit with
the numbers.

    python tools/time_metrics.py --params tests/golden/niqe_pris_params.npz [--iters 20]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from _pkgload import load_package  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return out.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def time_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    times.sort()
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--params", required=True, help="niqe_pris_params.npz")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    load_package()
    import numpy as np

    from grl_image_restoration_b200 import metrics

    prm = dict(np.load(args.params))

    print(f"device: {torch.cuda.get_device_name()}  power limit: {power_limit()}")
    g = torch.Generator(device="cuda").manual_seed(0)
    for h, w in ((1024, 1024), (1356, 2040)):
        for b in (1, 16):
            x = torch.rand(b, 3, h, w, device="cuda", generator=g)
            t = torch.rand(b, 3, h, w, device="cuda", generator=g)
            n = time_ms(lambda: metrics.niqe(x, prm), args.iters)
            p = time_ms(lambda: metrics.psnrb_fused(x, t), args.iters)
            print(f"{h}x{w} B={b:2d}: niqe {n / b:8.3f} ms/image   psnrb_fused {p / b:7.4f} ms/image  (median of {args.iters})")


if __name__ == "__main__":
    main()
