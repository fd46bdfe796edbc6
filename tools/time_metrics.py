"""CUDA-event time per image of the device metrics: metrics.niqe (features kernels + batched float64 distance),
metrics.psnrb_fused, and metrics.ssim_fused against the torch-op pair metrics.ssim(., "rgb") + metrics.ssim(., "y") it
replaces in the validation step, timed alternately, at B = 1 and 16, at 1024 x 1024 and 1356 x 2040 RGB.  For ssim_fused
it also prints the bytes it has to read (two fp32 images, once) over its time, and that time's share of the float64
bound: the kernel needs SSIM_DFMA_PER_VALUE float64 FMAs per map value, which at the H100 SXM data sheet's 33.5 TFLOP/s
of FP64 (non-tensor; for a 700 W card) takes longer than reading its input at 3.35 TB/s.  Prints the card's name and
power limit with the numbers.

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


# float64 FMAs per SSIM map value of ssim_tile_kernel (csrc/metric.cu): five sums of 11 taps along the row for the 26 rows a
# 16-row tile stages, five sums of 11 taps down the column
SSIM_DFMA_PER_VALUE = 5 * 11 * 26 / 16 + 5 * 11
H100_FP64_FMA_PER_S = 33.5e12 / 2
H100_HBM_BYTES_PER_S = 3.35e12


def alternated_ms(fns, iters, warmup=3):
    """Median CUDA-event time of each callable, the callables taking turns inside one loop."""
    for _ in range(warmup):
        for fn in fns:
            fn()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(iters):
        for fn, ts in zip(fns, times):
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            fn()
            end.record()
            end.synchronize()
            ts.append(start.elapsed_time(end))
    return [sorted(ts)[len(ts) // 2] for ts in times]


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
            fused, eager = alternated_ms([lambda: metrics.ssim_fused(x, t),
                                          lambda: (metrics.ssim(x, t, 0, "rgb"), metrics.ssim(x, t, 0, "y"))], args.iters)
            values, nbytes = b * 4 * h * w, 2 * x.numel() * 4  # three channels and the luma; two fp32 images read once
            t_fp64, t_hbm = values * SSIM_DFMA_PER_VALUE / H100_FP64_FMA_PER_S, nbytes / H100_HBM_BYTES_PER_S
            print(f"{h}x{w} B={b:2d}: ssim_fused {fused / b:7.4f} ms/image   torch-op ssim rgb + y {eager / b:8.3f} ms/image   "
                  f"x{eager / fused:.1f}   {nbytes / (fused * 1e-3) / 1e12:.3f} TB/s of input   "
                  f"{100 * t_fp64 / (fused * 1e-3):.0f} % of the FP64 bound ({t_fp64 * 1e3:.3f} ms; HBM bound {t_hbm * 1e3:.3f} ms)")


if __name__ == "__main__":
    main()
