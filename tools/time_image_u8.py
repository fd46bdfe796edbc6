"""CUDA-event time of the 8-bit image path on one GPU, with the card's name and power limit:

1. the two conversion kernels (functional.u8_to_f32 on the input, f32_to_u8 on the output) against the forward they
   wrap, on one per-GPU batch of the cfg4 workload (GRL-Base x4 SR, 16 tiles of 256 x 256, fp16 tensor cores);
2. psnr_fused, ssim_fused, psnrb_fused and niqe on 8-bit (B, H, W, 3) images against the same metric on fp32
   (B, 3, H, W) images, timed alternately, at 1024 x 1024 and 1356 x 2040 with B = 1 and 16.  For the two HBM-bound
   metrics (PSNR, PSNR-B) it also prints the bytes each has to read (two images, once) over its time.

Protocol of tools/time_metrics.py: median of 20 after 3 warm-ups.

    python tools/time_image_u8.py --params tests/golden/niqe_pris_params.npz [--iters 20] [--skip-forward]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _pkgload import load_package  # noqa: E402
from time_metrics import alternated_ms, power_limit, time_ms  # noqa: E402


def conversions(pkg, iters):
    import grl_oracle as orc  # weights only

    from grl_image_restoration_b200 import functional as K

    variant, task, scale, tile, per_gpu = "base", "sr", 4, 256, 16  # bench.py's cfg4, one GPU's batch
    cfg = pkg.configs.grl_config(variant, task, scale, tile)
    m = pkg.GRL(**cfg)
    m.load_state_dict(orc.synth_state_dict(cfg, 0, "init"), strict=False)
    m = m.cuda().eval()
    m.set_precision("fp16")
    g = torch.Generator(device="cuda").manual_seed(0)
    img = torch.randint(0, 256, (per_gpu, tile, tile, 3), device="cuda", dtype=torch.uint8, generator=g)
    x = K.u8_to_f32(img)
    y = m(x)
    t_fwd = time_ms(lambda: m(x), iters)
    t_in = time_ms(lambda: K.u8_to_f32(img), iters)
    t_out = time_ms(lambda: K.f32_to_u8(y), iters)
    t_all = time_ms(lambda: m.forward_u8(img), iters)
    print(f"cfg4 batch of {per_gpu} tiles {tile}x{tile} x{scale} fp16: forward {t_fwd:8.3f} ms   forward_u8 {t_all:8.3f} ms")
    for name, t, nbytes in (("u8_to_f32", t_in, img.numel() * 5), ("f32_to_u8", t_out, y.numel() * 5)):
        print(f"  {name} {tuple(img.shape if name == 'u8_to_f32' else y.shape)}: {t:7.4f} ms = {100 * t / t_fwd:.3f} % of "
              f"the forward   {nbytes / (t * 1e-3) / 1e12:.3f} TB/s (1 byte read + 4 written per element, or the reverse)")


def metrics_u8_vs_f32(params, iters):
    import numpy as np

    from grl_image_restoration_b200 import functional as K, metrics

    prm = dict(np.load(params))
    g = torch.Generator(device="cuda").manual_seed(0)
    for h, w in ((1024, 1024), (1356, 2040)):
        for b in (1, 16):
            a8 = torch.randint(0, 256, (b, h, w, 3), device="cuda", dtype=torch.uint8, generator=g)
            t8 = torch.randint(0, 256, (b, h, w, 3), device="cuda", dtype=torch.uint8, generator=g)
            a32, t32 = K.u8_to_f32(a8), K.u8_to_f32(t8)
            for name, fn, hbm in (("psnr_fused", lambda a, t: metrics.psnr_fused(a, t), True),
                                  ("ssim_fused", lambda a, t: metrics.ssim_fused(a, t), False),
                                  ("psnrb_fused", lambda a, t: metrics.psnrb_fused(a, t), True),
                                  ("niqe", lambda a, t: metrics.niqe(a, prm), False)):
                u8, f32 = alternated_ms([lambda: fn(a8, t8), lambda: fn(a32, t32)], iters)
                line = f"{h}x{w} B={b:2d} {name:11s}: uint8 {u8 / b:8.4f} ms/image   fp32 {f32 / b:8.4f} ms/image   x{f32 / u8:.2f}"
                if hbm:
                    line += (f"   read {2 * a8.numel() / (u8 * 1e-3) / 1e12:.2f} TB/s (uint8) / "
                             f"{2 * a32.numel() * 4 / (f32 * 1e-3) / 1e12:.2f} TB/s (fp32)")
                print(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--params", required=True, help="niqe_pris_params.npz")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--skip-forward", action="store_true", help="time the metrics only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_image_u8.py times CUDA kernels: no GPU found")
    pkg = load_package()
    print(f"device: {torch.cuda.get_device_name()}  power limit: {power_limit()}")
    with torch.no_grad():
        if not args.skip_forward:
            conversions(pkg, args.iters)
        metrics_u8_vs_f32(args.params, args.iters)


if __name__ == "__main__":
    main()
