"""CUDA-event time of the denoising test command's noisy input made on the device (awgn_list), next to the same input
made as the reference's dataset makes it (numpy's RandomState noise on the host, the float32 add, then the copy to the
device) and to the dn forwards it feeds, with the card's name and power limit.  One JSON line per measurement.

Lists (seeded random pixels; the noise's work depends only on the sizes and keys):
  cbsd68    68 colour images, half 480 x 320 and half 320 x 480, keys "CBSD68/<i>.png"
  urban100  100 colour images, half 1024 x 768 and half 768 x 1024, all keyed "Urban100/img" as the reference keys them
Arms: awgn_list at sigma 15 (median of --iters runs after a warm-up); the host recipe over the same list (wall clock
around the whole list, ending in a device synchronise; median of --host-iters); one forward of dn_grl_small_c3s15 and
one forward_tile of dn_grl_base_c3s15 at 256 / 32 on a 480 x 320 image (fp16 tensor cores, seeded weights).  The device
output is checked equal to the host recipe on the first and last images of each list before anything is printed.

    python tools/time_awgn.py [--iters 10] [--host-iters 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _pkgload import load_package  # noqa: E402
from time_metrics import alternated_ms, power_limit  # noqa: E402

SIGMA = 15
LISTS = {
    "cbsd68": ([(480, 320), (320, 480)] * 34, lambda i: f"CBSD68/{i:04d}.png"),
    "urban100": ([(1024, 768), (768, 1024)] * 50, lambda i: f"Urban100/img_{i + 1:03d}.png"),
}


def host_recipe(pkg, host_imgs, seeds):
    """The reference's pipeline: noise and add on the host, then the copy of img_lq to the device."""
    outs = []
    for x, s in zip(host_imgs, seeds):
        gt = torch.from_numpy(np.ascontiguousarray(x.transpose(2, 0, 1))).float().div(255)
        noise = np.random.RandomState(pkg.dn_seed(s)).normal(0, SIGMA / 255, gt.shape)
        outs.append((gt + torch.from_numpy(noise).float()).cuda())
    torch.cuda.synchronize()
    return outs


def model(pkg, ckpt):
    import grl_oracle as orc  # weights only

    *_, tile, overlap = pkg.configs.RELEASED[ckpt]
    cfg = pkg.configs.released_config(ckpt, tile or 128)
    m = pkg.GRL(**cfg)
    m.load_state_dict(orc.synth_state_dict(cfg, 0, "init"), strict=False)
    m = m.cuda().eval()
    m.set_precision("fp16")
    return m, tile, overlap


def emit(device, limit, **kw):
    print(json.dumps({"device": device, "power_limit": limit, **kw}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--host-iters", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_awgn.py times CUDA kernels: no GPU found")
    pkg = load_package()
    from grl_image_restoration_b200 import tiling

    device, limit = torch.cuda.get_device_name(), power_limit()
    with torch.no_grad():
        for name, (sizes, key) in LISTS.items():
            rng = np.random.default_rng(len(sizes))
            host = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
            imgs = [torch.from_numpy(x).cuda() for x in host]
            seeds = [key(i) for i in range(len(sizes))]
            lq = pkg.awgn_list(imgs, SIGMA, seeds)
            want = host_recipe(pkg, [host[0], host[-1]], [seeds[0], seeds[-1]])
            if not (torch.equal(lq[0], want[0]) and torch.equal(lq[-1], want[1])):
                raise SystemExit(f"{name}: device noise differs from the host recipe")
            (t_dev,) = alternated_ms([lambda: pkg.awgn_list(imgs, SIGMA, seeds)], args.iters, warmup=2)
            t_host = []
            for _ in range(args.host_iters):
                t0 = time.perf_counter()
                host_recipe(pkg, host, seeds)
                t_host.append((time.perf_counter() - t0) * 1e3)
            samples = 3 * sum(h * w for h, w in sizes)
            emit(device, limit, what="awgn_list", list=name, images=len(sizes), samples=samples, ms=round(t_dev, 3),
                 msamples_per_s=round(samples / t_dev / 1e3, 1))
            emit(device, limit, what="host_numpy_plus_copy", list=name, images=len(sizes), samples=samples,
                 ms=round(sorted(t_host)[len(t_host) // 2], 1))
        x = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (320, 480, 3), dtype=np.uint8)).cuda()
        lq = pkg.awgn_list([x], SIGMA, ["CBSD68/0001.png"])[0][None]
        (t_one,) = alternated_ms([lambda: pkg.awgn_list([x], SIGMA, ["CBSD68/0001.png"])], args.iters, warmup=2)
        emit(device, limit, what="awgn_list", list="one_480x320", images=1, samples=x.numel(), ms=round(t_one, 3))
        m, _, _ = model(pkg, "dn_grl_small_c3s15.ckpt")
        (t_small,) = alternated_ms([lambda: m(lq)], 5, warmup=2)
        emit(device, limit, what="forward dn_grl_small_c3s15 fp16", size="480x320", ms=round(t_small, 2))
        del m
        m, tile, overlap = model(pkg, "dn_grl_base_c3s15.ckpt")
        (t_base,) = alternated_ms([lambda: tiling.forward_tile(m, lq, tile, overlap)], 3, warmup=1)
        emit(device, limit, what=f"forward_tile dn_grl_base_c3s15 fp16 {tile}/{overlap}", size="480x320",
             ms=round(t_base, 2))


if __name__ == "__main__":
    main()
