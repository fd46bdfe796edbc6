"""CUDA-event time of the SR test command's LR input made on the device (imresize_list, MATLAB bicubic downscale), next
to the float64 numpy oracle on the host plus the copy of its result to the device, and to one SR forward of the LR image
it makes, with the card's name and power limit.  One JSON line per measurement.

Lists (seeded random pixels; the resize's work depends only on the sizes):
  div2k     100 colour images of 2040 x 1356 (DIV2K's HR size), s = 2, 3, 4
  urban100  100 colour images, half 1024 x 768 and half 768 x 1024, s = 2, 3, 4
  set14     14 colour images of 500 x 480 (about Set14's sizes), s = 2, 3, 4
Arms: imresize_list (median of --iters runs after a warm-up) with the bytes it must move (the 8-bit input once, the
float32 output once) over 3.35 TB/s, the H100 SXM data sheet's HBM3 bandwidth; the oracle (oracle/imresize_oracle.py,
float64 numpy, then .float().cuda()) on --host-images images of the list, per image; one fp16 forward of sr_grl_small
at that scale on the LR of one image of the list (seeded weights).  The device output is checked within the derived
bound of the oracle on the first image of each list before anything is printed.

    python tools/time_imresize.py [--iters 10] [--host-images 2]
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
from time_metrics import H100_HBM_BYTES_PER_S, alternated_ms, power_limit  # noqa: E402

import imresize_oracle as oracle  # noqa: E402

LISTS = {
    "div2k": [(1356, 2040)] * 100,
    "urban100": [(1024, 768), (768, 1024)] * 50,
    "set14": [(480, 500)] * 14,
}


def host_oracle(img, s):
    """The float64 oracle of one (H, W, 3) uint8 image, its float32 result copied to the device."""
    x = (img.astype(np.float64) / 255.0).astype(np.float32).astype(np.float64).transpose(2, 0, 1)
    return torch.from_numpy(oracle.resize(x, s)).float().cuda()


def model(pkg, s):
    import grl_oracle as orc  # weights only

    name = f"sr_grl_small_c3x{s}.ckpt"
    cfg = pkg.configs.released_config(name, 256)
    m = pkg.GRL(**cfg)
    m.load_state_dict(orc.synth_state_dict(cfg, 0, "init"), strict=False)
    m = m.cuda().eval()
    m.set_precision("fp16")
    return name, m


def emit(device, limit, **kw):
    print(json.dumps({"device": device, "power_limit": limit, **kw}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--host-images", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_imresize.py times CUDA kernels: no GPU found")
    pkg = load_package()
    device, limit = torch.cuda.get_device_name(), power_limit()
    with torch.no_grad():
        for name, sizes in LISTS.items():
            rng = np.random.default_rng(len(sizes))
            host = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
            imgs = [torch.from_numpy(x).cuda() for x in host]
            for s in oracle.SCALES:
                lr = pkg.imresize_list(imgs[:1], 1 / s)[0]
                v = pkg.functional.u8_to_f32(imgs[0][None])[0].double().cpu().numpy()
                if not (np.abs(lr.double().cpu().numpy() - oracle.resize(v, s)) <= oracle.host_bound(v, s)).all():
                    raise SystemExit(f"{name} s={s}: device output outside the bound of the oracle")
                (t_dev,) = alternated_ms([lambda: pkg.imresize_list(imgs, 1 / s)], args.iters, warmup=2)
                nbytes = sum(3 * h * w + 4 * 3 * (-(-h // s)) * (-(-w // s)) for h, w in sizes)
                emit(device, limit, what="imresize_list", list=name, scale=f"1/{s}", images=len(sizes),
                     ms=round(t_dev, 3), ms_per_image=round(t_dev / len(sizes), 4), bytes=nbytes,
                     hbm_floor_ms=round(nbytes / H100_HBM_BYTES_PER_S * 1e3, 3),
                     share_of_hbm=round(nbytes / H100_HBM_BYTES_PER_S * 1e3 / t_dev, 3))
                t_host = []
                for x in host[: args.host_images]:
                    t0 = time.perf_counter()
                    host_oracle(x, s)
                    torch.cuda.synchronize()
                    t_host.append((time.perf_counter() - t0) * 1e3)
                emit(device, limit, what="host_oracle_float64_plus_copy", list=name, scale=f"1/{s}",
                     ms_per_image=round(sorted(t_host)[len(t_host) // 2], 1))
                ckpt, m = model(pkg, s)
                (t_fwd,) = alternated_ms([lambda: m.forward_list([lr])], 3, warmup=1)
                (t_one,) = alternated_ms([lambda: pkg.imresize_list(imgs[:1], 1 / s)], args.iters, warmup=2)
                emit(device, limit, what=f"forward_list {ckpt} fp16", list=name, lr=list(lr.shape[1:]),
                     ms=round(t_fwd, 2), imresize_one_image_ms=round(t_one, 4),
                     imresize_share_of_forward=round(t_one / t_fwd, 5))
                del m
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
