"""CUDA-event time of the device JPEG round trip (jpeg_roundtrip_list) over lists shaped like the JPEG test sets, next to
one forward_tile_list_u8 of the released jpeg-Small model on the same list, with the card's name and power limit.

Lists (seeded random pixels; the round trip's work depends only on the sizes):
  classic5  5 gray images of 512 x 512
  live1     8 colour images, half 768 x 512 and half 512 x 768
  bsds500   8 images, half 481 x 321 and half 321 x 481, gray and colour
Arms, per list: jpeg_roundtrip_list at q = 10 (median of --iters runs after a warm-up); forward_tile_list_u8 of
jpeg_grl_small_c{1,3}q10 (fp16 tensor cores, seeded weights) at tile 288 / overlap 36 on the round trip's output; and,
where OpenCV is importable, cv2's encode + decode loop on the host over the same images (wall clock, one thread as
cv2 runs it).  The device output is checked equal to the host loop's before anything is printed.

    python tools/time_jpeg.py [--iters 20] [--lists classic5,live1,bsds500_c1,bsds500_c3]
"""
import argparse
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

LISTS = {
    "classic5": (1, [(512, 512)] * 5),
    "live1": (3, [(768, 512), (512, 768)] * 4),
    "bsds500_c1": (1, [(481, 321), (321, 481)] * 4),
    "bsds500_c3": (3, [(481, 321), (321, 481)] * 4),
}
Q = 10


def cv2_loop(imgs):
    try:
        import cv2
    except ImportError:
        return None, None
    outs, t0 = [], time.perf_counter()
    for x in imgs:
        p = [int(cv2.IMWRITE_JPEG_QUALITY), Q]
        if x.shape[2] == 3:
            enc = cv2.imencode(".jpg", cv2.cvtColor(x, cv2.COLOR_RGB2BGR), p)[1]
            outs.append(cv2.cvtColor(cv2.imdecode(enc, 1), cv2.COLOR_BGR2RGB))
        else:
            outs.append(cv2.imdecode(cv2.imencode(".jpg", x, p)[1], 0)[..., None])
    return (time.perf_counter() - t0) * 1e3, outs


def model(pkg, C):
    import grl_oracle as orc  # weights only

    ckpt = f"jpeg_grl_small_c{C}q10.ckpt"
    *_, tile, overlap = pkg.configs.RELEASED[ckpt]
    cfg = pkg.configs.released_config(ckpt, tile)
    m = pkg.GRL(**cfg)
    m.load_state_dict(orc.synth_state_dict(cfg, 0, "init"), strict=False)
    m = m.cuda().eval()
    m.set_precision("fp16")
    return m, tile, overlap


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--lists", default=",".join(LISTS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_jpeg.py times CUDA kernels: no GPU found")
    pkg = load_package()
    from grl_image_restoration_b200 import tiling

    print(f"device: {torch.cuda.get_device_name()}  power limit: {power_limit()}")
    models = {}
    with torch.no_grad():
        for name in args.lists.split(","):
            C, sizes = LISTS[name]
            rng = np.random.default_rng(len(sizes) * 10 + C)
            host = [rng.integers(0, 256, (h, w, C), dtype=np.uint8) for h, w in sizes]
            imgs = [torch.from_numpy(x).cuda() for x in host]
            lq = pkg.jpeg_roundtrip_list(imgs, Q)
            for x, y in zip(host, lq):
                if not torch.equal(pkg.jpeg_roundtrip_host(torch.from_numpy(x), Q), y.cpu()):
                    raise SystemExit(f"{name}: device round trip differs from the host expansion")
            t_cv, cv_out = cv2_loop(host)
            if cv_out is not None and not all(np.array_equal(a, b.cpu().numpy()) for a, b in zip(cv_out, lq)):
                raise SystemExit(f"{name}: device round trip differs from cv2")
            (t_dev,) = alternated_ms([lambda: pkg.jpeg_roundtrip_list(imgs, Q)], args.iters)
            if C not in models:
                models[C] = model(pkg, C)
            m, tile, overlap = models[C]
            fwd = lambda: tiling.forward_tile_list_u8(m, lq, tile, overlap)  # noqa: E731
            (t_fwd,) = alternated_ms([fwd], 3, warmup=1)
            mpix = sum(h * w for h, w in sizes) / 1e6
            cv = f"{t_cv:8.2f} ms" if t_cv is not None else "  (no cv2)"
            print(f"{name:11s} C={C} {len(sizes)} images {mpix:5.2f} Mpixel: jpeg_roundtrip_list {t_dev:7.3f} ms "
                  f"({mpix / t_dev * 1e3:7.1f} Mpixel/s) | cv2 loop {cv} | forward_tile_list_u8 jpeg-Small "
                  f"{tile}/{overlap} {t_fwd:9.1f} ms  (round trip = {100 * t_dev / t_fwd:.2f} % of the forward)")


if __name__ == "__main__":
    main()
