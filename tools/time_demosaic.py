"""Dev tool: cost of demosaicking packed RGGB Bayer planes on cuda:0.

1. The standalone kernel (functional.demosaic), timed alone over many launches, as GB/s of the HBM traffic it needs: the
   packed planes read once (16 B per quad) and the RGB image written once (48 B per quad).
2. A dm forward (GRL-Small, grl_config("small", "dm"), fp16 path) of packed planes with the demosaic fused into the head
   kernel (GRL(input_format="rggb")) against demosaic() followed by the RGB forward.  The two are timed alternately in the
   same run (CUDA events, median of --iters each); the difference is one fp32 round trip of the 3-channel image.
The card's name and power limit are read in the same run.

    python tools/time_demosaic.py [--iters 9] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _pkgload import load_package  # noqa: E402

KERNEL_SHAPES = [("16 x 256^2", (16, 4, 128, 128)), ("1 x 2048^2", (1, 4, 1024, 1024)), ("8 x 2048^2", (8, 4, 1024, 1024))]
FORWARD_BATCHES = [("1 x 256^2", 1), ("16 x 256^2", 16)]


def device_info():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def event_ms(fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=9)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_demosaic.py needs a CUDA device")
    pkg = load_package()
    import grl_oracle as orc  # weights only
    from grl_image_restoration_b200 import functional as K

    dev = device_info()
    print(f"device: {dev['name']}, power limit {dev['power_limit_w']} W")
    g = torch.Generator("cuda").manual_seed(0)
    kernel_rows = []
    for name, shape in KERNEL_SHAPES:
        x = torch.rand(shape, device="cuda", generator=g)
        for _ in range(3):
            K.demosaic(x)
        torch.cuda.synchronize()
        ms = sorted(event_ms(lambda: K.demosaic(x), reps=50) for _ in range(a.iters))[a.iters // 2]
        nbytes = 4 * (x.numel() + 3 * x.numel())  # 4 planes in, 3 channels at 4x the pixels out
        kernel_rows.append(dict(shape=name, cfa4=list(shape), ms=ms, gbps=nbytes / ms / 1e6))
        print(f"demosaic kernel {name}: {ms * 1e3:.1f} us, {nbytes / ms / 1e6:.0f} GB/s", flush=True)
        del x

    cfg = pkg.configs.grl_config("small", "dm", img_size=256)
    sd = orc.synth_state_dict(cfg, 0, "init")
    models = {}
    for fmt in ("rggb", "rgb"):
        m = pkg.GRL(input_format=fmt, **cfg)
        m.load_state_dict(sd, strict=False)
        m = m.cuda().eval()
        m.set_precision("fp16")
        models[fmt] = m
    forward_rows = []
    with torch.no_grad():
        for name, batch in FORWARD_BATCHES:
            cfa = torch.rand(batch, 4, 128, 128, device="cuda", generator=g)
            fused = lambda: models["rggb"](cfa)  # noqa: E731
            unfused = lambda: models["rgb"](K.demosaic(cfa))  # noqa: E731
            assert torch.equal(fused(), unfused())
            for _ in range(2):
                fused(), unfused()
            torch.cuda.synchronize()
            tf, tu = [], []
            for _ in range(a.iters):  # alternate, so drifting clocks hit both arms alike
                tf.append(event_ms(fused))
                tu.append(event_ms(unfused))
            f_ms, u_ms = sorted(tf)[a.iters // 2], sorted(tu)[a.iters // 2]
            forward_rows.append(dict(workload=name, batch=batch, fused_ms=f_ms, demosaic_then_forward_ms=u_ms,
                                     saving_ms=u_ms - f_ms, fused_min_ms=min(tf), unfused_min_ms=min(tu)))
            print(f"dm forward {name}: fused head {f_ms:.3f} ms, demosaic + forward {u_ms:.3f} ms, "
                  f"saving {u_ms - f_ms:+.3f} ms ({100 * (u_ms - f_ms) / u_ms:+.2f} %)", flush=True)
    result = dict(device=dev, precision="fp16", iters=a.iters, kernel=kernel_rows, forward=forward_rows)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
