"""Dev tool: cost of the x8 self-ensemble (GRL(self_ensemble=True)) against the plain forward on cuda:0, fp16 path.

Workloads: cfg4 (GRL-Base x4) with 1 and 16 tiles of 256^2, and cfg2 (GRL-Small x4, 16 tiles of 256^2).  For each:
the plain forward and the x8 forward (CUDA events, warm-ups first, median of --iters), their ratio, and the time of the
ensemble's own kernels (two gathers + one merge on the same shapes, timed alone over many launches) as a share of the x8
time.  The card's name and power limit are read in the same run.

    python tools/time_ensemble.py [--iters 3] [--out result.json]
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

WORKLOADS = [("cfg4_1tile", ("base", "sr", 4, 256), 1), ("cfg4_16tiles", ("base", "sr", 4, 256), 16),
             ("cfg2_16tiles", ("small", "sr", 4, 256), 16)]


def device_info():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def time_ms(fn, iters, warmup=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ensemble.py needs a CUDA device")
    pkg = load_package()
    import grl_oracle as orc  # weights only
    from grl_image_restoration_b200 import functional as K

    dev = device_info()
    print(f"device: {dev['name']}, power limit {dev['power_limit_w']} W")
    rows = []
    for name, model, batch in WORKLOADS:
        cfg = pkg.configs.grl_config(*model)
        m = pkg.GRL(**cfg)
        m.load_state_dict(orc.synth_state_dict(cfg, 0, "init"), strict=False)
        m = m.cuda().eval()
        m.set_precision("fp16")
        x = torch.rand(batch, 3, 256, 256, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
        with torch.no_grad():
            m.self_ensemble = False
            plain = time_ms(lambda: m(x), a.iters)
            m.self_ensemble = True
            x8 = time_ms(lambda: m(x), a.iters)
        s = cfg["upscale"]
        ya = torch.rand(4 * batch, 3, 256 * s, 256 * s, device="cuda")
        yb = torch.rand_like(ya)

        def glue():
            K.ens_gather(x, 0)
            K.ens_gather(x, 1)
            K.ens_merge(ya, yb, batch)

        glue_ms = time_ms(glue, 20, warmup=3)
        # HBM traffic of the three launches: each gather reads x once and writes 4 views; the merge reads 8 outputs
        # and writes one
        nbytes = 4 * (2 * 5 * x.numel() + 9 * batch * 3 * (256 * s) ** 2)
        r = dict(workload=name, model=list(model), tiles=batch, plain_ms=plain, x8_ms=x8, ratio=x8 / plain,
                 gather_merge_ms=glue_ms, gather_merge_share=glue_ms / x8, gather_merge_gbps=nbytes / glue_ms / 1e6)
        rows.append(r)
        print(f"{name}: plain {plain:.1f} ms, x8 {x8:.1f} ms, ratio {x8 / plain:.2f}; gather + merge {glue_ms:.3f} ms "
              f"({100 * glue_ms / x8:.3f} % of x8, {r['gather_merge_gbps']:.0f} GB/s)", flush=True)
        del m, ya, yb
        torch.cuda.empty_cache()
    result = dict(device=dev, precision="fp16", iters=a.iters, results=rows)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
