"""Dev tool: time GRL.forward for a named config on cuda:0 (CUDA events)."""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _pkgload import load_package  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--variant", default="base")
ap.add_argument("--task", default="sr", help="configs.grl_config task: sr, dn, deblur, jpeg, dm, bsr, defocus, defocus_dual")
ap.add_argument("--in-channels", type=int, default=3, help="dn / jpeg: 1 for the grayscale checkpoints")
ap.add_argument("--scale", type=int, default=4)
ap.add_argument("--size", type=int, default=256)
ap.add_argument("--batch", type=int, default=1)
ap.add_argument("--iters", type=int, default=3)
ap.add_argument("--precision", default=None)
ap.add_argument("--style", default="spread")
ap.add_argument("--cuda-graph", action="store_true", help="replay a captured CUDA graph of the forward (GRL.use_cuda_graph)")
ap.add_argument("--attn-variants", default="5", help="comma list of grl_tc_attn_variant values to time in turn (A/B in one process)")
a = ap.parse_args()
pkg = load_package()
import grl_oracle as orc  # noqa: E402  (weights only)

cfg = pkg.configs.grl_config(a.variant, a.task, a.scale, a.size, in_channels=a.in_channels)
m = pkg.GRL(**cfg)
m.load_state_dict(orc.synth_state_dict(cfg, 0, a.style), strict=False)
m = m.cuda().eval()
if a.precision is not None and hasattr(m, "set_precision"):
    m.set_precision(a.precision)
x = torch.rand(a.batch, cfg["in_channels"], a.size, a.size, device="cuda")
from grl_image_restoration_b200 import capi  # noqa: E402

if a.cuda_graph:
    m.use_cuda_graph = True
for variant in [int(v) for v in a.attn_variants.split(",")]:
    capi.lib().grl_tc_attn_variant(variant)
    if a.cuda_graph:
        m.reset_cuda_graphs()
    y0 = m(x)
    torch.cuda.synchronize()
    if variant == int(a.attn_variants.split(",")[0]):
        y_first = y0
    ts = []
    for _ in range(a.iters):
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        y = m(x)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = sorted(ts)[len(ts) // 2]
    print(f"{a.variant}/{a.task} x{a.scale} {a.size}^2 B={a.batch} prec={a.precision} attn_variant={variant}{" cuda-graph" if a.cuda_graph else ""}: {ms:.1f} ms/forward, "
          f"{a.batch * a.size * a.size / 1e6 / (ms / 1e3):.4f} Mpix/s, peak mem {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB, "
          f"max |y - y(first variant)| = {(y0 - y_first).abs().max().item():.3e}")
