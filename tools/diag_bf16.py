"""Dev tool: where does the bf16 path deviate from the fp32 path?  Per-block relative error with identical inputs."""
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _pkgload import load_package  # noqa: E402

pkg = load_package()
import grl_oracle as orc  # noqa: E402

variant = sys.argv[1] if len(sys.argv) > 1 else "base"
size = int(sys.argv[2]) if len(sys.argv) > 2 else 64
cfg = pkg.configs.grl_config(variant, "sr", 4, size)
for mode in ("synth", "scale10", "scale30"):
    sd = orc.synth_state_dict(cfg, 0)
    if mode != "synth":
        for k in sd:
            if k.endswith("logit_scale"):
                sd[k] = torch.full_like(sd[k], math.log(10.0 if mode == "scale10" else 30.0))
    m = pkg.GRL(**cfg)
    m.load_state_dict(sd, strict=False)
    m = m.cuda().eval()
    x = orc.synth_input((1, 3, size, size), seed=5).cuda()
    m.set_precision("fp32")
    stage_in = {}  # each stage's input in the fp32 forward
    hooks = [layer.register_forward_pre_hook(lambda mod, args, si=si: stage_in.__setitem__(si, args[0].clone()))
             for si, layer in enumerate(m.layers)]
    y32 = m(x)
    for h in hooks:
        h.remove()
    m.set_precision("bf16")
    y16 = m(x)
    psnr = (-10 * torch.log10(((y16 - y32) ** 2).mean())).item()
    print(f"[{mode}] end-to-end PSNR(bf16, fp32) = {psnr:.1f} dB  max-abs {(y16 - y32).abs().max().item():.3e}  out rms {y32.pow(2).mean().sqrt().item():.3f}")
    # per-block: same fp32 input through both paths
    m.set_precision("fp32")
    H, W = size, size
    tim = m.get_table_index_mask(x.device, (H, W))
    worst = []
    for si, layer in enumerate(m.layers):
        r = stage_in[si]
        for bi, blk in enumerate(layer.blocks):
            blk.precision = "fp32"
            o32 = blk(r, (H, W), tim)
            blk.precision = "bf16"
            o16 = blk(r, (H, W), tim)
            blk.precision = "fp32"
            upd = (o32 - r)
            rel = ((o16 - o32).pow(2).mean().sqrt() / upd.pow(2).mean().sqrt()).item()
            worst.append((rel, si, bi))
            r = o32
    worst.sort(reverse=True)
    print("   per-block rms(err)/rms(update): median %.4f  worst %s" % (sorted(w[0] for w in worst)[len(worst) // 2], [(round(a, 4), s, b) for a, s, b in worst[:4]]))
