"""Dev tool: every tensor-core GEMM launch of one cfg4 block (GRL-Base x4 SR, 256^2 tiles, B = 16), plus a stage conv,
timed in isolation on cuda:0.

The launches are the forward's own (tc.gemm_launches): qkv, the CAB convs, proj (LayerNorm), fc1, fc2 (LayerNorm) and
the small ones of the block, on synthetic operands of the launch's shapes.  For each launch: CUDA-event time (median
of --iters batches of --reps launches, after warm-up), the bytes and FLOPs the launch needs (computed from its shapes:
operands read once, outputs written once), TB/s against the data-sheet 3.35 TB/s and TFLOP/s against the dense
fp16 / bf16 989 TFLOP/s, and which of the two bounds applies.

--old LIB times a second build of libgrl_b200.so (for instance the parent commit's, built separately) on the same
operands, alternating with this tree's library batch by batch, and reports the largest |new - old| output difference.

    python tools/time_gemm.py [--old path/to/libgrl_b200.so] [--fmt fp16|bf16] [--out result.json]
"""
import argparse
import json
import os
import re
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _pkgload import load_package  # noqa: E402
from time_attention import device_info, event_ms, load_lib  # noqa: E402

HBM_PEAK = 3.35e12  # B/s, H100 SXM data sheet
TENSOR_PEAK = 989e12  # dense fp16 / bf16, H100 SXM data sheet
OUTPUTS = ("out_bf16", "out_f32", "out_nchw")


def traffic(args):
    """(bytes, FLOPs) a launch needs: A, W, bias and the residual / CAB inputs read once, every output written once."""
    conv = args["taps"] == 9
    rows = args["image"][0] * args["image"][1] * args["image"][2] if conv else args["M"]
    nbytes = 0
    for k in ("x16", "w16", "bias", "res_f32", "cab_y", "cab_gate", "gamma", "beta", "slot_scale") + OUTPUTS:
        v = args.get(k)
        if v is not None and not isinstance(v, (int, float)):
            nbytes += torch.Size(v.shape).numel() * torch.empty((), dtype=v.dtype).element_size()
    return nbytes, 2 * rows * args["npad"] * args["kpad"] * args["taps"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old", default=None, help="a second libgrl_b200.so to time alternately on the same operands")
    ap.add_argument("--fmt", default="fp16", choices=("fp16", "bf16"))
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=21)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_gemm.py needs a CUDA device")
    pkg = load_package()
    from grl_image_restoration_b200 import capi, tc

    libs = {"new": capi.lib()}
    if a.old:
        libs["old"] = load_lib(a.old, capi)

    cfg = pkg.configs.grl_config("base", "sr", 4, 256)
    model = pkg.GRL(**cfg).to("cuda:0").eval()
    model.set_precision(a.fmt)
    launches = tc.gemm_launches(model, (a.batch, 3, 256, 256))
    block = re.match(r"(.*?block\d+)\.", next(ln.name for ln in launches if "block" in ln.name)).group(1)
    chosen = [ln for ln in launches if ln.name.startswith(block + ".")]
    conv = next((ln for ln in launches if "block" not in ln.name and ln.args["taps"] == 9 and "stage" in ln.name), None)
    if conv is not None:
        chosen.append(conv)
    g = torch.Generator("cuda").manual_seed(0)

    def tensor(spec, name):
        if name in ("gamma", "slot_scale"):
            return 0.5 + torch.rand(spec.shape, device="cuda", generator=g).to(spec.dtype)
        return (torch.randn(spec.shape, device="cuda", generator=g) * (0.1 if name == "w16" else 1.0)).to(spec.dtype)

    dev = device_info()
    print(f"device: {dev['name']}, power limit {dev['power_limit_w']} W, {a.fmt} operands, B = {a.batch}, block {block}",
          flush=True)
    rows = []
    for ln in chosen:
        ins = {k: tensor(v, k) for k, v in ln.args.items() if isinstance(v, tc.Spec) and k not in OUTPUTS}
        outs = {name: {k: torch.zeros(v.shape, device="cuda", dtype=v.dtype) for k, v in ln.args.items()
                       if isinstance(v, tc.Spec) and k in OUTPUTS} for name in libs}

        def launcher(name, kw):
            def run():
                saved, capi._lib = capi._lib, libs[name]
                try:
                    tc.gemm(**kw)
                finally:
                    capi._lib = saved
            return run

        fns = {name: launcher(name, {**ln.args, **ins, **outs[name]}) for name in libs}
        for name in libs:
            for _ in range(3):
                fns[name]()
        torch.cuda.synchronize()
        ts = {name: [] for name in libs}
        for _ in range(a.iters):  # alternate, so drifting clocks hit both libraries alike
            for name in libs:
                ts[name].append(event_ms(fns[name], a.reps))
        nbytes, flops = traffic(ln.args)
        row = dict(launch=ln.name, bytes=nbytes, flops=flops,
                   bound="bandwidth" if nbytes / HBM_PEAK >= flops / TENSOR_PEAK else "tensor")
        for name in libs:
            ms = sorted(ts[name])[a.iters // 2]
            row[name] = dict(ms=ms, tb_s=nbytes / (ms * 1e-3) / 1e12, tflops=flops / (ms * 1e-3) / 1e12,
                             share=max(nbytes / HBM_PEAK, flops / TENSOR_PEAK) / (ms * 1e-3))
        msg = "  ".join(f"{name} {row[name]['ms']:.3f} ms ({row[name]['tb_s']:.2f} TB/s, {row[name]['tflops']:.0f} TFLOP/s, "
                        f"{100 * row[name]['share']:.0f} % of the {row['bound']} bound)" for name in libs)
        if "old" in libs:
            row["max_abs_diff"] = max((outs["new"][k].float() - outs["old"][k].float()).abs().max().item()
                                      for k in outs["new"])
            row["speedup"] = row["old"]["ms"] / row["new"]["ms"]
            msg += f"  speed-up {row['speedup']:.2f}x  max |new - old| {row['max_abs_diff']:.3e}"
        print(f"{ln.name:<28} {nbytes / 1e6:8.1f} MB {flops / 1e9:8.1f} GFLOP  {msg}", flush=True)
        rows.append(row)
    result = dict(device=dev, fmt=a.fmt, batch=a.batch, iters=a.iters, reps=a.reps, launches=rows)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
