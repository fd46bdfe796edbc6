"""Dev tool: each attention launch of one cfg4 block (GRL-Base x4 SR, 256^2 tiles, B = 16) timed in isolation on cuda:0.

The launches are the ones BlockPlan.run issues (tc.attention_launches): window attention of a shifted (masked) and an
unshifted block, stripe pass 1 (anchors attend to the stripe's tokens) and stripe pass 2 (tokens attend to the anchors).
Operands are synthetic but laid out as in production: packed 32-wide head slots, L2-normalised q / k / anchors with the
logit scale on the query side, the ones column in V where head_dim < 32, 4-copy bias tables.

For each launch: CUDA-event time (median of --iters batches of --reps launches, after warm-up), score elements per second
against the ex2 (MUFU, 16 / clk / SM) bound at the card's maximum SM clock, and tensor FLOP/s of the padded d = 32
products (128 FLOP per score) against the dense fp16 / bf16 data-sheet peak (989 TFLOP/s).  The maximum clock gives the
highest bound, so the MUFU share is never overstated; the SM clock read right after the timed loop is printed beside it
(a power-capped card may have run slower).

--old LIB times a second build of libgrl_b200.so (for instance the parent commit's, built separately) on the same
operands, alternating with this tree's library batch by batch, and reports the largest |new - old| output difference.

    python tools/time_attention.py [--old path/to/libgrl_b200.so] [--fmt fp16|bf16] [--out result.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from _pkgload import load_package  # noqa: E402

MUFU_PER_CLK_SM = 16
FLOP_PER_SCORE = 4 * 32  # Q K^T and P V at the padded head dim
TENSOR_PEAK = 989e12  # dense fp16 / bf16, H100 SXM data sheet


def device_info():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_clock_mhz": None, "max_sm_clock_mhz": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        pl, clk, mx = q.stdout.strip().splitlines()[0].split(",")
        info["power_limit_w"], info["sm_clock_mhz"], info["max_sm_clock_mhz"] = float(pl), float(clk), float(mx)
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def event_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def load_lib(path, capi):
    handle = ctypes.CDLL(os.path.abspath(path))
    for name, (res, args) in capi._SIGNATURES.items():
        fn = getattr(handle, name)
        fn.restype, fn.argtypes = res, args
    if handle.grl_abi_version() != capi.ABI_VERSION:
        raise SystemExit(f"{path}: ABI version {handle.grl_abi_version()}, this tree has {capi.ABI_VERSION}")
    return handle


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old", default=None, help="a second libgrl_b200.so to time alternately on the same operands")
    ap.add_argument("--fmt", default="fp16", choices=("fp16", "bf16"))
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_attention.py needs a CUDA device")
    pkg = load_package()
    from grl_image_restoration_b200 import capi, tc

    libs = {"new": capi.lib()}
    if a.old:
        libs["old"] = load_lib(a.old, capi)

    def run_with(name, fn):
        saved, capi._lib = capi._lib, libs[name]
        try:
            fn()
        finally:
            capi._lib = saved

    cfg = pkg.configs.grl_config("base", "sr", 4, 256)
    model = pkg.GRL(**cfg)
    blocks = [m for m in model.modules() if hasattr(m, "window_shift") and hasattr(m, "attn")]
    masked = next(b for b in blocks if b.window_shift)
    plain = next(b for b in blocks if not b.window_shift)
    B, H, W = a.batch, 256, 256
    dt = torch.float16 if a.fmt == "fp16" else torch.bfloat16
    g = torch.Generator("cuda").manual_seed(0)
    scale = 14.0  # |logit| range in log2 units

    def slots(rows, n, heads_q, d, ones):
        """(rows, n * 32) 16-bit slots: unit vectors in the first d columns; the first heads_q slots carry the scale."""
        x = torch.zeros(rows, n, 32, device="cuda")
        x[..., :d] = F.normalize(torch.randn(rows, n, d, device="cuda", generator=g), dim=-1)
        x[:, :heads_q] *= scale
        if ones:
            x[..., 31] = 1.0
        return x.view(rows, n * 32).to(dt)

    cases = []
    for label, blk, roles in (("window (masked)", masked, ("window",)), ("window (unmasked)", plain, ("window",)),
                              ("stripe", masked, ("stripe1", "stripe2"))):
        launches = {ln.role: ln for ln in tc.attention_launches(blk, (H, W))}
        hw, hs = blk.attn.window_attn.num_heads, blk.attn.stripe_attn.num_heads
        c = blk.dim // 2
        anc = launches["stripe1"].gq
        La, nWs = anc.H * anc.W, (anc.H // anc.wh) * (anc.W // anc.ww)
        # window q | k | v, then stripe q | k | v; V slots carry the ones column where head_dim < 32
        qkv = torch.cat([slots(B * H * W, hw, hw, c // hw, False), slots(B * H * W, hw, 0, c // hw, False),
                         slots(B * H * W, hw, 0, c // hw, c // hw < 32), slots(B * H * W, hs, hs, c // hs, False),
                         slots(B * H * W, hs, 0, c // hs, False), slots(B * H * W, hs, 0, c // hs, c // hs < 32)], 1)
        bufs = {"qkv": qkv, "anchor": slots(B * La, hs, hs, c // hs, False)}
        for name in libs:
            bufs[f"merged:{name}"] = torch.zeros(B * H * W, tc.round_up((hw + hs) * 32, 64), device="cuda", dtype=dt)
            bufs[f"x1:{name}"] = torch.zeros(B * nWs * hs * anc.wh * anc.ww, 32, device="cuda", dtype=dt)
        for role in roles:
            ln = launches[role]
            if role == "window" and ln.use_mask != (blk is masked):
                raise SystemExit("unexpected mask flag on the window launch")
            rows = (ln.gq.wh + ln.gk.wh - 1) * (ln.gq.ww + ln.gk.ww - 1)
            table = torch.rand(ln.heads, rows, device="cuda", generator=g) * 16 * tc.LOG2E
            nW = (ln.gq.H // ln.gq.wh) * (ln.gq.W // ln.gq.ww)
            elems = B * nW * ln.heads * (ln.gq.wh * ln.gq.ww) * (ln.gk.wh * ln.gk.ww)
            cases.append(dict(label=f"{label} {role}", ln=ln, bias=tc.shifted_copies(table), bufs=bufs, elems=elems))

    def launch(case, name):
        ln, bufs = case["ln"], case["bufs"]

        def buf(ref, reading):
            key = ref[0]
            if key in ("merged", "x1"):
                # pass 2 reads the X1 that this tree's pass 1 wrote, so both libraries see identical operands
                key = f"{key}:{'new' if reading else name}"
            return bufs[key], ref[1]

        (q, qo), (k, ko), (v, vo), (o, oo) = buf(ln.q, True), buf(ln.k, True), buf(ln.v, True), buf(ln.out, False)
        return lambda: run_with(name, lambda: tc.attention(ln.gq, ln.gk, q, qo, k, ko, v, vo, o, oo, B, ln.heads,
                                                           case["bias"], ln.use_mask, v_dense=ln.v_dense,
                                                           o_dense=ln.o_dense, ones_col=ln.ones_col))

    dev = device_info()
    print(f"device: {dev['name']}, power limit {dev['power_limit_w']} W, max SM clock {dev['max_sm_clock_mhz']} MHz, "
          f"{a.fmt} operands, B = {B}", flush=True)
    mclk = dev["max_sm_clock_mhz"]
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    rows = []
    for case in cases:
        fns = {name: launch(case, name) for name in libs}
        for name in libs:  # the outputs compared are those of one launch on the shared operands
            for _ in range(3):
                fns[name]()
        torch.cuda.synchronize()
        ts = {name: [] for name in libs}
        for _ in range(a.iters):  # alternate, so drifting clocks hit both libraries alike
            for name in libs:
                ts[name].append(event_ms(fns[name], a.reps))
        clk = device_info()["sm_clock_mhz"]
        row = dict(launch=case["label"], score_elems=case["elems"], sm_clock_after_mhz=clk, max_sm_clock_mhz=mclk)
        for name in libs:
            ms = sorted(ts[name])[a.iters // 2]
            rate = case["elems"] / (ms * 1e-3)
            row[name] = dict(ms=ms, min_ms=min(ts[name]), score_elems_per_s=rate,
                             mufu_share=rate / (MUFU_PER_CLK_SM * nsm * mclk * 1e6) if mclk else None,
                             tflops=rate * FLOP_PER_SCORE / 1e12, tensor_share=rate * FLOP_PER_SCORE / TENSOR_PEAK)
        out = case["ln"].out
        if "old" in libs:
            o_new, o_old = case["bufs"][f"{out[0]}:new"], case["bufs"][f"{out[0]}:old"]
            row["max_abs_diff"] = (o_new.float() - o_old.float()).abs().max().item()
            row["speedup"] = row["old"]["ms"] / row["new"]["ms"]
        rows.append(row)
        msg = "  ".join(f"{name} {row[name]['ms']:.3f} ms ({row[name]['score_elems_per_s'] / 1e9:.0f} G/s = "
                        f"{100 * (row[name]['mufu_share'] or 0):.0f} % MUFU, {row[name]['tflops']:.0f} TFLOP/s = "
                        f"{100 * row[name]['tensor_share']:.1f} % tensor)" for name in libs)
        if "old" in libs:
            msg += f"  speed-up {row['speedup']:.2f}x  max |new - old| {row['max_abs_diff']:.3e}"
        print(f"{case['label']:<28} {msg}  [SM clock after the loop {clk} MHz]", flush=True)
    result = dict(device=dev, fmt=a.fmt, batch=B, iters=a.iters, reps=a.reps, launches=rows)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
