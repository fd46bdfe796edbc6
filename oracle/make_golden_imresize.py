"""TEST INFRASTRUCTURE.  Writes the bicubic-downscale fixtures under tests/golden/ from the reference's own functions,
utils/matlab_functions.py's calculate_weights_indices (:20-88) and imresize (:92-188), the SR dataset's online LR
(data/datasets/restoration_sr.py:127-141):

    python oracle/make_golden_imresize.py            # validate + (re)write fixtures
    python oracle/make_golden_imresize.py --check    # validate, and compare with the committed fixtures

Tables: for s in {2, 3, 4} and every side n in 1 .. 130 and 510, 1356, 2040, the reference's weight row, tap count, first
input index, pad lengths and output size, whether every output row has the same weights and indices s o + c + k, and
whether imresize fails on a side of that length (its symmetric copy needs both pads <= n, or n = 1, which it
broadcasts).  Outputs: imresize of seeded
float32 and 8-bit images (8-bit ones as img / 255.0, as the dataset calls it), RGB and gray, sides that are and are not
multiples of s, the smallest sides the reference accepts (1, and 4, 6, 7 for s = 2, 3, 4), and extreme values in the outer rows and columns so that a
padding mistake shows.

Every case is checked before anything is written: the tables against oracle/imresize_oracle.py's exact weights and
geometry, each output within oracle.reference_bound of the float64 oracle.

Fixtures: tests/golden/imresize_cases.json (tables and case list) and tests/golden/imresize.npz (per scale
taps<s> (T,) float32, the reference's weight row; per case <name>/input ((H, W, C) uint8 or (C, H, W) float32) and
<name>/output (C, h, w) float32).
"""
import argparse
import importlib.util
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import _ref_import  # noqa: E402
import imresize_oracle as oracle  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
LENGTHS = list(range(1, 131)) + [510, 1356, 2040]


def _matlab_functions():
    path = os.path.join(_ref_import.REF_ROOT, "utils", "matlab_functions.py")
    spec = importlib.util.spec_from_file_location("ref_matlab_functions", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _cases():
    """name -> (kind, C, H, W, s, seed)."""
    out = {}
    for s in oracle.SCALES:
        mn = {2: 4, 3: 6, 4: 7}[s]
        out[f"s{s}_u8_c3_24x36"] = ("u8", 3, 24, 36, s, 10 + s)
        out[f"s{s}_u8_c3_37x29"] = ("u8", 3, 37, 29, s, 20 + s)
        out[f"s{s}_u8_c1_31x22"] = ("u8", 1, 31, 22, s, 30 + s)
        out[f"s{s}_f32_c3_19x26"] = ("f32", 3, 19, 26, s, 40 + s)
        out[f"s{s}_f32_c1_33x41"] = ("f32", 1, 33, 41, s, 50 + s)
        out[f"s{s}_u8_c3_min{mn}x{mn}"] = ("u8", 3, mn, mn, s, 60 + s)
        out[f"s{s}_f32_c1_min{mn}x17"] = ("f32", 1, mn, 17, s, 70 + s)
        out[f"s{s}_u8_c1_1x9"] = ("u8", 1, 1, 9, s, 80 + s)
        out[f"s{s}_f32_c3_1x1"] = ("f32", 3, 1, 1, s, 90 + s)
    return out


def synth(kind, C, H, W, seed):
    """Seeded content with the outer two rows and columns at extreme, alternating values."""
    rng = np.random.default_rng(seed)
    if kind == "u8":
        img = rng.integers(0, 256, (H, W, C), dtype=np.uint8)
        img[:, 0], img[:, -1] = 0, 255
        if H > 2:
            img[0], img[-1], img[1, ::2], img[-2, 1::2] = 255, 0, 0, 255
        return img
    img = rng.random((C, H, W), dtype=np.float32)
    img[:, 0], img[:, -1], img[:, :, 0], img[:, :, -1] = 1.0, -0.25, 0.0, 1.25
    return img


def ref_input(kind, img):
    """The float32 (C, H, W) tensor imresize works on: img / 255.0 in float64 cast by imresize's .float()."""
    if kind == "u8":
        return torch.from_numpy((img / 255.0).transpose(2, 0, 1)).float()
    return torch.from_numpy(img)


def tables(mf):
    rows, taps, bad = {}, {}, []
    for s in oracle.SCALES:
        w_exact, c_exact = oracle.weights(s)
        for n in LENGTHS:
            out = -(-n // s)
            w, idx, ps, pe = mf.calculate_weights_indices(n, out, 1 / s, "cubic", 4, True)
            first = idx[:, 0].long() - ps  # 0-based first input of each output
            c = int(first[0])
            uniform = bool((w == w[0]).all()) and bool((first - s * torch.arange(out) == c).all()) and \
                bool((idx - idx[:, :1] == torch.arange(w.shape[1])).all())
            try:
                mf.imresize(torch.zeros(1, n, 8), 1 / s)
                fails = False
            except RuntimeError:
                fails = True
            rows[f"{s}/{n}"] = {"T": int(w.shape[1]), "c": c, "out": out, "pad_s": ps, "pad_e": pe, "uniform": uniform,
                                "fails": fails}
            want_ps, want_pe = oracle.pads(n, s)
            if not uniform or w.shape[1] != len(w_exact) or c != c_exact or (ps, pe) != (want_ps, want_pe) or \
                    fails != (n > 1 and (ps > n or pe > n)):
                bad.append(f"table s={s} n={n}")
            taps.setdefault(s, w[0].numpy().copy())
            if not np.array_equal(taps[s], w[0].numpy()):
                bad.append(f"taps s={s} n={n} differ from n={LENGTHS[0]}")
    return rows, taps, bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    mf = _matlab_functions()
    rows, taps, bad = tables(mf)
    arrays = {f"taps{s}": t for s, t in taps.items()}
    cases = _cases()
    for name, (kind, C, H, W, s, seed) in cases.items():
        img = synth(kind, C, H, W, seed)
        x = ref_input(kind, img)
        y = mf.imresize(x, 1 / s)
        want = oracle.resize(x.double().numpy(), s)
        err, bound = np.abs(y.double().numpy() - want), oracle.reference_bound(x.double().numpy(), s, taps[s])
        ratio = float(np.max(err / np.maximum(bound, np.finfo(np.float64).tiny)))
        ok = y.dtype == torch.float32 and tuple(y.shape) == (C, -(-H // s), -(-W // s)) and bool((err <= bound).all())
        print(f"{name}: {tuple(y.shape)} error / bound {ratio:.3f} {'ok' if ok else 'MISMATCH'}")
        if not ok:
            bad.append(name)
        arrays[f"{name}/input"] = img
        arrays[f"{name}/output"] = y.numpy()
    if bad:
        sys.exit(f"{len(bad)} mismatches: {bad[:20]}")
    meta = {"lengths": LENGTHS, "tables": rows,
            "cases": {k: dict(zip(("kind", "C", "H", "W", "s", "seed"), v)) for k, v in cases.items()}}
    if args.check:
        with open(os.path.join(GOLD, "imresize_cases.json")) as f:
            same = json.load(f) == meta
        old = np.load(os.path.join(GOLD, "imresize.npz"))
        same = same and set(old.files) == set(arrays) and all(np.array_equal(old[k], v) for k, v in arrays.items())
        if not same:
            sys.exit("the committed fixtures differ from what the reference computes")
        print("committed fixtures reproduced")
        return
    with open(os.path.join(GOLD, "imresize_cases.json"), "w") as f:
        json.dump(meta, f, indent=1)
    np.savez_compressed(os.path.join(GOLD, "imresize.npz"), **arrays)
    print(f"wrote {len(cases)} cases and {len(rows)} table rows to {GOLD}")


if __name__ == "__main__":
    main()
