"""TEST INFRASTRUCTURE.  Writes the JPEG round-trip fixtures under tests/golden/ from the codec the reference calls
(JPEGDataset.jpeg_compress, data/datasets/restoration_jpeg.py:62-79: cv2.imencode(".jpg", [IMWRITE_JPEG_QUALITY, q]) +
cv2.imdecode, RGB <-> BGR around a colour image, one component for a gray one).  Runs wherever OpenCV is importable:

    python oracle/make_golden_jpeg.py            # validate + (re)write fixtures
    python oracle/make_golden_jpeg.py --check    # validate only

For every case it checks the integer restatement (oracle/jpeg_oracle.py) against the codec, half by half, and refuses
to write anything on a mismatch:
  - the quantisation tables parsed from the codec's bitstream (oracle/jpeg_bitstream.py) equal quant_tables(q);
  - the quantised coefficients parsed from the bitstream equal jpeg_oracle.encode;
  - jpeg_oracle.decode of the parsed coefficients equals the codec's decoded pixels;
  - jpeg_oracle.roundtrip equals the codec's round trip.

Fixtures: tests/golden/jpeg_cases.json (name -> channels, H, W, quality, content, seed), tests/golden/jpeg_gray.npz and
tests/golden/jpeg_color.npz (per case: <name>/input, <name>/output, <name>/qt (components, 64) natural order as parsed,
<name>/coef<k> (rows, cols, 8, 8) int16 per component as parsed) and tests/golden/jpeg_tables.npz (qt (100, 2, 64): the
luma / chroma tables parsed from a colour stream at every quality 1..100).
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import jpeg_bitstream  # noqa: E402
import jpeg_oracle as jo  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
QUALITIES = (1, 5, 10, 20, 30, 40, 50, 75, 90, 100)
# the sizes below 8 and around one MCU (9 x 3 and 6 x 4: chroma at most 2 samples wide, which the decoder upsamples by
# replication), then (16 + r, 16 + (7r + 3) % 16): every residue of H and of W mod 16
SIZES = [(1, 1), (3, 5), (7, 9), (9, 3), (6, 4), (16, 16), (17, 33), (31, 18), (100, 72)]
SIZES += [(16 + r, 16 + (7 * r + 3) % 16) for r in range(16)]


def cv2_encode(img, q):
    import cv2

    params = [int(cv2.IMWRITE_JPEG_QUALITY), int(q)]
    src = cv2.cvtColor(img, cv2.COLOR_RGB2BGR) if img.shape[2] == 3 else img
    ok, enc = cv2.imencode(".jpg", src, params)
    assert ok
    return enc


def cv2_decode(enc, C):
    import cv2

    if C == 3:
        return cv2.cvtColor(cv2.imdecode(enc, 1), cv2.COLOR_BGR2RGB)
    return cv2.imdecode(enc, 0)[..., None]


def codec_case(img, q):
    """The codec's view of one image: (round trip, parsed stream)."""
    enc = cv2_encode(img, q)
    return cv2_decode(enc, img.shape[2]), jpeg_bitstream.parse(enc.tobytes())


def check_case(img, q, out, parsed):
    """Every check of the module docstring; returns a list of failures (empty = exact)."""
    H, W, C = img.shape
    lq, cq = jo.quant_tables(q)
    qt = [parsed["qt"][c[3]] for c in parsed["components"]]
    fails = []
    if [(c[1], c[2]) for c in parsed["components"]] != ([(1, 1)] if C == 1 else [(2, 2), (1, 1), (1, 1)]):
        fails.append(f"sampling factors {parsed['components']}")
    if not all(np.array_equal(a, b) for a, b in zip(qt, [lq, cq, cq])):
        fails.append("quantisation tables")
    enc = jo.encode(img, q)
    if not all(np.array_equal(a, b) for a, b in zip(enc, parsed["coefs"])):
        fails.append("coefficients")
    if not np.array_equal(jo.decode(parsed["coefs"], qt, H, W), out):
        fails.append("decode of the parsed coefficients")
    if not np.array_equal(jo.roundtrip(img, q), out):
        fails.append("round trip")
    return fails


def cases():
    """name -> (C, H, W, q, content, seed)."""
    out, i = {}, 0
    for C in (1, 3):
        for H, W in SIZES:
            q, content = QUALITIES[i % len(QUALITIES)], jo.CONTENTS[i % len(jo.CONTENTS)]
            out[f"c{C}_{H}x{W}_q{q}_{content}"] = (C, H, W, q, content, 1000 + i)
            i += 1
        # the released checkpoints' quality on a test-set-like image of every content
        for content in jo.CONTENTS:
            out[f"c{C}_100x72_q10_{content}"] = (C, 100, 72, 10, content, 1000 + i)
            i += 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    table, arrays, bad = {}, {1: {}, 3: {}}, []
    for name, (C, H, W, q, content, seed) in cases().items():
        img = jo.synth_image(content, H, W, C, seed)
        out, parsed = codec_case(img, q)
        fails = check_case(img, q, out, parsed)
        print(f"{name}: {'exact' if not fails else 'MISMATCH ' + ', '.join(fails)}")
        bad += [(name, f) for f in fails]
        table[name] = {"channels": C, "H": H, "W": W, "quality": q, "content": content, "seed": seed}
        a = arrays[C]
        a[f"{name}/input"], a[f"{name}/output"] = img, out
        a[f"{name}/qt"] = np.stack([parsed["qt"][c[3]] for c in parsed["components"]]).astype(np.uint8)
        for k, coef in enumerate(parsed["coefs"]):
            a[f"{name}/coef{k}"] = coef.astype(np.int16)
    qt_all = np.zeros((100, 2, 64), np.uint8)
    probe = jo.synth_image("random", 16, 16, 3, 7)
    for q in range(1, 101):
        parsed = codec_case(probe, q)[1]
        tabs = [parsed["qt"][c[3]] for c in parsed["components"]]
        qt_all[q - 1] = np.stack(tabs[:2])
        if not all(np.array_equal(a, b) for a, b in zip(tabs[:2], jo.quant_tables(q))):
            bad.append((f"tables q={q}", "quantisation tables"))
    print(f"tables q = 1..100: {'exact' if not any(n.startswith('tables') for n, _ in bad) else 'MISMATCH'}")
    if bad:
        sys.exit(f"{len(bad)} mismatches: {bad[:10]}")
    if args.check:
        return
    with open(os.path.join(GOLD, "jpeg_cases.json"), "w") as f:
        json.dump(table, f, indent=1)
    np.savez_compressed(os.path.join(GOLD, "jpeg_gray.npz"), **arrays[1])
    np.savez_compressed(os.path.join(GOLD, "jpeg_color.npz"), **arrays[3])
    np.savez_compressed(os.path.join(GOLD, "jpeg_tables.npz"), qt=qt_all)
    print(f"wrote {len(table)} cases and the tables of q = 1..100 to {GOLD}")


if __name__ == "__main__":
    main()
