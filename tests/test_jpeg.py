"""CPU tests of the JPEG round trip (the JPEG test command's degraded input): the integer restatement
(oracle/jpeg_oracle.py) and the library's host expansion of csrc/grl_jpeg.h, exact against the codec's bytes stored in
tests/golden/jpeg_* (written by oracle/make_golden_jpeg.py from cv2), and live against cv2 where it is importable."""
import json
import os

import numpy as np
import pytest
import torch

import jpeg_bitstream
import jpeg_oracle as jo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

with open(os.path.join(GOLD, "jpeg_cases.json")) as f:
    CASES = json.load(f)
_NPZ = {C: np.load(os.path.join(GOLD, f"jpeg_{'gray' if C == 1 else 'color'}.npz")) for C in (1, 3)}


def case(name):
    c = CASES[name]
    z = _NPZ[c["channels"]]
    ncomp = 1 if c["channels"] == 1 else 3
    return (c, z[f"{name}/input"], z[f"{name}/output"], z[f"{name}/qt"].astype(np.int64),
            [z[f"{name}/coef{k}"].astype(np.int64) for k in range(ncomp)])


def test_fixture_coverage():
    """The stored cases span gray and colour, every quality of the list, every residue of H and W mod 16 and sizes
    below one block."""
    for C in (1, 3):
        cs = [c for c in CASES.values() if c["channels"] == C]
        assert {c["quality"] for c in cs} >= {1, 5, 10, 20, 30, 40, 50, 75, 90, 100}
        assert {c["H"] % 16 for c in cs} == set(range(16)) and {c["W"] % 16 for c in cs} == set(range(16))
        assert {c["content"] for c in cs} == set(jo.CONTENTS)
        assert any(c["H"] < 8 and c["W"] < 8 for c in cs)


def test_oracle_tables_equal_parsed_tables_every_quality():
    qt = np.load(os.path.join(GOLD, "jpeg_tables.npz"))["qt"].astype(np.int64)
    for q in range(1, 101):
        lq, cq = jo.quant_tables(q)
        assert np.array_equal(lq, qt[q - 1, 0]) and np.array_equal(cq, qt[q - 1, 1]), q


def test_library_tables_equal_parsed_tables_every_quality(pkg):
    qt = np.load(os.path.join(GOLD, "jpeg_tables.npz"))["qt"].astype(np.int64)
    for q in range(1, 101):
        assert np.array_equal(pkg.jpeg_quant_tables(q).numpy(), qt[q - 1]), q


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_encoder_half(name):
    """Tables and quantised coefficients of every coded block, as parsed from the codec's bitstream."""
    c, img, _, qt, coefs = case(name)
    lq, cq = jo.quant_tables(c["quality"])
    assert all(np.array_equal(a, b) for a, b in zip(qt, [lq, cq, cq]))
    enc = jo.encode(img, c["quality"])
    assert len(enc) == len(coefs)
    for k, (a, b) in enumerate(zip(enc, coefs)):
        assert a.shape == b.shape and np.array_equal(a, b), (name, k, int((a != b).sum()))


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_decoder_half(name):
    """The codec's pixels from the parsed coefficients alone."""
    c, img, out, qt, coefs = case(name)
    assert np.array_equal(jo.decode(coefs, list(qt), c["H"], c["W"]), out)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_and_library_roundtrip(name, pkg):
    c, img, out, _, _ = case(name)
    assert np.array_equal(jo.roundtrip(img, c["quality"]), out)
    got = pkg.jpeg_roundtrip_host(torch.from_numpy(img), c["quality"]).numpy()
    assert got.shape == out.shape and np.array_equal(got, out), (name, int((got != out).sum()))


def test_bitstream_parser_refuses_progressive():
    cv2 = pytest.importorskip("cv2")
    img = jo.synth_image("random", 16, 16, 3, 0)
    ok, enc = cv2.imencode(".jpg", img, [int(cv2.IMWRITE_JPEG_QUALITY), 50, int(cv2.IMWRITE_JPEG_PROGRESSIVE), 1])
    assert ok
    with pytest.raises(ValueError, match="not baseline"):
        jpeg_bitstream.parse(enc.tobytes())


def test_host_refusals(pkg):
    img = torch.zeros(8, 8, 3, dtype=torch.uint8)
    for q in (0, 101, 10.0, True, "10"):
        with pytest.raises(ValueError):
            pkg.jpeg_roundtrip_host(img, q)
        with pytest.raises(ValueError):
            pkg.jpeg_quant_tables(q)
    with pytest.raises(ValueError):
        pkg.jpeg_roundtrip_host(torch.zeros(8, 8, 2, dtype=torch.uint8), 10)
    with pytest.raises(ValueError):
        pkg.jpeg_roundtrip_host(img.float(), 10)


def test_c_entry_point_refusals(pkg):
    """The device entry point validates its whole list before anything launches (no device is needed to be refused)."""
    from grl_image_restoration_b200 import capi

    lib = capi.lib()

    def refs(*specs):
        arr = (capi.GrlImageRef * max(1, len(specs)))()
        for r, (data, h, w, kind) in zip(arr, specs):
            r.data, r.H, r.W, r.kind = data, h, w, kind
        return arr

    good = refs((16, 8, 8, capi.IMAGE_U8))
    assert lib.grl_jpeg_workspace(good, 1, 3) == 64 + 2 * 16 and lib.grl_jpeg_workspace(good, 1, 1) == 0
    bad = [
        (good, good, 1, 2, 10, "C = 2"),
        (good, good, 1, 3, 0, "quality 0"),
        (good, good, 1, 3, 101, "quality 101"),
        (refs((16, 8, 8, capi.IMAGE_F32)), good, 1, 1, 10, "kinds"),
        (refs((0, 8, 8, capi.IMAGE_U8)), good, 1, 1, 10, "null data"),
        (good, refs((16, 8, 9, capi.IMAGE_U8)), 1, 1, 10, "sizes"),
        (refs((16, 0, 8, capi.IMAGE_U8)), refs((16, 0, 8, capi.IMAGE_U8)), 1, 1, 10, "sizes"),
    ]
    for s, d, n, C, q, msg in bad:
        assert lib.grl_jpeg_roundtrip_u8(s, d, n, C, q, None, 0, None) == -1
        assert msg in lib.grl_last_error().decode()
    assert lib.grl_jpeg_roundtrip_u8(good, good, 1, 3, 10, None, 0, None) == -1  # null workspace
    assert lib.grl_jpeg_roundtrip_u8(good, good, 1, 3, 10, 16, 95, None) == -3  # workspace too small


@pytest.mark.parametrize("C", [1, 3])
def test_live_against_cv2(C, pkg):
    """Fresh seeded images, compared with the codec itself where OpenCV is importable."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2024 + C)
    for i in range(12):
        H, W = (int(v) for v in rng.integers(1, 70, 2))
        q = int(rng.integers(1, 101))
        img = jo.synth_image(jo.CONTENTS[i % len(jo.CONTENTS)], H, W, C, int(rng.integers(1 << 30)))
        params = [int(cv2.IMWRITE_JPEG_QUALITY), q]
        if C == 3:
            enc = cv2.imencode(".jpg", cv2.cvtColor(img, cv2.COLOR_RGB2BGR), params)[1]
            want = cv2.cvtColor(cv2.imdecode(enc, 1), cv2.COLOR_BGR2RGB)
        else:
            enc = cv2.imencode(".jpg", img, params)[1]
            want = cv2.imdecode(enc, 0)[..., None]
        got = pkg.jpeg_roundtrip_host(torch.from_numpy(img), q).numpy()
        assert np.array_equal(got, want), (H, W, C, q)
        assert np.array_equal(jo.roundtrip(img, q), want), (H, W, C, q)
