"""CPU tests of the seeded AWGN (the denoising test command's noisy input): the library's host copy of csrc/grl_awgn.h
bit for bit against numpy's RandomState in float64, dn_seed against the reference's key, the goldens written from the
reference's DnDataset (oracle/make_golden_awgn.py) reproduced exactly, the device's double-double log correctly rounded,
each plausible mistake shown to be caught, and the C entry points' refusals."""
import hashlib
import json
import math
import os
from fractions import Fraction

import numpy as np
import pytest
import torch

from engine_oracle import to_tensor

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

with open(os.path.join(GOLD, "awgn_cases.json")) as f:
    CASES = json.load(f)
_NPZ = np.load(os.path.join(GOLD, "awgn.npz"))

NAMES = ["CBSD68/0001.png", "Urban100/img_004.png", "McMaster/18.tif", "Set12/07.png"]
COUNTS = [0, 1, 2, 3, 311, 312, 313, 623, 624, 625, 10 ** 5 + 3]


def case(name):
    c = CASES[name]
    return c, _NPZ[f"{name}/input"], torch.from_numpy(_NPZ[f"{name}/gt"]), torch.from_numpy(_NPZ[f"{name}/lq"])


def crop8(img):
    return img[: img.shape[0] // 8 * 8, : img.shape[1] // 8 * 8]


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("sigma", [0, 2.5, 15, 25, 50])
def test_noise_host_equals_numpy(name, sigma, pkg):
    key = pkg.dn_seed(name)
    for count in COUNTS:
        want = np.random.RandomState(key).normal(0, sigma / 255, count)
        got = pkg.awgn_noise_host(name, count, sigma)
        assert got.dtype == torch.float64 and got.shape == (count,)
        assert np.array_equal(got.numpy(), want), (name, sigma, count)
        assert torch.equal(pkg.awgn_noise_host(list(key), count, sigma), got)


def test_dn_seed(pkg):
    for name in NAMES + ["", "a_b_c", "Urban100/img_100.png"]:
        want = np.frombuffer(hashlib.sha256(name.split("_")[0].encode("utf-8")).digest(), dtype="uint32")
        got = pkg.dn_seed(name)
        assert got.dtype == np.uint32 and got.shape == (8,) and np.array_equal(got, want), name
    # the reference keys on the path up to its first "_": every Urban100 image shares one stream
    assert np.array_equal(pkg.dn_seed("Urban100/img_004.png"), pkg.dn_seed("Urban100/img_092.png"))
    assert np.array_equal(pkg.dn_seed("Urban100/img_004.png"), pkg.dn_seed("Urban100/img"))
    assert not np.array_equal(pkg.dn_seed("CBSD68/0001.png"), pkg.dn_seed("CBSD68/0002.png"))
    with pytest.raises(ValueError):
        pkg.dn_seed(b"CBSD68/0001.png")


def test_golden_coverage():
    cs = list(CASES.values())
    assert {c["channels"] for c in cs} == {1, 3} and {c["sigma"] for c in cs} == {15, 25, 50}
    assert any(c["H"] == 1 and c["W"] == 1 for c in cs)
    assert any(c["H"] % 8 and c["W"] % 8 for c in cs)
    urban = [c for c in cs if c["key"].startswith("Urban100/") and c["channels"] == 3]
    assert len({c["key"] for c in urban}) >= 2 and len({c["key"].split("_")[0] for c in urban}) == 1


@pytest.mark.parametrize("name", sorted(CASES))
def test_goldens_reproduce(name, pkg):
    """The dataset's img_gt and img_lq from the host noise, the float32 to_tensor and the float32 add."""
    c, img, gt, lq = case(name)
    g8 = crop8(img)
    assert torch.equal(to_tensor(g8), gt)
    noise = pkg.awgn_noise_host(c["key"], gt.numel(), c["sigma"]).float().reshape(gt.shape)
    assert torch.equal(gt + noise, lq), name


def test_urban_goldens_share_one_stream(pkg):
    """Two Urban100 images of different sizes: the reference drew the smaller one's noise as the prefix of the larger
    one's stream."""
    (ca, _, ga, la), (cb, _, gb, lb) = case("c3_urban_30x41_s15"), case("c3_urban_26x37_s15")
    assert ca["key"] != cb["key"] and gb.numel() < ga.numel()
    stream = pkg.awgn_noise_host(ca["key"], ga.numel(), ca["sigma"]).float()
    assert torch.equal(ga + stream.reshape(ga.shape), la)
    assert torch.equal(gb + stream[: gb.numel()].reshape(gb.shape), lb)


def test_device_log_is_correctly_rounded(pkg):
    """awgn_log_cr, the device's log, on the CPU: equal to log correctly rounded (decimal, 50 digits) on random r2 in
    (0, 1), r2 just below 1, tiny r2, the reduction's boundaries and the r2 of real candidates."""
    from decimal import Decimal, getcontext

    from grl_image_restoration_b200 import functional as F

    getcontext().prec = 50
    rng = np.random.default_rng(5)
    xs = [rng.random(4000), 1 - rng.random(500) * 2.0 ** -30, rng.random(500) * 2.0 ** -60,
          np.array([0.5, 0.25, 2.0 ** -104, 1 - 2.0 ** -53, 0.7071067811865475, 0.7071067811865476, 0.7071067811865477])]
    # r2 of the polar candidates of one stream
    rs = np.random.RandomState(pkg.dn_seed("CBSD68/0001.png"))
    u = rs.random_sample(4000) * 2 - 1
    xs.append((u[0::2] * u[0::2] + u[1::2] * u[1::2]))
    x = np.concatenate(xs)
    x = x[(x > 0) & (x < 1)]
    got = F.awgn_log_host(torch.from_numpy(x)).numpy()
    bad = [v for v, g in zip(x, got) if g != float(Decimal(float(v)).ln())]
    assert not bad, bad[:5]
    # where the host libm's log is correctly rounded (nearly everywhere), the host copy's log agrees with the device's
    agree = sum(math.log(v) == g for v, g in zip(x, got))
    assert agree >= 0.99 * len(x)


# ---- each plausible mistake is caught ---------------------------------------------------------------------------------
def _words(key):
    """The tempered MT19937 words of RandomState(key), from its seeded state (a pure-Python restatement)."""
    mt = [int(v) for v in np.random.RandomState(key).get_state()[1]]
    while True:
        for i in range(624):
            y = (mt[i] & 0x80000000) | (mt[(i + 1) % 624] & 0x7FFFFFFF)
            mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ (0x9908B0DF if y & 1 else 0)
        for y in mt:
            y ^= y >> 11
            y ^= (y << 7) & 0x9D2C5680
            y ^= (y << 15) & 0xEFC60000
            yield y ^ (y >> 18)


def _gauss(key, count, mistake=None):
    w = _words(key)

    def unit():
        return ((next(w) >> 5) * 67108864.0 + (next(w) >> 6)) / 9007199254740992.0

    out = []
    while len(out) < count:
        if mistake == "trig":
            u1, u2 = unit(), unit()
            if u1 == 0.0:
                continue
            r = math.sqrt(-2.0 * math.log(u1))
            out += [r * math.cos(2 * math.pi * u2), r * math.sin(2 * math.pi * u2)]
            continue
        x1, x2 = 2.0 * unit() - 1.0, 2.0 * unit() - 1.0
        if mistake == "fma":  # fma(x1, x1, x2 * x2)
            r2 = float(Fraction(x1) * Fraction(x1) + Fraction(x2 * x2))
        else:
            r2 = x1 * x1 + x2 * x2
        if r2 >= 1.0 or r2 == 0.0:
            continue
        f = math.sqrt(-2.0 * math.log(r2) / r2)
        out += [f * x1, f * x2] if mistake == "swap" else [f * x2, f * x1]
    return np.array(out[:count])


@pytest.mark.parametrize("mistake", [None, "swap", "trig", "fma"])
def test_float64_mistakes_are_caught(mistake, pkg):
    """The restatement matches numpy (the control); each mistake in it is visible in float64 noise, which
    test_noise_host_equals_numpy compares bit for bit."""
    key = pkg.dn_seed("CBSD68/0001.png")
    want = np.random.RandomState(key).normal(0, 15 / 255, 2000)
    got = 0.0 + 15 / 255 * _gauss(key, 2000, mistake)
    assert np.array_equal(got, want) == (mistake is None), mistake


@pytest.mark.parametrize("mistake", ["scale_f32", "stream_per_channel", "whole_name"])
def test_image_mistakes_are_caught(mistake):
    """Each mistake in how the noise meets the image gives an img_lq other than the reference's golden."""
    c, img, gt, lq = case("c3_urban_30x41_s15")
    scale, key = c["sigma"] / 255, c["key"].split("_")[0]
    seed = np.frombuffer(hashlib.sha256(key.encode("utf-8")).digest(), dtype="uint32")
    if mistake == "scale_f32":
        g = np.random.RandomState(seed).normal(0, 1, gt.shape)
        noise = torch.from_numpy(g).float() * torch.tensor(scale, dtype=torch.float32)
    elif mistake == "stream_per_channel":
        noise = torch.stack([torch.from_numpy(np.random.RandomState(seed).normal(0, scale, gt.shape[1:])).float()
                             for _ in range(gt.shape[0])])
    else:
        whole = np.frombuffer(hashlib.sha256(c["key"].encode("utf-8")).digest(), dtype="uint32")
        noise = torch.from_numpy(np.random.RandomState(whole).normal(0, scale, gt.shape)).float()
    control = gt + torch.from_numpy(np.random.RandomState(seed).normal(0, scale, gt.shape)).float()
    assert torch.equal(control, lq)
    assert not torch.equal(gt + noise, lq), mistake


# ---- refusals -----------------------------------------------------------------------------------------------------------
def test_host_refusals(pkg):
    for sigma in (-1, float("nan"), float("inf"), True, "15", None):
        with pytest.raises(ValueError):
            pkg.awgn_noise_host("CBSD68/0001.png", 4, sigma)
    for seed in ([1] * 7, [1] * 9, [-1] + [0] * 7, [2 ** 32] + [0] * 7, [0.5] * 8, b"x", 3):
        with pytest.raises(ValueError):
            pkg.awgn_noise_host(seed, 4, 15)
    for count in (-1, 2.0, True):
        with pytest.raises(ValueError):
            pkg.awgn_noise_host("CBSD68/0001.png", count, 15)
    assert pkg.awgn_noise_host(np.arange(8, dtype=np.uint32), 0, 15).shape == (0,)


def test_c_entry_point_refusals(pkg):
    """The device entry point validates its whole list before anything launches (no device is needed to be refused)."""
    import ctypes

    from grl_image_restoration_b200 import capi

    lib = capi.lib()

    def refs(*specs):
        arr = (capi.GrlImageRef * max(1, len(specs)))()
        for r, (data, h, w, kind) in zip(arr, specs):
            r.data, r.H, r.W, r.kind = data, h, w, kind
        return arr

    keys = np.zeros((2, 8), np.uint32)
    kp = keys.ctypes.data_as(ctypes.c_void_p)
    src, dst = refs((16, 8, 8, capi.IMAGE_U8)), refs((32, 8, 8, capi.IMAGE_F32))
    bad = [
        (src, dst, kp, 1, 2, 0.1, "C = 2"),
        (src, dst, kp, 1, 3, -0.1, "scale"),
        (src, dst, kp, 1, 3, float("nan"), "scale"),
        (src, dst, kp, 1, 3, float("inf"), "scale"),
        (src, dst, kp, -1, 3, 0.1, "n = -1"),
        (src, dst, None, 1, 3, 0.1, "null"),
        (dst, dst, kp, 1, 3, 0.1, "kinds"),
        (src, src, kp, 1, 3, 0.1, "kinds"),
        (refs((0, 8, 8, capi.IMAGE_U8)), dst, kp, 1, 3, 0.1, "null data"),
        (src, refs((32, 8, 9, capi.IMAGE_F32)), kp, 1, 3, 0.1, "sizes"),
        (refs((16, 0, 8, capi.IMAGE_U8)), refs((32, 0, 8, capi.IMAGE_F32)), kp, 1, 3, 0.1, "sizes"),
        (refs((16, 40000, 40000, capi.IMAGE_U8)), refs((32, 40000, 40000, capi.IMAGE_F32)), kp, 1, 3, 0.1, "too large"),
    ]
    for s, d, k, n, C, scale, msg in bad:
        assert lib.grl_awgn_u8(s, d, k, n, C, scale, None) == -1, msg
        assert msg in lib.grl_last_error().decode(), (msg, lib.grl_last_error())
    assert lib.grl_awgn_u8(None, None, None, 0, 3, 0.1, None) == 0  # an empty list launches nothing
    out = np.zeros(4)
    assert lib.grl_awgn_noise_host(kp, 4, -1.0, out.ctypes.data_as(ctypes.c_void_p)) == -1
    assert lib.grl_awgn_noise_host(None, 4, 0.1, out.ctypes.data_as(ctypes.c_void_p)) == -1
    assert lib.grl_awgn_noise_host(kp, -1, 0.1, out.ctypes.data_as(ctypes.c_void_p)) == -1
    x = np.array([0.5, 0.0])
    assert lib.grl_awgn_log_host(x.ctypes.data_as(ctypes.c_void_p), 2, out.ctypes.data_as(ctypes.c_void_p)) == -1
