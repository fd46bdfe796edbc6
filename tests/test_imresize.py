"""CPU tests of the bicubic downscale (MATLAB's imresize with antialiasing at 1/2, 1/3, 1/4; csrc/grl_resize.h): the host
taps and geometry against the reference's calculate_weights_indices, the host copy and the reference's own outputs
within derived bounds of the float64 oracle (oracle/imresize_oracle.py), each plausible mistake shown to break the bound,
and the refusals of the C entry points and of evaluate(synthesize_lr=True).

The bounds.  Let v be the float32 input (exact in float64), w the exact taps (rationals rounded once to float64 by the
oracle), u = 2^-24, T = 4s the tap count, and P = sum_j sum_i |w_j| |w_i| |v_ij| the resize of |v| with |w|
(oracle.abs_resize), where i runs over the H pass's taps and j over the W pass's.

Host copy.  Its taps are w_k (1 + a_k), |a_k| <= u (one float32 rounding of a double value whose own error is a few
2^-53, folded into g below).  A pass sums the exact products w_k v_k in float64, an error factor (1 + t), |t| <= g, and
rounds once to float32, (1 + d), |d| <= u.  So t_o = sum_i w_i v_i (1 + e_i) with |e_i| <= (1 + u)^2 (1 + g) - 1, and
the W pass on t gives sum_j sum_i w_j w_i v_ij (1 + e_ij) with |e_ij| <= (1 + u)^4 (1 + g)^2 - 1.  The oracle's own
float64 evaluation adds at most another (1 + g)^2, g = gamma_{2T+2} = (2T + 2) 2^-53 / (1 - (2T + 2) 2^-53):
    |host - oracle| <= ((1 + u)^4 (1 + g)^4 - 1) P                                      (oracle.host_bound)
about 4u P: the tap roundings and the one rounding per pass.

Reference.  Its taps w_r differ from w by eps_k = |w_r,k - w_k| (below 2^-23, checked here), and each float32 mv, whatever
its summation order, is within gamma_T = T u / (1 - T u) of the exact sum relative to sum |w_r| |v|.  Two passes:
    |ref - sum w_r w_r v| <= ((1 + gamma_T)^2 - 1) P_r,   P_r = P with |w_r|,
and sum (w_r,i w_r,j - w_i w_j) v = sum (w_r,i (w_r,j - w_j) + (w_r,i - w_i) w_j) v is at most E = the resize of |v| with
(|w_r|, eps) plus that with (eps, |w|).  With the oracle's (1 + g)^2:
    |ref - oracle| <= ((1 + gamma_T)^2 (1 + g)^2 - 1) P_r + (1 + g)^2 E                 (oracle.reference_bound)

The mutation controls must exceed the host bound on the fixtures: a wrong pad, tap set, centre or input scale moves an
output by a visible fraction of the content, against about 2.4e-7 P.  With the 1 / s factor, the exact tap rows of these
integer downscales already sum to 1, so normalisation only shows when that factor is also left out; the unnormalised
control drops both."""
import json
import os

import numpy as np
import pytest
import torch

import imresize_oracle as oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(GOLD, "imresize_cases.json")) as f:
    META = json.load(f)
_NPZ = np.load(os.path.join(GOLD, "imresize.npz"))
CASES = META["cases"]


def fixture(name):
    """(float32 (C, H, W) input as the reference resizes it, the reference's output, s)."""
    c = CASES[name]
    img = _NPZ[f"{name}/input"]
    x = torch.from_numpy((img / 255.0).transpose(2, 0, 1)).float() if c["kind"] == "u8" else torch.from_numpy(img)
    return x, torch.from_numpy(_NPZ[f"{name}/output"]), c["s"]


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def test_fixture_coverage():
    cs = list(CASES.values())
    assert {c["s"] for c in cs} == set(oracle.SCALES) and {c["C"] for c in cs} == {1, 3}
    assert {c["kind"] for c in cs} == {"u8", "f32"}
    for s in oracle.SCALES:
        mine = [c for c in cs if c["s"] == s]
        assert any(c["H"] % s == 0 and c["W"] % s == 0 for c in mine) and any(c["H"] % s and c["W"] % s for c in mine)
        assert any(c["H"] == 1 for c in mine) and any(c["H"] == {2: 4, 3: 6, 4: 7}[s] for c in mine)
    assert set(META["lengths"]) >= set(range(1, 131)) | {510, 1356, 2040}
    assert os.path.getsize(os.path.join(GOLD, "imresize.npz")) < 1 << 20


@pytest.mark.parametrize("s", oracle.SCALES)
def test_host_geometry_against_the_reference(s, pkg):
    """Tap count, first input, output size and pad lengths equal the reference's for every fixture length, every output
    row of the reference uses one weight row and inputs s o + c + k, and the host refuses exactly the lengths where the
    reference's imresize fails."""
    from grl_image_restoration_b200 import functional as F

    fails = []
    for n in META["lengths"]:
        row = META["tables"][f"{s}/{n}"]
        assert row["uniform"], (s, n)
        if row["fails"]:
            fails.append(n)
            with pytest.raises(RuntimeError, match="too small"):
                F.imresize_taps(n, 1 / s)
            with pytest.raises(RuntimeError, match="too small"):
                F.imresize_host(torch.zeros(1, 1, n, 8), 1 / s)
            continue
        _, g = F.imresize_taps(n, 1 / s)
        assert g == {k: row[k] for k in ("T", "c", "out", "pad_s", "pad_e")}, (s, n, g, row)
        assert F.imresize_host(torch.zeros(1, 1, n, 8), 1 / s).shape == (1, 1, row["out"], -(-8 // s))
    assert fails == list(range(2, {2: 4, 3: 6, 4: 7}[s])), (s, fails)


@pytest.mark.parametrize("s", oracle.SCALES)
def test_host_taps(s, pkg):
    """The host taps are the exact taps correctly rounded to float32; against the reference's float32 taps they are equal
    bit for bit for s = 2 and 4 (dyadic weights).  For s = 3 the reference evaluates the cubic on float32 products with
    1/3: its taps are within 1 ulp for |w| >= 1/9, its three zero taps are exactly 0, and the two small outer taps (-1/81,
    -2/81) are off by tens of ulps, within 2^-23 (one ulp of their sum, 1) absolutely."""
    from grl_image_restoration_b200 import functional as F

    taps, g = F.imresize_taps(64, 1 / s)
    exact, c = oracle.weights(s)
    assert g["T"] == len(exact) == 4 * s and g["c"] == c
    assert np.array_equal(taps.numpy(), exact.astype(np.float32))
    ref = _NPZ[f"taps{s}"]
    assert ref.dtype == np.float32 and ref.shape == taps.shape
    if s in (2, 4):
        assert np.array_equal(ref, taps.numpy())
        return
    d = np.abs(ref.astype(np.float64) - taps.numpy())
    big = np.abs(exact) >= 1 / 9 - 1e-12
    assert (d[big] <= ulp32(taps.numpy()[big])).all(), d
    assert np.array_equal(ref == 0, exact == 0) and int((exact == 0).sum()) == 3
    assert (d <= 2.0 ** -23).all() and d.max() > 0, d


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_and_reference_within_their_bounds(name, pkg):
    from grl_image_restoration_b200 import functional as F

    x, ref, s = fixture(name)
    want = oracle.resize(x.double().numpy(), s)
    host = F.imresize_host(x[None], 1 / s)[0]
    assert host.shape == ref.shape and host.dtype == torch.float32
    hb = oracle.host_bound(x.double().numpy(), s)
    assert (np.abs(host.double().numpy() - want) <= hb).all(), name
    rb = oracle.reference_bound(x.double().numpy(), s, _NPZ[f"taps{s}"])
    assert (np.abs(ref.double().numpy() - want) <= rb).all(), name


def _mutants(kind):
    m = {
        "edge padding": dict(pad="edge"),
        "no antialiasing": dict(antialias=False),
        "unnormalised": dict(normalise=False, prefactor=False),
        "window shifted by one": dict(shift=1),
        "centre without (1 - s) / 2": dict(centre=False),
    }
    if kind == "u8":
        m["255 for k / 255"] = "x255"
    return m


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c["H"] > 1 and c["W"] > 1))
def test_mutation_controls_break_the_bound(name):
    x, _, s = fixture(name)
    v = x.double().numpy()
    want = oracle.resize(v, s)
    hb = oracle.host_bound(v, s)
    for label, kw in _mutants(CASES[name]["kind"]).items():
        got = oracle.resize(v * 255, s) if kw == "x255" else oracle.resize(v, s, **kw)
        assert got.shape == want.shape, label
        assert (np.abs(got - want) > hb).any(), (name, label)


def test_scale_argument(pkg):
    from grl_image_restoration_b200 import functional as F

    for s in oracle.SCALES:
        assert F._resize_factor(1 / s) == s
    for bad in (1, 2, 0.5 + 1e-9, 1 / 5, 1 / 1.5, 0.3333, 0.0, -0.5, float("nan"), float("inf"), True, "0.5", None):
        with pytest.raises(ValueError, match="1/2, 1/3 and 1/4"):
            F._resize_factor(bad)


def test_c_entry_refusals(pkg):
    """Bad arguments are refused before anything is launched; null device pointers are never dereferenced."""
    import ctypes

    from grl_image_restoration_b200 import capi, functional as F

    L = capi.lib()
    for s in (0, 1, 5, -2):
        assert L.grl_imresize_f32(None, 1, 3, 64, 64, s, None, None) != 0
        assert b"scale" in L.grl_last_error()
    for C in (0, 9):
        assert L.grl_imresize_f32(None, 1, C, 64, 64, 2, None, None) != 0
    assert L.grl_imresize_f32(None, 1, 3, 64, 64, 2, None, None) != 0 and b"null" in L.grl_last_error()
    for H, W in ((3, 64), (64, 2), (5, 64), (0, 64)):
        assert L.grl_imresize_f32(ctypes.c_void_p(16), 1, 3, H, W, 3, ctypes.c_void_p(16), None) != 0
        assert b"too small" in L.grl_last_error()
    assert L.grl_imresize_f32(None, 0, 3, 64, 64, 2, None, None) == 0  # an empty batch launches nothing
    geom = (ctypes.c_int32 * 5)()
    taps = (ctypes.c_float * 16)()
    assert L.grl_imresize_taps_host(64, 6, taps, geom) != 0
    assert L.grl_imresize_taps_host(64, 2, None, geom) != 0

    def refs(items, kind):
        r = (capi.GrlImageRef * len(items))()
        for x, (data, H, W) in zip(r, items):
            x.data, x.H, x.W, x.kind = data, H, W, kind
        return r

    src = refs([(16, 40, 30)], capi.IMAGE_U8)
    assert L.grl_imresize_u8_list(src, refs([(16, 20, 15)], capi.IMAGE_F32), 1, 2, 2, None) != 0  # C = 2
    assert L.grl_imresize_u8_list(src, refs([(16, 20, 15)], capi.IMAGE_F32), 1, 3, 7, None) != 0  # scale
    assert L.grl_imresize_u8_list(None, None, 1, 3, 2, None) != 0
    assert L.grl_imresize_u8_list(src, refs([(16, 20, 15)], capi.IMAGE_U8), 1, 3, 2, None) != 0  # kind
    assert L.grl_imresize_u8_list(src, refs([(None, 20, 15)], capi.IMAGE_F32), 1, 3, 2, None) != 0
    assert L.grl_imresize_u8_list(src, refs([(16, 20, 16)], capi.IMAGE_F32), 1, 3, 2, None) != 0  # output size
    assert b"need 20 x 15" in L.grl_last_error()
    assert L.grl_imresize_u8_list(refs([(16, 40, 3)], capi.IMAGE_U8), refs([(16, 20, 2)], capi.IMAGE_F32), 1, 3, 2,
                                  None) != 0
    assert b"too small" in L.grl_last_error()
    with pytest.raises(ValueError):
        F.imresize_taps(64, 2)


def test_evaluate_synthesize_lr_refusals(pkg):
    """synthesize_lr=True belongs to the SR recipes and replaces lqs; both mistakes are refused before any image is read
    (the images here are CPU tensors, which a run would refuse later)."""
    gts = [torch.zeros(16, 16, 3, dtype=torch.uint8)]
    for name in ("dn_grl_base_c3s15.ckpt", "jpeg_grl_small_c3q10.ckpt", "dm_grl_small.ckpt", "bsr_grl_base.ckpt",
                 "db_motion_grl_base_gopro.ckpt"):
        with pytest.raises(ValueError, match="synthesize_lr"):
            pkg.evaluate(None, name, gts, synthesize_lr=True)
    with pytest.raises(ValueError, match="synthesize_lr"):
        pkg.evaluate(None, "sr_grl_tiny_c3x2.ckpt", gts, lqs=gts, synthesize_lr=True)
    from grl_image_restoration_b200 import evaluation

    with pytest.raises(ValueError, match="synthesize_lr"):
        evaluation.model_inputs("sr_grl_base_c3x4.ckpt", gts, lqs=gts, synthesize_lr=True)
