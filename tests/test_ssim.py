"""The SSIM closed form of csrc/grl_ssim.h, through its host entry points grl_ssim_taps_host and grl_ssim_host, against
values produced by the reference's own ssim (tests/golden/ssim.npz, written by oracle/make_golden_ssim.py) and against the
float64 restatement oracle/ssim_oracle.py in both forms: the reference's 2-D float32 window and the kernel's separable one.

SSIM_SCORE_GATE (metric_cases.py) is the distance allowed between a score of this project and the reference's.  The
reference convolves and sums in fp32.  Measured on the goldens (RGB / luma): flat 5.0e-7 / 4.6e-6, letterbox 4.5e-6 /
4.9e-6, sr_b2 8.1e-6 / 9.5e-6, gray 8.1e-6, tiny 7.4e-8 / 1.9e-8, clamp 3.0e-6 / 7.3e-6.  The float64 oracle with the
reference's own 2-D float32 window lies within 2.7e-7 of the host computation on every one of them and as far from the
reference as the host computation does, so the residue is the rounding of the reference's fp32 sums; the gate is twice
the worst of it.  The engine logs 4 decimals.
"""
import ctypes

import numpy as np
import pytest
import torch

import ssim_oracle
from metric_cases import SSIM_CASES, SSIM_GOLDEN, SSIM_SCORE_GATE, golden_pair, golden_scores, host_ssim


def grid8(img):
    """tensor_round as the kernels take it: the integers k = rint(clamp(x) * 255) in fp32, as float64."""
    v = np.clip(img.numpy().astype(np.float32), np.float32(0), np.float32(1))
    return np.rint(v * np.float32(255.0)).astype(np.float64)


def luma8(k, rounded=True):
    """metric.cu's luma8 on (B, 3, h, w) integers: an fp32 multiply and two fp32 fmas (exact in float64, then rounded once),
    + 16, rounded to the 8-bit grid."""
    c = [np.float32(v) / np.float32(255.0) for v in (65.481, 128.553, 24.966)]
    acc = (k[:, 0] * np.float64(c[0])).astype(np.float32)
    acc = (k[:, 1] * np.float64(c[1]) + acc.astype(np.float64)).astype(np.float32)
    acc = (k[:, 2] * np.float64(c[2]) + acc.astype(np.float64)).astype(np.float32)
    y = (acc + np.float32(16.0)).astype(np.float64)
    return (np.rint(y) if rounded else y)[:, None]


def planes(restored, target, border, luma=False, rounded_luma=True):
    """The two float64 (B, C', h, w) planes k / 255 the metric is taken on."""
    ka, kb = grid8(restored), grid8(target)
    if border:
        ka, kb = ka[..., border:-border, border:-border], kb[..., border:-border, border:-border]
    if luma and ka.shape[1] == 3:
        ka, kb = luma8(ka, rounded_luma), luma8(kb, rounded_luma)
    return ka / 255.0, kb / 255.0


def oracle_scores(restored, target, border, **kw):
    return (ssim_oracle.ssim(*planes(restored, target, border), **kw),
            ssim_oracle.ssim(*planes(restored, target, border, luma=True), **kw))


def test_taps_equal_the_reference_window(pkg):
    from grl_image_restoration_b200 import capi

    t = np.zeros(11)
    capi.check(capi.lib().grl_ssim_taps_host(t.ctypes.data_as(ctypes.c_void_p)))
    want = np.load(SSIM_GOLDEN)["taps"]
    assert want.dtype == np.float64 and t.tobytes() == want.tobytes()  # gaussian(11, 1.5), bit for bit
    assert t.tobytes() == ssim_oracle.taps().tobytes()
    assert {"grl_ssim_f32", "grl_ssim_workspace", "grl_ssim_host", "grl_ssim_taps_host"} <= set(capi.header_symbols())


@pytest.mark.parametrize("case", SSIM_CASES)
def test_host_equals_the_separable_oracle(pkg, case):
    """Same taps, same separable order of summation, float64 on both sides: what is left is the fma chains against
    NumPy's multiply-adds, a few ulp per map value."""
    g = np.load(SSIM_GOLDEN)
    restored, target = golden_pair(g, case)
    border = int(g[f"{case}_border"])
    s, sy, m, my = host_ssim(restored, target, border, maps=True)
    want, want_y = oracle_scores(restored, target, border)
    assert np.abs(s - want).max() <= 1e-13 and np.abs(sy - want_y).max() <= 1e-13
    assert np.abs(m - ssim_oracle.ssim_map(*planes(restored, target, border))).max() <= 1e-11
    if restored.shape[1] == 3:
        assert np.abs(my - ssim_oracle.ssim_map(*planes(restored, target, border, luma=True))).max() <= 1e-11


def window_bound(a, b):
    """First-order bound on |score(separable) - score(2-D float32 window)| from the windows' difference alone.  Every
    weight of float32(t t^T) is within eps = 2^-24 (6e-8) relative of t_i t_j and the data are non-negative, so each
    windowed sum S moves by at most eps S; var = E[x^2] - mu^2 then moves by eps (E[x^2] + 2 mu^2), and likewise cov."""
    t = ssim_oracle.taps()
    w2 = np.outer(t, t)
    eps = float(np.abs(w2.astype(np.float32).astype(np.float64) / w2 - 1).max())
    assert 0 < eps <= 2.0**-24
    blur = lambda x: ssim_oracle._blur(x, t, "separable", "zero")  # noqa: E731
    mu_a, mu_b, e_aa, e_bb, e_ab = blur(a), blur(b), blur(a * a), blur(b * b), blur(a * b)
    c1, c2 = 1e-4, 9e-4
    n1, d1 = 2 * mu_a * mu_b + c1, mu_a**2 + mu_b**2 + c1
    n2, d2 = 2 * (e_ab - mu_a * mu_b) + c2, e_aa - mu_a**2 + e_bb - mu_b**2 + c2
    dn1, dd1 = eps * 4 * mu_a * mu_b, eps * 2 * (mu_a**2 + mu_b**2)
    dn2, dd2 = eps * 2 * (e_ab + 2 * mu_a * mu_b), eps * (e_aa + e_bb + 2 * mu_a**2 + 2 * mu_b**2)
    per_pixel = (dn1 * np.abs(n2) + np.abs(n1) * dn2) / (d1 * d2) + np.abs(n1 * n2) / (d1 * d2) * (dd1 / d1 + dd2 / d2)
    return 1.01 * per_pixel.mean((-3, -2, -1))  # 1 % for the second-order terms


@pytest.mark.parametrize("case", SSIM_CASES)
def test_host_against_the_2d_window_oracle(pkg, case):
    g = np.load(SSIM_GOLDEN)
    restored, target = golden_pair(g, case)
    border = int(g[f"{case}_border"])
    s, sy = host_ssim(restored, target, border)
    want, want_y = oracle_scores(restored, target, border, window="2d")
    bound = window_bound(*planes(restored, target, border))
    bound_y = window_bound(*planes(restored, target, border, luma=True))
    assert (np.abs(s - want) <= bound + 1e-13).all(), (np.abs(s - want), bound)
    assert (np.abs(sy - want_y) <= bound_y + 1e-13).all(), (np.abs(sy - want_y), bound_y)
    # measured: 2.7e-7 at worst (sr_b2, luma), far inside the worst-case bound (1e-4 on the flat case)
    assert max(np.abs(s - want).max(), np.abs(sy - want_y).max()) <= 5e-7


@pytest.mark.parametrize("case", SSIM_CASES)
def test_host_matches_the_reference(pkg, case):
    g = np.load(SSIM_GOLDEN)
    restored, target = golden_pair(g, case)
    border = int(g[f"{case}_border"])
    keep = restored.clone()
    s, sy = host_ssim(restored, target, border)
    assert torch.equal(restored, keep)
    want, want_y = golden_scores(g, case)
    assert np.abs(s - want).max() <= SSIM_SCORE_GATE, (s, want)
    assert np.abs(sy - want_y).max() <= SSIM_SCORE_GATE, (sy, want_y)
    if restored.shape[1] == 1:
        assert sy.tobytes() == s.tobytes()


def test_letterbox_map_is_exactly_one(pkg):
    """Where every pixel under the window is black in both images the five sums are exactly 0 and the map is C1 C2 / C1 C2:
    the 12 black rows at either end leave 7 rows whose 11-row window sees nothing else."""
    g = np.load(SSIM_GOLDEN)
    restored, target = golden_pair(g, "letterbox")
    border = int(g["letterbox_border"])
    assert not grid8(restored)[..., :12, :].any() and not grid8(target)[..., -12:, :].any()
    _, _, m, my = host_ssim(restored, target, border, maps=True)
    for mm in (m, my):
        assert (mm[..., :7, :] == 1.0).all() and (mm[..., -7:, :] == 1.0).all()
        assert (mm[..., 12:-12, :] != 1.0).any()


@pytest.mark.parametrize("shape", [(2, 3, 23, 31), (1, 1, 5, 3), (1, 3, 1, 1)])
def test_identical_images_score_exactly_one(pkg, shape):
    x = torch.rand(shape, generator=torch.Generator().manual_seed(3))
    s, sy, m, my = host_ssim(x, x.clone(), maps=True)
    assert (s == 1.0).all() and (sy == 1.0).all() and (m == 1.0).all()


def test_refusals(pkg):
    from grl_image_restoration_b200 import capi, metrics

    L = capi.lib()
    dummy = ctypes.c_void_p(16)
    assert L.grl_ssim_workspace(2, 3, 48, 56, 4) == 2 * 2 * 2 * 3 * 8  # 40 x 48 after the shave: 2 x 3 tiles of 32 x 16
    for entry in (lambda *a: L.grl_ssim_f32(dummy, dummy, *a, dummy, 1 << 20, dummy, dummy, None, None, None),
                  lambda *a: L.grl_ssim_host(dummy, dummy, *a, dummy, dummy, None, None)):
        assert entry(1, 3, 16, 40, 8) == -1 and b"border 8" in L.grl_last_error()  # 2 * border == min(H, W)
        assert entry(1, 2, 32, 32, 0) == -1 and b"C == 1 or 3" in L.grl_last_error()
        assert entry(1, 4, 32, 32, 0) == -1
        assert entry(1, 3, 32, 32, -1) == -1
    assert L.grl_ssim_workspace(1, 2, 32, 32, 0) == 0 and L.grl_ssim_workspace(1, 3, 16, 40, 8) == 0
    ws = L.grl_ssim_workspace(1, 3, 32, 32, 0)
    assert L.grl_ssim_f32(dummy, dummy, 1, 3, 32, 32, 0, dummy, ws - 8, dummy, dummy, None, None, None) == -1
    assert b"workspace" in L.grl_last_error()
    assert L.grl_ssim_f32(None, dummy, 1, 3, 32, 32, 0, dummy, ws, dummy, dummy, None, None, None) == -1
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.ssim_fused(torch.rand(1, 3, 32, 32), torch.rand(1, 3, 32, 32))
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.validation_metrics_fused(torch.rand(1, 3, 32, 32), torch.rand(1, 3, 32, 32))


# ------------------------------------------------------------------------------------------------ mutation controls
# Each changes one thing the definition fixes, in the oracle or in what the host computation is given.  Those listed in
# PINNED move some golden past the gate; the others are checked to stay inside it, so that the statement "the goldens
# do not pin this" is itself under test.
def mutated_scores(g, case, mutation):
    restored, target = golden_pair(g, case)
    border = int(g[f"{case}_border"])
    if mutation == "no_shave":
        return host_ssim(restored, target, 0)
    if mutation == "unrounded_luma":
        return (ssim_oracle.ssim(*planes(restored, target, border)),
                ssim_oracle.ssim(*planes(restored, target, border, luma=True, rounded_luma=False)))
    kw = {"reflect_padding": dict(pad="reflect"), "renormalised": dict(renormalise=True), "valid_only": dict(valid_only=True),
          "unrounded_taps": dict(rounded_taps=False), "constants_for_255": dict(c_scale=65025.0)}[mutation]
    return oracle_scores(restored, target, border, **kw)


def worst_distance(mutation):
    g, worst = np.load(SSIM_GOLDEN), 0.0
    for case in SSIM_CASES:
        if case == "tiny" and mutation in ("reflect_padding", "valid_only"):
            continue  # 7 x 9: no reflection of 5 pixels, no valid window
        if mutation == "no_shave" and not int(g[f"{case}_border"]):
            continue
        s, sy = mutated_scores(g, case, mutation)
        want, want_y = golden_scores(g, case)
        worst = max(worst, np.abs(s - want).max(), np.abs(sy - want_y).max())
    return worst


PINNED = ["reflect_padding", "renormalised", "valid_only", "unrounded_luma", "no_shave", "constants_for_255"]
NOT_PINNED = ["unrounded_taps"]


@pytest.mark.parametrize("mutation", PINNED)
def test_mutation_fails_the_gate(pkg, mutation):
    assert worst_distance(mutation) > SSIM_SCORE_GATE, f"mutation {mutation} passes the gate: the goldens do not pin it"


@pytest.mark.parametrize("mutation", NOT_PINNED)
def test_mutation_the_goldens_do_not_pin(pkg, mutation):
    """Taps kept at full precision instead of 6 decimals: 9.3e-6 from the goldens at worst, which is the reference's own
    fp32 residue and no more.  The taps are pinned bit for bit by test_taps_equal_the_reference_window instead."""
    assert worst_distance(mutation) <= SSIM_SCORE_GATE
