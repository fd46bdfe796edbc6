"""NIQE of the blind-SR test command, host side: the luma closed form against the NumPy chain on every 8-bit triple,
the resize taps and gamma tables, and the NumPy oracle (oracle/niqe_oracle.py) against the unmodified reference
(tests/golden/niqe_*.npz from oracle/make_golden_niqe.py).

Score gate: |score - reference| <= 2e-3 (the engine prints 4 decimals).  The oracle differs from the reference by at most
6.8e-4 on these goldens (flat case); the differences come from the reference's fp32 means and its fp32 resize sums,
which flip an alpha where a fit lies within about 1e-6 of a decision midpoint of the r_gam table."""
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["smooth", "flat", "b2"]
SCORE_GATE = 2e-3
ALPHA_COLS = [0, 2, 6, 10, 14, 18, 20, 24, 28, 32]


def params():
    return dict(np.load(os.path.join(GOLD, "niqe_pris_params.npz")))


def numpy_luma_chain(rgb8):
    """calculate_niqe's chain (niqe.py:143-156, :75-111, :529-542) on tensor_round'ed data, with NumPy's own dot over a
    3-D (H, W, 3) array as in the reference."""
    p = rgb8.astype(np.float32) / np.float32(255.0)
    img = (p * 255).astype(np.float32)
    img = img.astype(np.float32) / 255.0
    y = np.dot(img, [24.966, 128.553, 65.481]) + 16.0
    y = (y / 255.0).astype(np.float32)
    return (y * 255.0).round()


def test_luma_host_equals_numpy_chain_on_all_triples(pkg):
    import ctypes

    from grl_image_restoration_b200 import capi

    k = np.arange(256, dtype=np.uint8)
    rgb = np.empty((256, 256, 256, 3), np.uint8)
    rgb[..., 0], rgb[..., 1], rgb[..., 2] = k[:, None, None], k[None, :, None], k[None, None, :]
    got = np.empty((256, 256, 256), np.float32)
    capi.check(capi.lib().grl_niqe_luma_host(ctypes.c_void_p(rgb.ctypes.data), rgb.shape[0] * 65536,
                                             ctypes.c_void_p(got.ctypes.data)))
    for r in range(256):
        assert np.array_equal(got[r], numpy_luma_chain(rgb[r])), r
    # BGR weights on RGB data: pure red and pure blue swap relative to MATLAB's luma
    assert got[255, 0, 0] == 41.0 and got[0, 0, 255] == 81.0


def test_half_taps_match_reference_weights(pkg):
    import ctypes

    import niqe_oracle
    from grl_image_restoration_b200 import capi

    w = np.empty(8, np.float32)
    capi.check(capi.lib().grl_niqe_half_taps_host(ctypes.c_void_p(w.ctypes.data)))
    for case in CASES:
        ref = np.load(os.path.join(GOLD, f"niqe_{case}.npz"))["weights"]
        assert ref.shape[1] == 8
        assert np.array_equal(ref, np.broadcast_to(w, ref.shape))  # every output row uses the same taps, bit for bit
    assert np.array_equal(w, niqe_oracle.HALF_TAPS)


def test_gamma_tables_match_numpy_and_scipy(pkg):
    from scipy.special import gamma

    from grl_image_restoration_b200 import metrics

    t = metrics.niqe_tables().numpy()
    gam = np.arange(0.2, 10.001, 0.001)
    assert t.shape == (4, 9801) and np.array_equal(t[0], gam)
    rec = np.reciprocal(gam)
    r_gam = np.square(gamma(rec * 2)) / (gamma(rec) * gamma(rec * 3))
    assert np.abs(t[1] / r_gam - 1).max() <= 1e-13
    assert np.abs(t[2] / np.sqrt(gamma(1 / gam) / gamma(3 / gam)) - 1).max() <= 1e-13
    assert np.abs(t[3] / (gamma(2 / gam) / gamma(1 / gam)) - 1).max() <= 1e-13
    assert np.all(np.diff(t[1]) > 0), "r_gam is increasing: the argmin has one decision midpoint per neighbour"


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_reference(pkg, case):
    import niqe_oracle

    g = np.load(os.path.join(GOLD, f"niqe_{case}.npz"))
    prm, tab = params(), niqe_oracle.tables()
    for i, img in enumerate(g["rgb8"]):
        r = niqe_oracle.niqe(img, prm, int(g["border"]), tab)
        assert np.array_equal(r["y"], g["y"][i].astype(np.float32))
        # two fp32 passes of 8 taps over values <= 1, times 255: the reference's fp32 sums differ by a few ulp of 255
        assert np.abs(r["half"] - g["half"][i]).max() <= 8 * 255 * 2.0 ** -24 * 1.25
        f, want = r["feats"], g["feats"][i]
        assert np.array_equal(np.isnan(f), np.isnan(want))
        agree = (f[:, ALPHA_COLS] == want[:, ALPHA_COLS])
        assert agree.mean() >= 0.98
        rows = agree.all(1)
        rel = np.abs(f[rows] - want[rows]) / (np.abs(want[rows]) + 1e-2)
        assert np.nanmax(rel) <= 5e-3
        assert abs(r["score"] - g["score"][i]) <= SCORE_GATE, (r["score"], g["score"][i])


def test_flat_golden_has_nan_blocks_and_float64_misses_it(pkg):
    """The flat-patch golden exercises the NaN path: constant 96 x 96 regions give an MSCN of exactly 0 in fp32, so a
    fit has no negative values, alpha 0.2 and NaN moments.  The same pipeline in float64 scores far off."""
    import niqe_oracle

    g = np.load(os.path.join(GOLD, "niqe_flat.npz"))
    prm = params()
    want = g["feats"][0]
    nan_rows = np.isnan(want).any(1)
    assert nan_rows.sum() >= 4
    assert np.all(want[nan_rows][:, ALPHA_COLS[:5]] == 0.2)
    y = g["y"][0].astype(np.float64)
    win = prm["gaussian_window"]

    def conv(x):
        p = np.pad(x, 3, mode="edge")
        return sum(p[i:i + x.shape[0], j:j + x.shape[1]] * win[6 - i, 6 - j] for i in range(7) for j in range(7))

    def mscn64(x):
        mu = conv(x)
        return (x - mu) / (np.sqrt(np.abs(conv(x * x) - mu * mu)) + 1)

    tab = niqe_oracle.tables()
    f1, _ = niqe_oracle.features(mscn64(y), 96, tab)
    f2, _ = niqe_oracle.features(mscn64(niqe_oracle.half(g["y"][0].astype(np.float32)).astype(np.float64)), 48, tab)
    s64 = niqe_oracle.distance(np.concatenate([f1, f2], 1), prm["mu_pris_param"], prm["cov_pris_param"])
    assert abs(s64 - g["score"][0]) > 100 * SCORE_GATE


def test_niqe_params_and_malformed_inputs(pkg, tmp_path):
    import ctypes

    from grl_image_restoration_b200 import capi, metrics

    prm = params()
    path = os.path.join(GOLD, "niqe_pris_params.npz")
    for a, b in zip(metrics.niqe_params(path), metrics.niqe_params(prm)):
        assert torch.equal(a, b)
    with pytest.raises(RuntimeError, match="shape"):
        metrics.niqe_params(dict(prm, gaussian_window=np.ones((5, 5))))
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.niqe(torch.rand(1, 3, 128, 128), prm)
    L, dummy = capi.lib(), ctypes.c_void_p(16)
    assert L.grl_niqe_luma_f32(dummy, 1, 1, 128, 128, 0, dummy, None) == -1
    assert b"C == 3" in L.grl_last_error()
    assert L.grl_niqe_luma_f32(dummy, 1, 3, 100, 128, 4, dummy, None) == -1
    assert b"96 x 96" in L.grl_last_error()
    assert L.grl_niqe_workspace(1, 100, 128, 4) == 0
    assert L.grl_niqe_workspace(2, 200, 200, 4) > 0
    win = (ctypes.c_double * 49)()
    assert L.grl_niqe_features_f32(dummy, 1, 3, 200, 200, 4, win, dummy, dummy, 0, dummy, None) == -1
    assert b"workspace" in L.grl_last_error()
