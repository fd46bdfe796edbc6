"""NIQE on the device (csrc/niqe.cu + metrics.niqe_distance) stage by stage against the NumPy oracle on the kernels' own
inputs, end to end against the unmodified reference (tests/golden/niqe_*.npz), and mutation controls that must fail
the score gate of tests/test_niqe.py."""
import os

import numpy as np
import pytest
import torch

import niqe_oracle
from test_niqe import ALPHA_COLS, CASES, GOLD, SCORE_GATE, params

pytestmark = pytest.mark.gpu
ULP255 = 255 * 2.0 ** -23  # one fp32 ulp at the top of the 8-bit range


def golden(case):
    return np.load(os.path.join(GOLD, f"niqe_{case}.npz"))


def as_input(rgb8, device):
    return torch.from_numpy(rgb8.astype(np.float32) / np.float32(255.0)).to(device)


@pytest.fixture(scope="module")
def tab():
    return niqe_oracle.tables()


@pytest.mark.parametrize("case", CASES)
def test_stages_against_oracle(pkg, device, tab, case):
    from grl_image_restoration_b200 import metrics

    g, prm = golden(case), params()
    win = prm["gaussian_window"]
    s = {k: v.cpu().numpy() for k, v in metrics.niqe_stages(as_input(g["rgb8"], device), prm, int(g["border"])).items()}
    for i in range(g["rgb8"].shape[0]):
        assert np.array_equal(s["y"][i], g["y"][i].astype(np.float32)), "luma must be bit-exact"
        for key, src, bs in (("mscn1", s["y"][i], 96), ("mscn2", s["half"][i], 48)):
            want = niqe_oracle.mscn(src, win)
            diff = s[key][i] != want
            # the 49-tap float64 sums run in scipy's order on both sides; allow isolated 1-ulp differences only
            assert diff.mean() <= 1e-4, (key, int(diff.sum()))
            assert np.all(np.abs(s[key][i][diff] - want[diff]) <= np.spacing(np.abs(want[diff]).astype(np.float32)))
            blk, wb = niqe_oracle.blocks(s[key][i], bs), niqe_oracle.blocks(want, bs)
            flat = (wb == 0).reshape(len(wb), -1).all(1)  # a constant region with its halo
            assert case != "flat" or flat.any()
            assert np.all(blk[flat] == 0), "a flat block needs an MSCN of exactly 0"
        want_half = niqe_oracle.half(s["y"][i])
        # float64 sums of 8 taps stored to fp32 twice, then x255: within 2 ulp of 255 of the oracle's identical sums
        assert np.abs(s["half"][i] - want_half).max() <= 2 * ULP255
        f1, m1 = niqe_oracle.features(s["mscn1"][i], 96, tab)
        f2, m2 = niqe_oracle.features(s["mscn2"][i], 48, tab)
        want, margin = np.concatenate([f1, f2], 1), np.concatenate([m1, m2], 1)
        got = s["feats"][i]
        assert np.array_equal(np.isnan(got), np.isnan(want))
        # float64 moments of <= 9216 terms in another order: |relative error of rhatnorm| << 1e-9
        sure = margin > 1e-9 * (1 + np.abs(np.nan_to_num(want[:, ALPHA_COLS])))
        assert np.array_equal(got[:, ALPHA_COLS][sure], want[:, ALPHA_COLS][sure])
        rows = (got[:, ALPHA_COLS] == want[:, ALPHA_COLS]).all(1)
        assert rows.mean() >= 0.95
        assert np.nanmax(np.abs(got[rows] - want[rows]) / (np.abs(want[rows]) + 1e-6)) <= 1e-9


@pytest.mark.parametrize("case", CASES)
def test_score_matches_reference(pkg, device, case):
    from grl_image_restoration_b200 import metrics

    g = golden(case)
    x = as_input(g["rgb8"], device)
    keep = x.clone()
    got = metrics.niqe(x, os.path.join(GOLD, "niqe_pris_params.npz"), border=int(g["border"]))
    assert torch.equal(x, keep), "niqe must not modify its input"
    assert got.dtype == torch.float64 and got.shape == (x.shape[0],)
    err = (got.cpu() - torch.from_numpy(g["score"])).abs().max().item()
    print(f"niqe {case}: device {got.cpu().tolist()} reference {g['score'].tolist()} |diff| {err:.2e}")
    assert err <= SCORE_GATE
    again = metrics.niqe(x, params(), border=int(g["border"]))
    assert torch.equal(got, again), "two runs must be bit-identical"


def test_batch_equals_single_images(pkg, device):
    from grl_image_restoration_b200 import metrics

    g, prm = golden("b2"), params()
    x = as_input(g["rgb8"], device)
    fb = metrics.niqe_features(x, prm, 4)
    for i in range(x.shape[0]):
        assert torch.equal(fb[i:i + 1], metrics.niqe_features(x[i:i + 1].contiguous(), prm, 4))
    sb = metrics.niqe(x, prm, 4)
    singles = torch.cat([metrics.niqe(x[i:i + 1].contiguous(), prm, 4) for i in range(x.shape[0])])
    assert torch.allclose(sb, singles, rtol=0, atol=1e-10)


@pytest.mark.parametrize("hw", [(1024, 1024), (1356, 2040)])
def test_realistic_size_against_oracle(pkg, device, tab, hw):
    from grl_image_restoration_b200 import metrics

    h, w = hw
    rng = np.random.default_rng(h + w)
    yy, xx = np.mgrid[0:h, 0:w] / max(h, w)
    base = np.stack([np.sin(9 * xx + 4 * yy), np.cos(7 * yy - 5 * xx), np.sin(6 * (xx + yy))]) * 70 + 128
    rgb8 = np.clip(base + rng.normal(0, 10, (3, h, w)), 0, 255).round().astype(np.uint8)
    prm = params()
    got = metrics.niqe(as_input(rgb8[None], device), prm).item()
    want = niqe_oracle.niqe(rgb8, prm, 0, tab)["score"]
    print(f"niqe {h}x{w}: device {got:.6f} oracle {want:.6f} |diff| {abs(got - want):.2e}")
    assert abs(got - want) <= SCORE_GATE


def _score_from(feats_rows, prm):
    return niqe_oracle.distance(feats_rows, prm["mu_pris_param"], prm["cov_pris_param"])


def test_mutations_fail_the_gate(pkg, device, tab):
    """Each deliberate change, applied to the device's own intermediate images, moves some golden's score past the gate."""
    from grl_image_restoration_b200 import metrics

    prm = params()
    win = prm["gaussian_window"]
    worst = {"rgb_luma": 0.0, "float64_mscn": 0.0, "no_roll_wrap": 0.0}
    for case in CASES:
        g = golden(case)
        b = int(g["border"])
        s = {k: v.cpu().numpy() for k, v in metrics.niqe_stages(as_input(g["rgb8"], device), prm, b).items()}
        for i, want in enumerate(g["score"]):
            # RGB (MATLAB) luma instead of the reference's BGR weights
            y = niqe_oracle.crop(metrics.rgb_to_y(torch.from_numpy(g["rgb8"][i:i + 1].astype(np.float32) / 255.0))[0, 0]
                                 .mul(255).round().numpy(), b)
            f = np.concatenate([niqe_oracle.features(niqe_oracle.mscn(y, win), 96, tab)[0],
                                niqe_oracle.features(niqe_oracle.mscn(niqe_oracle.half(y), win), 48, tab)[0]], 1)
            worst["rgb_luma"] = max(worst["rgb_luma"], abs(_score_from(f, prm) - want))

            # MSCN in float64
            def mscn64(x):
                x = x.astype(np.float64)
                p = np.pad(x, 3, mode="edge")
                conv = lambda z: sum(np.pad(z, 3, mode="edge")[i2:i2 + z.shape[0], j:j + z.shape[1]] * win[6 - i2, 6 - j]
                                     for i2 in range(7) for j in range(7))
                del p
                mu = conv(x)
                return (x - mu) / (np.sqrt(np.abs(conv(x * x) - mu * mu)) + 1)

            f = np.concatenate([niqe_oracle.features(mscn64(s["y"][i]), 96, tab)[0],
                                niqe_oracle.features(mscn64(s["half"][i]), 48, tab)[0]], 1)
            worst["float64_mscn"] = max(worst["float64_mscn"], abs(_score_from(f, prm) - want))
            # products of neighbours without the wrap at the block edge
            rows = []
            for m, bs in ((s["mscn1"][i], 96), (s["mscn2"][i], 48)):
                blk = niqe_oracle.blocks(m, bs)
                n = len(blk)
                fr = np.empty((n, 18))
                idx, ls, rs, _ = niqe_oracle.aggd(blk.reshape(n, -1), tab)
                fr[:, 0], fr[:, 1] = tab[0][idx], (ls * tab[2][idx] + rs * tab[2][idx]) / 2
                for k, (a, c) in enumerate(niqe_oracle.SHIFTS):
                    sh = np.roll(blk, (a, c), axis=(1, 2))
                    prod = blk * sh
                    prod = prod[:, a:, 1:] if c == 1 else (prod[:, a:, :-1] if c == -1 else prod[:, a:, :])
                    idx, ls, rs, _ = niqe_oracle.aggd(prod.reshape(n, -1), tab)
                    bl, br = ls * tab[2][idx], rs * tab[2][idx]
                    fr[:, 2 + 4 * k:6 + 4 * k] = np.stack([tab[0][idx], (br - bl) * tab[3][idx], bl, br], 1)
                rows.append(fr)
            worst["no_roll_wrap"] = max(worst["no_roll_wrap"], abs(_score_from(np.concatenate(rows, 1), prm) - want))
    print("mutation worst |score - reference|:", worst)
    for name, v in worst.items():
        assert v > SCORE_GATE, f"mutation {name} passes the gate"
