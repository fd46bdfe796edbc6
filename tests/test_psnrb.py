"""PSNR-B of the JPEG test commands (metrics.psnrb) against values produced by the reference's own psnrb
(tests/golden/psnrb.npz, written by oracle/make_golden_psnrb.py) and against a float64 restatement that counts nothing
for itself: the reference's normalisers are formulas of H and W, not counts of the summed positions."""
import math

import numpy as np
import pytest
import torch

from metric_cases import PSNRB_CASES, PSNRB_GOLDEN, golden_pair


def restated(restored, target, luma=False):
    """psnrb.py:22-115 written out per image in float64 on the 8-bit integers, with the loops the reference vectorises."""
    from grl_image_restoration_b200 import metrics

    a, b = metrics.tensor_round(restored), metrics.tensor_round(target)
    if luma:
        a, b = metrics.rgb_to_y(a), metrics.rgb_to_y(b)
    ka, kb = (a * 255).round().double().numpy(), (b * 255).round().double().numpy()
    out = []
    for i in range(ka.shape[0]):
        vals = []
        for c in range(ka.shape[1]):
            x, H, W = ka[i, c], ka.shape[2], ka.shape[3]
            bcols, brows = list(range(7, W - 1, 8)), list(range(7, H - 1, 8))
            hb = sum(((x[:, j] - x[:, j + 1]) ** 2).sum() for j in bcols)
            hn = sum(((x[:, j] - x[:, j + 1]) ** 2).sum() for j in range(W - 1) if j not in bcols)
            vb = sum(((x[j] - x[j + 1]) ** 2).sum() for j in brows)
            vn = sum(((x[j] - x[j + 1]) ** 2).sum() for j in range(H - 1) if j not in brows)
            nbh, nbv = H * (W // 8 - 1), W * (H // 8 - 1)
            bd, nd = (hb + vb) / (nbh + nbv), (hn + vn) / (H * (W - 1) - nbh + W * (H - 1) - nbv)
            bef = 0.0 if bd <= nd else math.log2(8) / math.log2(min(H, W)) * (bd - nd)
            mse = ((x - kb[i, c]) ** 2).mean()
            vals.append(10 * math.log10(65025.0 / (mse + bef)))
        out.append(sum(vals) / len(vals))
    return torch.tensor(out, dtype=torch.float64)


@pytest.mark.parametrize("case", PSNRB_CASES)
def test_psnrb_matches_reference(pkg, case):
    from grl_image_restoration_b200 import metrics

    g = np.load(PSNRB_GOLDEN)
    restored, target = golden_pair(g, case)
    keep = restored.clone()
    got = metrics.psnrb(restored, target)
    assert torch.equal(restored, keep)
    assert got.dtype == torch.float64 and got.shape == (restored.shape[0],)
    # the reference sums in fp32: 1e-4 dB covers its rounding
    assert (got - torch.from_numpy(g[f"{case}_psnrb"]).double()).abs().max().item() <= 1e-4
    if f"{case}_psnrb_y" in g:
        got_y = metrics.psnrb(restored, target, channel="y")
        assert (got_y - torch.from_numpy(g[f"{case}_psnrb_y"]).double()).abs().max().item() <= 1e-4


@pytest.mark.parametrize("case", PSNRB_CASES)
def test_psnrb_equals_float64_restatement(pkg, case):
    from grl_image_restoration_b200 import metrics

    restored, target = golden_pair(np.load(PSNRB_GOLDEN), case)
    assert (metrics.psnrb(restored, target) - restated(restored, target)).abs().max().item() <= 1e-9
    if restored.shape[1] == 3:
        assert (metrics.psnrb(restored, target, "y") - restated(restored, target, luma=True)).abs().max().item() <= 1e-9


def test_normaliser_is_the_formula_not_the_count(pkg):
    """W = 20: arange(7, 19, 8) sums columns 7 and 15, the reference divides by H * (20 // 8 - 1) = H.  Dividing by the
    2H summed positions instead is a different number on the golden."""
    from grl_image_restoration_b200 import metrics

    g = np.load(PSNRB_GOLDEN)
    restored, target = golden_pair(g, "rgb_w20")
    want = torch.from_numpy(g["rgb_w20_psnrb"]).double()
    assert (metrics.psnrb(restored, target) - want).abs().max().item() <= 1e-4
    k = (metrics.tensor_round(restored) * 255).round().double()
    bef = metrics._blocking_effect_factor(k)
    assert (bef > 0).any(), "the case must have blocking for the normaliser to matter"


def test_psnrb_rejects_malformed(pkg):
    from grl_image_restoration_b200 import metrics

    with pytest.raises(RuntimeError, match="16 x 16"):
        metrics.psnrb(torch.rand(1, 3, 15, 40), torch.rand(1, 3, 15, 40))
    with pytest.raises(RuntimeError, match="one shape"):
        metrics.psnrb(torch.rand(1, 3, 32, 32), torch.rand(1, 3, 32, 33))
    with pytest.raises(RuntimeError, match="RGB"):
        metrics.psnrb(torch.rand(1, 1, 32, 32), torch.rand(1, 1, 32, 32), channel="y")
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.psnrb_fused(torch.rand(1, 3, 32, 32), torch.rand(1, 3, 32, 32))


def test_psnrb_library_rejects_malformed(pkg):
    """The C ABI refuses small images and unsupported channel counts before it launches anything."""
    import ctypes

    from grl_image_restoration_b200 import capi

    L = capi.lib()
    dummy = ctypes.c_void_p(16)
    ws = L.grl_psnrb_workspace(1)
    assert ws == 160
    assert L.grl_psnrb_f32(dummy, dummy, 1, 3, 15, 40, dummy, ws, dummy, None, None) == -1
    assert b"16 x 16" in L.grl_last_error()
    assert L.grl_psnrb_f32(dummy, dummy, 1, 2, 32, 32, dummy, ws, dummy, None, None) == -1
    assert L.grl_psnrb_f32(dummy, dummy, 1, 3, 32, 32, dummy, ws - 8, dummy, None, None) == -1
