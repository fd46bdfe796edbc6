"""The fused PSNR-B kernel (csrc/metric.cu behind grl_psnrb_f32) against the reference's own psnrb
(tests/golden/psnrb.npz) and the torch-op definition metrics.psnrb, plus mutation controls that must fail the 1e-4 dB
gate."""
import math
import os

import numpy as np
import pytest
import torch

from test_psnrb import CASES, golden_case

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "psnrb.npz")


@pytest.mark.parametrize("case", CASES)
def test_fused_psnrb_matches_reference(pkg, device, case):
    from grl_image_restoration_b200 import metrics

    g = np.load(GOLDEN)
    restored, target = (t.to(device) for t in golden_case(g, case))
    keep = restored.clone()
    p, py = metrics.psnrb_fused(restored, target)
    assert torch.equal(restored, keep)
    assert (p.cpu() - torch.from_numpy(g[f"{case}_psnrb"]).double()).abs().max().item() <= 1e-4
    want_y = g[f"{case}_psnrb_y"] if f"{case}_psnrb_y" in g else g[f"{case}_psnrb"]
    assert (py.cpu() - torch.from_numpy(want_y).double()).abs().max().item() <= 1e-4
    assert (p.cpu() - metrics.psnrb(restored.cpu(), target.cpu())).abs().max().item() <= 1e-10


@pytest.mark.parametrize("shape", [(1, 3, 16, 16), (2, 1, 16, 40), (3, 3, 67, 45), (2, 3, 256, 256), (1, 1, 96, 20),
                                   (1, 3, 1356, 2040), (1, 3, 2040, 1356)])
def test_fused_psnrb_vs_torch_ops(pkg, device, shape):
    from grl_image_restoration_b200 import metrics

    g = torch.Generator().manual_seed(11)
    a = (torch.rand(shape, generator=g) * 1.3 - 0.15).to(device)
    b = torch.rand(shape, generator=g).to(device)
    p, py = metrics.psnrb_fused(a, b)
    assert (p - metrics.psnrb(a, b)).abs().max().item() <= 1e-10
    if shape[1] == 3:
        assert (py - metrics.psnrb(a, b, "y")).abs().max().item() <= 2e-3  # luma: rare round-to-8-bit ties
    else:
        assert torch.equal(py, p)
    p2, py2 = metrics.psnrb_fused(a, b)
    assert torch.equal(p, p2) and torch.equal(py, py2)  # integer sums: bit-identical run to run


def _mutated(restored, target, counts=False, on_target=False):
    """metrics.psnrb with one deliberate change (float64, 8-bit integers)."""
    from grl_image_restoration_b200 import metrics

    ka = metrics._grid8(metrics.tensor_round(restored))
    kb = metrics._grid8(metrics.tensor_round(target))
    H, W = ka.shape[-2:]
    src = kb if on_target else ka
    if counts:
        dh = (src[..., :, :-1] - src[..., :, 1:]).pow(2)
        dv = (src[..., :-1, :] - src[..., 1:, :]).pow(2)
        bh = torch.arange(W - 1, device=src.device) % 8 == 7
        bv = torch.arange(H - 1, device=src.device) % 8 == 7
        n_b = H * int(bh.sum()) + W * int(bv.sum())
        n_n = H * int((~bh).sum()) + W * int((~bv).sum())
        bd = (dh[..., bh].sum((-2, -1)) + dv[..., bv, :].sum((-2, -1))) / n_b
        nd = (dh[..., ~bh].sum((-2, -1)) + dv[..., ~bv, :].sum((-2, -1))) / n_n
        bef = torch.where(bd <= nd, torch.zeros_like(bd), math.log2(8) / math.log2(min(H, W)) * (bd - nd))
    else:
        bef = metrics._blocking_effect_factor(src)
    mse = (ka - kb).pow(2).mean((-2, -1))
    return (10 * torch.log10(65025.0 / (mse + bef))).mean(1)


@pytest.mark.parametrize("mutation", ["counts", "on_target"])
def test_mutations_fail_the_gate(pkg, device, mutation):
    g = np.load(GOLDEN)
    worst = 0.0
    for case in CASES:
        restored, target = golden_case(g, case)
        got = _mutated(restored, target, counts=mutation == "counts", on_target=mutation == "on_target")
        worst = max(worst, (got - torch.from_numpy(g[f"{case}_psnrb"]).double()).abs().max().item())
    assert worst > 1e-4, f"mutation {mutation} passes the gate: the goldens do not pin it"
