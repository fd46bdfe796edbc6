"""Parity at BASELINE.json's native shapes against outputs of the UNMODIFIED reference (tests/golden/native_*.npz,
written by oracle/make_golden_native.py in the build container: reference fp32 CPU forward on seeded weights/inputs).

  cfg2 GRL-Small x4 256^2 | cfg3 GRL-Base DN sigma 50 256^2 (w32, 64x128, df2, no upsampler, input residual)
  cfg4 GRL-Base x4 256^2  | cfg5 GRL-Base motion deblur 480^2 tile (w12, 48x96, df4) and the whole 1280x720 frame
Gates (BASELINE.json): fp32 path <= 1e-3 max-abs; 16-bit operand path |PSNR(cand, GT) - PSNR(ref, GT)| <= 0.01 dB with
the reference's PSNR definition over the FULL output, and PSNR(cand, ref) >= 56 dB on the stored sub-sampled reference.
"""
import os

import numpy as np
import pytest
import torch

from support import build, native_model

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

GT_SEED = 9


def load(case):
    path = os.path.join(GOLD, f"native_{case}.npz")
    if not os.path.exists(path):
        pytest.skip(f"{path} not generated")
    return np.load(path)


def compare(oracle, y, gold, scale):
    s = int(gold["stride"])
    ref_sub = torch.from_numpy(gold["sub"])
    assert list(y.shape) == list(gold["shape"])
    sub = y[..., ::s, ::s]
    err = (sub - ref_sub).abs().max().item()
    p_cr = (-10 * torch.log10(((sub - ref_sub) ** 2).mean())).item()
    gt = torch.rand(y.shape, generator=torch.Generator().manual_seed(GT_SEED))
    p_cand = oracle.psnr(y, gt, scale if scale > 1 else 0)
    d_psnr = (p_cand.double() - torch.from_numpy(gold["psnr_ref_gt"])).abs().max().item()
    return err, p_cr, d_psnr


@pytest.mark.parametrize("case", ["cfg4_init", "cfg4_spread", "cfg3_init", "cfg3_spread", "cfg2_init", "cfg2_spread",
                                  "cfg5_init", "cfg5_spread"])
def test_fp32_path_vs_reference_native_shape(pkg, oracle, device, case):
    gold = load(case)
    shape_name, style = case.split("_")
    m, x, scale = native_model(pkg, oracle, shape_name, style, device, "fp32")
    y = m(x.to(device)).cpu()
    err, p_cr, d_psnr = compare(oracle, y, gold, scale)
    print(f"{case} [fp32]: max-abs vs reference {err:.3e}  PSNR(cand, ref) {p_cr:.1f} dB  |dPSNR vs GT| {d_psnr:.2e} dB")
    assert err <= 1e-3
    assert d_psnr <= 0.01


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("case", ["cfg4_init", "cfg3_init", "cfg2_init", "cfg5_init"])
def test_tensor_core_path_psnr_gate_native_shape(pkg, oracle, device, case, precision):
    """The constructor-distributed weights ("init") are the regime the 0.01 dB gate is defined on.  fp16 operands are
    the shipping format and must meet both gates; bf16 operands must meet the 0.01 dB gate, their PSNR(cand, ref) is
    reported (8-bit mantissas: SURVEY.md section 7)."""
    gold = load(case)
    shape_name, style = case.split("_")
    m, x, scale = native_model(pkg, oracle, shape_name, style, device, precision)
    y = m(x.to(device)).cpu()
    assert torch.isfinite(y).all()
    err, p_cr, d_psnr = compare(oracle, y, gold, scale)
    print(f"{case} [{precision}]: max-abs vs reference {err:.3e}  PSNR(cand, ref) {p_cr:.1f} dB  |dPSNR vs GT| {d_psnr:.2e} dB")
    assert d_psnr <= 0.01
    if precision == "fp16":
        assert p_cr >= 56.0


def test_cfg5_whole_frame_tiled(pkg, oracle, device):
    """1280x720 frame through tiling.forward_tile (tile 480 / overlap 48 -> 6 tiles) vs the reference model driven by
    the engine's own tile loop (engines/base.py:90-116)."""
    from grl_image_restoration_b200 import tiling

    gold = load("cfg5_frame")
    cfg = pkg.configs.grl_config("base", "deblur", 1, 480)
    m = build(pkg, oracle, cfg, device, "fp32", style="init")
    x = oracle.synth_input((1, 3, 720, 1280), seed=1234)
    for precision, gate in (("fp32", 1e-3), ("fp16", None)):
        m.set_precision(precision)
        y = tiling.forward_tile(m, x.to(device), int(gold["tile"]), int(gold["overlap"]), max_batch=3).cpu()
        err, p_cr, d_psnr = compare(oracle, y, gold, 1)
        print(f"cfg5 frame [{precision}]: max-abs {err:.3e}  PSNR(cand, ref) {p_cr:.1f} dB  |dPSNR vs GT| {d_psnr:.2e} dB")
        assert d_psnr <= 0.01
        if gate is not None:
            assert err <= gate
        else:
            assert p_cr >= 56.0
