"""Tiled inference (SURVEY.md 8f row 1): batched tiles == the reference engine's sequential forward_tile."""
import pytest
import torch

from engine_oracle import forward_tile

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-3), ("fp16", 2e-2)])
def test_forward_tile_matches_engine_semantics(pkg, oracle, device, precision, tol):
    from grl_image_restoration_b200 import tiling

    cfg = pkg.configs.micro_config(img_size=32, upscale=2)
    sd = oracle.synth_state_dict(cfg, seed=0, style="init")
    m = pkg.GRL(**cfg)
    m.load_state_dict(sd, strict=False)
    m = m.to(device).eval()
    m.set_precision(precision)
    x = oracle.synth_input((2, 3, 40, 56), seed=11)
    with torch.no_grad():
        ref = forward_tile(lambda t: oracle.grl_forward(sd, cfg, t), x, 32, 8, 2)
    y = tiling.forward_tile(m, x.to(device), 32, 8, max_batch=5).cpu()
    assert y.shape == ref.shape == (2, 3, 80, 112)
    assert (y - ref).abs().max().item() <= tol
    assert tiling.tile_origins(40, 32, 8) == [0, 8] and tiling.tile_origins(56, 32, 8) == [0, 24]
