"""The anchor_proj_type / anchor_one_stage / conv_type switches on the CPU: the restatement against the reference's
goldens, state-dict names and shapes, the constructor's validity check, the gather weight packing, and the released
configs' launch lists (unchanged by the switches)."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import switch_cases as sw

CASES = sw.switch_cases()["cases"]
VALID = [n for n, c in CASES.items() if c["valid"]]


def _load(name):
    z = np.load(os.path.join(sw.GOLD, f"switches_{name}.npz"))
    return torch.from_numpy(z["x"]), torch.from_numpy(z["y"])


@pytest.mark.parametrize("name", VALID)
def test_restatement_matches_reference_golden(oracle, name):
    c = CASES[name]
    x, y = _load(name)
    sd = sw.synth_state_dict(oracle, c["kwargs"], _all_shapes(c))
    with torch.no_grad():
        got = sw.grl_forward(oracle, sd, c["kwargs"], x)
    assert torch.equal(got, y)


def _all_shapes(c):
    """The full {name: shape} of the reference network: grl_oracle's parameters with the switched anchor / stage-conv
    entries the golden records in their place."""
    import grl_oracle

    base = {k: list(v) for k, v in grl_oracle.param_shapes(c["kwargs"]).items()
            if ".anchor." not in k and not (k.startswith("layers.") and ".conv." in k and ".blocks." not in k)
            and not k.startswith("conv_after_body")}
    base.update(c["param_shapes"])
    return base


@pytest.mark.parametrize("name", VALID)
def test_state_dict_matches_reference(pkg, name):
    from make_golden_zoo import param_summary

    c = CASES[name]
    m = pkg.GRL(**c["kwargs"])
    shapes = {k: list(v.shape) for k, v in m.state_dict().items() if k.split("_")[0] not in ("table", "index", "mask")}
    assert param_summary(shapes) == c["params"]
    assert _all_shapes(c) == shapes


@pytest.mark.parametrize("name", VALID)
def test_reference_checkpoint_loads_strictly(pkg, oracle, tmp_path, name):
    from grl_image_restoration_b200 import checkpoint

    c = CASES[name]
    sd = sw.synth_state_dict(oracle, c["kwargs"], _all_shapes(c))
    path = tmp_path / "ref.ckpt"
    torch.save({"state_dict": {f"model.{k}": v for k, v in sd.items()}}, path)
    m = pkg.GRL(**c["kwargs"])
    checkpoint.load_reference_checkpoint(m, str(path))
    for k, v in m.state_dict().items():
        if k in sd:
            assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize("name", list(CASES))
def test_constructor_rejects_exactly_what_the_reference_cannot_run(pkg, name):
    c = CASES[name]
    if c["valid"]:
        pkg.GRL(**c["kwargs"])
    else:
        with pytest.raises(ValueError):
            pkg.GRL(**c["kwargs"])


def test_out_proj_type_is_ignored(pkg):
    cfg = pkg.configs.micro_config()
    a = pkg.GRL(**{**cfg, "out_proj_type": "anything"})
    b = pkg.GRL(**cfg)
    assert {k: v.shape for k, v in a.state_dict().items()} == {k: v.shape for k, v in b.state_dict().items()}


def test_unknown_switch_values_raise(pkg):
    cfg = pkg.configs.micro_config()
    with pytest.raises(ValueError):
        pkg.GRL(**{**cfg, "conv_type": "2conv"})
    with pytest.raises(ValueError):
        pkg.GRL(**{**cfg, "anchor_proj_type": "pool"})
    for key in ("anchor_proj_type", "qkv_proj_type"):
        with pytest.raises(NotImplementedError, match="separable_conv_act"):
            pkg.GRL(**{**cfg, key: "separable_conv"})


@pytest.mark.parametrize("k,stride,pad,row_major", [(3, 2, 1, True), (5, 4, 2, True), (2, 2, 0, False)])
def test_gather_packing_matches_float64_unfold(pkg, k, stride, pad, row_major):
    """patch rows in K.anchor_gather's layout (an unfold, taps reordered) times K.pack_conv_weight's (N, tap*C + c)
    weight == the convolution (row-major taps), or PatchMerging's cat + Linear (column-major taps), in float64."""
    from grl_image_restoration_b200 import functional as K

    g = torch.Generator().manual_seed(k)
    B, C, H, W, N = 2, 5, 12, 8, 7
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    cols = F.unfold(x, k, padding=pad, stride=stride)  # (B, C*k*k, L), index c*k*k + ky*k + kx
    cols = cols.view(B, C, k, k, -1)
    cols = (cols.permute(0, 4, 2, 3, 1) if row_major else cols.permute(0, 4, 3, 2, 1)).reshape(B, -1, k * k * C)
    Ho, Wo = K.gather_size(H, W, k, stride, pad)
    if row_major:
        w = torch.randn(N, C, k, k, generator=g, dtype=torch.float64)
        ref = F.conv2d(x, w, stride=stride, padding=pad).flatten(2).transpose(1, 2)
        got = cols @ K.pack_conv_weight(w).t()
    else:
        w = torch.randn(N, 4 * C, generator=g, dtype=torch.float64)
        u = x.permute(0, 2, 3, 1)
        ref = F.linear(torch.cat([u[:, 0::2, 0::2], u[:, 1::2, 0::2], u[:, 0::2, 1::2], u[:, 1::2, 1::2]], -1), w)
        ref = ref.reshape(B, -1, N)
        got = cols @ w.t()
    assert got.shape == (B, Ho * Wo, N)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


def test_released_launch_lists_unchanged(pkg):
    with open(os.path.join(sw.GOLD, "switches_released_listing.json")) as f:
        want = json.load(f)
    assert sw.released_listings(pkg) == want
