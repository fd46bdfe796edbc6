"""x8 self-ensemble, host side: the closed-form view maps (grl_geometry.h d8_src / d8_inv through grl_d8_index_host)
against augment_img_tensor4's index maps, and the CPU oracle composed as 8 independent forwards against the unmodified
reference's per-view and merged outputs (tests/golden/ensemble_*.npz, oracle/make_golden_ensemble.py)."""
import pytest
import torch

from engine_oracle import INVERSE, augment
from support import ensemble_cases

SIZES = [(1, 1), (1, 7), (5, 3), (28, 44), (64, 64)]


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("mode", range(8))
def test_d8_index_matches_torch_ops(pkg, mode, H, W):
    from grl_image_restoration_b200 import functional as K

    img = torch.arange(H * W, dtype=torch.int32).view(1, 1, H, W)
    view = augment(img, mode)[0, 0]
    fwd = K.d8_index(mode, H, W)
    assert fwd.shape == view.shape and torch.equal(fwd, view)
    inv = K.d8_index(mode, H, W, inverse=True)
    assert inv.shape == (H, W)
    # inv_m o T_m is the identity, and the inverse map reads the image back out of the view
    assert torch.equal(augment(view[None, None], INVERSE.get(mode, mode))[0, 0], img[0, 0])
    assert torch.equal(view.flatten()[inv.flatten().long()].view(H, W), img[0, 0])
    assert torch.equal(fwd.flatten()[inv.flatten().long()], img.flatten())


def test_d8_index_rejects_bad_arguments(pkg):
    from grl_image_restoration_b200 import capi, functional as K

    with pytest.raises(RuntimeError, match="d8_index"):
        K.d8_index(8, 4, 4)
    assert capi.lib().grl_d8_index_host(0, 0, 4, 0, None) == -1


@pytest.mark.parametrize("name", ["micro_cab_x2", "micro_dn"])
def test_d8_index_reproduces_reference_views(pkg, golden_loader, name):
    """The views the reference's augment_img_tensor4 produced, gathered through the host expansion."""
    from grl_image_restoration_b200 import functional as K

    g = golden_loader(f"ensemble_{name}.npz")
    x = g["input"]
    B, C, H, W = x.shape
    planes = x.reshape(B * C, H * W)
    for mode in range(8):
        idx = K.d8_index(mode, H, W).long()
        v = planes[:, idx.flatten()].view(B, C, *idx.shape)
        assert torch.equal(v, g[f"view{mode}/input"]), mode


@pytest.mark.parametrize("name", ["micro_cab_x2", "micro_dn"])
def test_oracle_ensemble_matches_reference(pkg, oracle, golden_loader, name):
    """Contract: y = 0.125 * (V_0 + ... + V_7) in mode order, V_m = inv_m(forward(T_m(x))) -- 8 independent forwards,
    each padded on its own.  The oracle per view and composed, against the reference's stored outputs."""
    c = ensemble_cases()[name]
    cfg = c["cfg"]
    g = golden_loader(f"ensemble_{name}.npz")
    x = oracle.synth_input((c["batch"], cfg["in_channels"], *c["hw"]), seed=c["input_seed"], noise_sigma=c["sigma"])
    assert torch.equal(x, g["input"])
    sd = oracle.synth_state_dict(cfg, seed=c["seed"], style=c["style"])
    acc, worst = None, 0.0
    for mode in range(8):
        with torch.no_grad():
            out = oracle.grl_forward(sd, cfg, augment(x, mode).contiguous())
        ref = g[f"view{mode}/output"]
        assert out.shape == ref.shape
        worst = max(worst, (out - ref).abs().max().item())
        back = augment(out, INVERSE.get(mode, mode))
        acc = back.clone() if acc is None else acc + back
    y = acc * 0.125
    err = (y - g["merged"]).abs().max().item()
    s = cfg["upscale"]
    assert y.shape == (c["batch"], cfg["in_channels"], c["hw"][0] * s, c["hw"][1] * s)
    print(f"{name}: oracle vs reference, per view max-abs {worst:.3e}, merged max-abs {err:.3e}")
    assert worst <= 2e-6 * max(1.0, g["merged"].abs().max().item()) and err <= 2e-6


def test_self_ensemble_flag(pkg):
    cfg = pkg.configs.micro_config()
    m = pkg.GRL(**cfg)
    assert m.self_ensemble is False and m.ensemble_max_batch == 16
    m2 = pkg.GRL(self_ensemble=True, **cfg)
    assert m2.self_ensemble is True
    assert m.state_dict().keys() == m2.state_dict().keys()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m2(torch.rand(1, 3, 32, 32))
