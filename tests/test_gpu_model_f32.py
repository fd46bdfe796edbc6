"""End-to-end fp32 parity: GRL.forward on the GPU vs (a) outputs of the unmodified reference stored in
tests/golden, (b) the CPU oracle on fresh seeds.  Gate from BASELINE.json: <= 1e-3 max-abs in fp32."""
import pytest
import torch

from support import build

pytestmark = pytest.mark.gpu
GATE = 1e-3


@pytest.mark.parametrize("name", ["cfg1_tiny_x2_64", "micro_cab_x2", "micro_pad_dn", "micro_groups", "micro_odd_d",
                                  "micro_gray"])
def test_golden_reference_outputs(pkg, oracle, cases, golden_loader, device, name):
    c = cases[name]
    cfg = c["cfg"]
    m = build(pkg, oracle, cfg, device, "fp32", style="spread")
    x = oracle.synth_input((c["batch"], cfg["in_channels"], *c["hw"]), seed=1234, noise_sigma=c["sigma"])
    y = m(x.to(device)).cpu()
    ref = golden_loader(f"model_{name}.npz")["output"]
    assert y.shape == ref.shape
    err = (y - ref).abs().max().item()
    print(f"{name}: max-abs vs reference = {err:.3e}")
    assert err <= GATE


@pytest.mark.parametrize("variant,task,scale,size,hw", [("tiny", "sr", 4, 64, (64, 64)), ("base", "sr", 4, 64, (64, 64)),
                                                        ("small", "dn", 1, 128, (100, 120)),
                                                        ("tiny", "deblur", 1, 96, (96, 96))])
def test_released_configs_vs_oracle(pkg, oracle, device, variant, task, scale, size, hw):
    cfg = pkg.configs.grl_config(variant, task, scale, size)
    m = build(pkg, oracle, cfg, device, "fp32", style="spread", seed=3)
    sd = oracle.synth_state_dict(cfg, seed=3)
    x = oracle.synth_input((1, 3, *hw), seed=77, noise_sigma=50.0 if task == "dn" else 0.0)
    with torch.no_grad():
        ref = oracle.grl_forward(sd, cfg, x)
    y = m(x.to(device)).cpu()
    err = (y - ref).abs().max().item()
    print(f"{variant}/{task}: max-abs vs oracle = {err:.3e}; psnr(cand, oracle) = "
          f"{(-10 * torch.log10(((y - ref) ** 2).mean())).item():.1f} dB")
    assert y.shape == ref.shape and err <= GATE


def test_full_size_properties_base_sr_256(pkg, oracle, device):
    """BASELINE cfg4 geometry (GRL-Base x4, 256x256 tiles): size-independent properties instead of a 2-minute CPU
    oracle run -- batch invariance (tiles are independent), determinism, finite output, output shape."""
    cfg = pkg.configs.grl_config("base", "sr", 4, 256)
    m = build(pkg, oracle, cfg, device, "fp32", style="spread", seed=1)
    x = oracle.synth_input((2, 3, 256, 256), seed=1234).to(device)
    y = m(x)
    assert y.shape == (2, 3, 1024, 1024) and torch.isfinite(y).all()
    y0 = m(x[:1])
    assert (y0 - y[:1]).abs().max().item() <= 1e-5  # batch-invariant
    assert torch.equal(m(x[:1]), y0)  # run-to-run deterministic
    xs = torch.flip(x, dims=(0,))
    assert (m(xs) - torch.flip(y, dims=(0,))).abs().max().item() <= 1e-5


def test_resolution_change_and_engine_contract(pkg, oracle, device):
    """img_size != input size (tables rebuilt on the fly, grl.py:449-453), output is a fresh contiguous tensor the
    caller may mutate in place (engines/base.py:113, utils_image.py:31)."""
    cfg = pkg.configs.micro_config(img_size=32)
    m = build(pkg, oracle, cfg, device, "fp32", style="spread")
    sd = oracle.synth_state_dict(cfg, seed=0)
    x = oracle.synth_input((1, 3, 48, 80), seed=5)
    with torch.no_grad():
        ref = oracle.grl_forward(sd, cfg, x)
    xd = x.to(device)
    y = m(xd)
    assert (y.cpu() - ref).abs().max().item() <= GATE
    assert y.is_contiguous() and y.device == xd.device and y.dtype == xd.dtype
    y.clamp_(0, 1)
    assert torch.equal(xd.cpu(), x)  # input untouched
