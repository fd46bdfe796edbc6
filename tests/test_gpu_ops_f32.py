"""fp32 CUDA operators and modules vs the CPU oracle and tensors of the unmodified reference (run with -m gpu).
Tolerance: BASELINE.json's fp32 gate is 1e-3 max-abs; these checks use 2e-4.  The kernels themselves are tested on
every released launch path against float64 with derived bounds in test_gpu_f32_paths.py."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
TOL = 2e-4


def rnd(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale


def test_native_library_loaded(pkg, device):
    from grl_image_restoration_b200 import capi

    assert capi.lib().grl_device_ok() == 1, "not an sm_90 device"
    with open("/proc/self/maps") as f:
        assert "libgrl_b200.so" in f.read()


def _affine_sd(heads, seed):
    return {"logit_scale": torch.log(torch.tensor([4.0, 50.0, 150.0, 10.0][:heads])).view(heads, 1, 1),
            "cpb_mlp.0.weight": rnd((512, 2), seed, 0.7), "cpb_mlp.0.bias": rnd((512,), seed + 1, 0.05),
            "cpb_mlp.2.weight": rnd((heads, 512), seed + 2, 0.15)}


def _load_affine(mod, sd, device):
    mod.load_state_dict(sd)
    return mod.to(device)


def test_bias_table_and_affine(pkg, oracle, device):
    heads, ws = 3, (8, 4)
    sd = _affine_sd(heads, 30)
    table = oracle.coords_table(list(ws))
    index = oracle.position_index(list(ws))
    mask = oracle.shift_mask([16, 8], list(ws), [4, 2])
    attn = rnd((2 * mask.shape[0], heads, 32, 32), 33)
    ref = oracle.affine({"t." + k: v for k, v in sd.items()}, "t.", attn, table, index, mask)
    mod = _load_affine(pkg.AffineTransform(heads), sd, device)
    out = mod(attn.to(device), table.to(device), index.to(device), mask.to(device))
    assert (out.cpu() - ref).abs().max().item() <= 1e-4
    t = F.linear(torch.relu(F.linear(table, sd["cpb_mlp.0.weight"], sd["cpb_mlp.0.bias"])), sd["cpb_mlp.2.weight"])
    refb = (16 * torch.sigmoid(t)).view(-1, heads).t()
    assert (mod.bias_table(table.to(device)).cpu() - refb).abs().max().item() <= 1e-5


def test_block_and_stage_against_reference_taps(pkg, oracle, cases, golden_loader, device):
    """Module-by-module against tensors captured from the UNMODIFIED reference (tests/golden)."""
    cfg = cases["micro_cab_x2"]["cfg"]
    gold = golden_loader("model_micro_cab_x2.npz")
    for bi in range(4):
        gold.update(golden_loader(f"model_micro_cab_x2_block{bi}.npz"))
    m = pkg.GRL(**cfg)
    m.load_state_dict(oracle.synth_state_dict(cfg, seed=0), strict=False)
    m = m.to(device).eval()
    hw = (16, 32)
    xb = gold["block_input"].to(device)
    tim = m.get_table_index_mask(device, hw)
    for bi in range(4):
        blk = m.layers[0].blocks[bi]
        t = blk._get_table_index_mask(tim)
        assert (blk.attn.anchor(xb, hw).cpu() - gold[f"block{bi}/anchor"]).abs().max().item() <= TOL
        assert (blk.attn(xb, hw, t).cpu() - gold[f"block{bi}/attn_out"]).abs().max().item() <= TOL
        assert (blk.conv(xb, hw).cpu() - gold[f"block{bi}/cab"]).abs().max().item() <= TOL
        assert (blk(xb, hw, tim).cpu() - gold[f"block{bi}/out"]).abs().max().item() <= TOL
    assert (m.layers[0](xb, hw, tim).cpu() - gold["stage0/out"]).abs().max().item() <= 5e-4
