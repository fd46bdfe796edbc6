"""The oracle (oracle/grl_oracle.py) replayed against fixtures that were produced by the UNMODIFIED reference
(oracle/make_golden.py).  CPU only; this is what pins the parity oracle."""
import numpy as np
import pytest
import torch

from support import sha


GEOS = ["sr_small_128", "dn_small_128", "deblur_96x192", "jpeg_144", "dm_64", "yaml_default_64", "groups_g1_32",
        "micro_16x32", "micro_32_df1", "sr_base_256", "dn_base_128x256"]


@pytest.mark.parametrize("name", GEOS)
def test_oracle_geometry_digests(oracle, geometry_golden, name):
    g = geometry_golden["geometries"][name]
    if name in ("sr_base_256", "dn_base_128x256") and torch.get_num_threads() < 2:
        pytest.skip("large geometry")
    cfg = dict(window_size=g["window"], stripe_size=g["stripe"], stripe_groups=g["groups"],
               anchor_window_down_factor=g["df"])
    tim = oracle.table_index_mask(cfg, tuple(g["x_size"]))
    for k, digest in g["sha256"].items():
        assert list(tim[k].shape) == g["shape"][k], k
        assert sha(tim[k]) == digest, f"{name}:{k}"


def test_oracle_small_geometry_full(oracle, geometry_golden, golden_loader):
    small = golden_loader("geometry_small.npz")
    for name in ("micro_16x32", "micro_32_df1"):
        g = geometry_golden["geometries"][name]
        cfg = dict(window_size=g["window"], stripe_size=g["stripe"], stripe_groups=g["groups"],
                   anchor_window_down_factor=g["df"])
        tim = oracle.table_index_mask(cfg, tuple(g["x_size"]))
        for k, v in tim.items():
            assert torch.equal(v, small[f"{name}/{k}"]), (name, k)


@pytest.mark.parametrize("name", ["cfg1_tiny_x2_64", "micro_cab_x2", "micro_pad_dn", "micro_groups", "micro_odd_d",
                                  "micro_gray"])
def test_oracle_model_outputs(oracle, cases, golden_loader, name):
    c = cases[name]
    cfg = c["cfg"]
    sd = oracle.synth_state_dict(cfg, seed=0)
    x = oracle.synth_input((c["batch"], cfg["in_channels"], *c["hw"]), seed=1234, noise_sigma=c["sigma"])
    with torch.no_grad():
        y = oracle.grl_forward(sd, cfg, x)
    ref = golden_loader(f"model_{name}.npz")["output"]
    assert y.shape == ref.shape
    assert (y - ref).abs().max().item() <= 2e-6 * max(1.0, ref.abs().max().item())


def test_oracle_block_taps(oracle, cases, golden_loader):
    c = cases["micro_cab_x2"]
    cfg = c["cfg"]
    gold = golden_loader("model_micro_cab_x2.npz")
    for bi in range(4):
        gold.update(golden_loader(f"model_micro_cab_x2_block{bi}.npz"))
    sd = oracle.synth_state_dict(cfg, seed=0)
    xb = gold["block_input"]
    hw = (16, 32)
    tim = oracle.table_index_mask(cfg, hw)
    for bi in range(4):
        taps = {}
        with torch.no_grad():
            y = oracle.transformer_block(sd, f"layers.0.blocks.{bi}.", xb, hw, oracle.block_settings(cfg, 0, bi), tim, taps)
            taps["cab"] = oracle.cab(sd, f"layers.0.blocks.{bi}.conv.", xb, hw)
        for k in ("anchor", "x_window", "x_stripe", "attn_out", "cab"):
            assert (taps[k] - gold[f"block{bi}/{k}"]).abs().max().item() <= 5e-6, (bi, k)
        assert (y - gold[f"block{bi}/out"]).abs().max().item() <= 1e-5
    with torch.no_grad():
        ys = oracle.transformer_stage(sd, cfg, 0, xb, hw, tim)
    assert (ys - gold["stage0/out"]).abs().max().item() <= 2e-5


def test_oracle_psnr(oracle, golden_loader):
    gold = golden_loader("model_micro_cab_x2.npz")
    v = oracle.psnr(gold["psnr/a"], gold["psnr/b"], 4)
    assert torch.equal(v, gold["psnr/value_border4"])


def test_param_counts(oracle, pkg, geometry_golden):
    counts = geometry_golden["param_counts"]
    # paper Table 5 / SURVEY.md section 4: 0.89 / 0.91 / 3.49 / 20.20 M
    assert counts["tiny_sr_x2"] == 885420 and counts["base_sr_x4"] == 20201299 and counts["small_sr_x4"] == 3487715
    for key, (v, t, s, sz) in {"tiny_sr_x2": ("tiny", "sr", 2, 64), "base_dn_x1": ("base", "dn", 1, 128)}.items():
        shapes = oracle.param_shapes(pkg.configs.grl_config(v, t, s, sz))
        assert sum(int(np.prod(x)) for x in shapes.values()) == counts[key]


def test_routed_style_keeps_init_elsewhere(oracle, cases):
    """"routed" differs from "init" exactly in the routed parameter groups, and those are distinct per head / row."""
    cfg = cases["micro_odd_d"]["cfg"]
    a, r = oracle.synth_state_dict(cfg, style="init"), oracle.synth_state_dict(cfg, style="routed")
    routed = lambda n: ("logit_scale" in n or "cpb_mlp" in n or ".norm" in n or n.startswith("norm_")  # noqa: E731
                        or n.endswith(("qkv.body.bias", "reduction.bias", "proj.bias", "fc1.bias", "fc2.bias")))
    for n in a:
        assert torch.equal(a[n], r[n]) != routed(n), n
        if n.endswith("logit_scale"):
            assert r[n].unique().numel() == r[n].numel() and (r[n].min() >= 1.6) and (r[n].max() <= 5.02)
    p = "layers.0.blocks.0.attn."
    assert not torch.equal(r[p + "stripe_attn.attn_transform1.logit_scale"], r[p + "stripe_attn.attn_transform2.logit_scale"])
