"""bf16 tensor-core path, network level.  Gates (BASELINE.json / SURVEY.md 8d): |PSNR(cand, GT) - PSNR(ref, GT)| <= 0.01 dB
with the reference's PSNR definition (tensor_round + shave + per-image mean), and PSNR(cand, ref) reported."""
import pytest
import torch

from support import build

pytestmark = pytest.mark.gpu


def test_block_and_stage_bf16_vs_reference_taps(pkg, oracle, cases, golden_loader, device):
    cfg = cases["micro_cab_x2"]["cfg"]
    gold = golden_loader("model_micro_cab_x2.npz")
    for bi in range(4):
        gold.update(golden_loader(f"model_micro_cab_x2_block{bi}.npz"))
    m = build(pkg, oracle, cfg, device, "fp16", style="spread")
    assert m.precision == "fp16"
    hw = (16, 32)
    xb = gold["block_input"].to(device)
    tim = m.get_table_index_mask(device, hw)
    for bi in range(4):
        y = m.layers[0].blocks[bi](xb, hw, tim).cpu()
        ref = gold[f"block{bi}/out"]
        err = (y - ref).abs()
        print(f"block {bi}: bf16 max-abs {err.max().item():.3e} mean-abs {err.mean().item():.3e} (ref rms {ref.pow(2).mean().sqrt().item():.2f})")
        assert err.max().item() <= 1.0 and err.mean().item() <= 2e-2
    ys = m.layers[0](xb, hw, tim).cpu()
    err = (ys - gold["stage0/out"]).abs()
    print(f"stage: bf16 max-abs {err.max().item():.3e} mean-abs {err.mean().item():.3e}")
    assert err.mean().item() <= 0.15


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("variant,task,scale,size,hw", [("tiny", "sr", 2, 64, (64, 64)), ("small", "sr", 4, 64, (64, 64)),
                                                        ("base", "sr", 4, 64, (64, 64)), ("small", "dn", 1, 128, (100, 120)),
                                                        ("tiny", "deblur", 1, 96, (96, 96))])
def test_psnr_gate_vs_oracle(pkg, oracle, device, variant, task, scale, size, hw, precision):
    """Weights drawn like the reference's constructor does (style "init"): the realistic sensitivity regime.
    fp16 operands must meet the 0.01 dB gate with PSNR(cand, ref) >= 56 dB (SURVEY.md 8d); bf16 operands are
    reported (they cannot: 8-bit mantissas give ~45-50 dB, as SURVEY.md section 7 predicted)."""
    cfg = pkg.configs.grl_config(variant, task, scale, size)
    m = build(pkg, oracle, cfg, device, precision, style="init", seed=3)
    sd = oracle.synth_state_dict(cfg, seed=3, style="init")
    x = oracle.synth_input((1, 3, *hw), seed=77, noise_sigma=50.0 if task == "dn" else 0.0)
    with torch.no_grad():
        ref = oracle.grl_forward(sd, cfg, x)
    y = m(x.to(device)).cpu()
    assert y.shape == ref.shape and torch.isfinite(y).all()
    gt = torch.rand(ref.shape, generator=torch.Generator().manual_seed(9))
    b = scale if scale > 1 else 0
    d_psnr = abs(oracle.psnr(y, gt, b).mean().item() - oracle.psnr(ref, gt, b).mean().item())
    p_cr = (-10 * torch.log10(((y - ref) ** 2).mean())).item()
    print(f"{variant}/{task} [{precision}]: max-abs {(y - ref).abs().max().item():.3e}  PSNR(cand, ref) {p_cr:.1f} dB  |dPSNR vs GT| {d_psnr:.4f} dB")
    assert d_psnr <= 0.01
    assert p_cr >= (56.0 if precision == "fp16" else 40.0)


@pytest.mark.parametrize("variant,task,scale,size,hw", [("base", "sr", 4, 64, (64, 64)), ("tiny", "sr", 2, 64, (64, 64))])
def test_harsh_weights_report(pkg, oracle, device, variant, task, scale, size, hw):
    """The "spread" synthetic weights (logit scales up to the clamp at 100, random LayerNorm affine) make the network
    near-chaotic; reported for transparency with a loose sanity bound."""
    cfg = pkg.configs.grl_config(variant, task, scale, size)
    m = build(pkg, oracle, cfg, device, "fp16", style="spread", seed=3)
    sd = oracle.synth_state_dict(cfg, seed=3)
    x = oracle.synth_input((1, 3, *hw), seed=77)
    with torch.no_grad():
        ref = oracle.grl_forward(sd, cfg, x)
    y = m(x.to(device)).cpu()
    p_cr = (-10 * torch.log10(((y - ref) ** 2).mean())).item()
    print(f"{variant}/{task} [fp16, spread weights]: PSNR(cand, ref) {p_cr:.1f} dB  max-abs {(y - ref).abs().max().item():.3e}")
    assert p_cr >= 25.0


def test_fp16_fp32_switch(pkg, oracle, device):
    """Switching one model from the fp16 tensor-core path to the fp32 path.  (Batch composition, bit for bit, is
    test_gpu_tc_scale.py::test_batch_composition_bitwise.)"""
    cfg = pkg.configs.grl_config("base", "sr", 4, 256)
    m = build(pkg, oracle, cfg, device, "fp16", style="init", seed=1)
    x = oracle.synth_input((1, 3, 256, 256), seed=1234).to(device)
    y = m(x)
    assert y.shape == (1, 3, 1024, 1024) and torch.isfinite(y).all()
    m.set_precision("fp32")
    y32 = m(x)
    p = (-10 * torch.log10(((y - y32) ** 2).mean())).item()
    print(f"base sr 256: PSNR(fp16 path, fp32 path) = {p:.1f} dB, max-abs {(y - y32).abs().max().item():.3e}")
    assert p >= 25.0


@pytest.mark.parametrize("name", ["cfg1_tiny_x2_64", "micro_cab_x2", "micro_pad_dn", "micro_groups", "micro_odd_d", "micro_gray"])
def test_head_tail_fusion_all_heads(pkg, oracle, cases, device, name):
    """The fused head (reflect / zero pad + normalise + layout + pack in one kernel) and tails (PixelShuffle as a store
    pattern, x / range + mean + crop + bchw in the last conv's epilogue) of the tensor-core path against the fp32 path
    (torch-op head / tail, exact-parity kernels) for every head type: pixelshuffle, pixelshuffledirect (x3),
    nearest+conv, no upsampler with the input residual, 1-channel input, inputs that need padding."""
    c = cases[name]
    cfg = c["cfg"]
    sd = oracle.synth_state_dict(cfg, seed=0, style="init")
    m = pkg.GRL(**cfg)
    m.load_state_dict(sd, strict=False)
    m = m.to(device).eval()
    if m.set_precision("auto") == "fp32":
        pytest.skip("architecture outside the tensor-core path")
    x = oracle.synth_input((c["batch"], cfg["in_channels"], *c["hw"]), seed=1234, noise_sigma=c["sigma"]).to(device)
    y16 = m(x)
    m.set_precision("fp32")
    y32 = m(x)
    assert y16.shape == y32.shape and y16.is_contiguous() and torch.isfinite(y16).all()
    p = (-10 * torch.log10(((y16 - y32) ** 2).mean())).item()
    print(f"{name}: fp16 path vs fp32 path PSNR {p:.1f} dB, max-abs {(y16 - y32).abs().max().item():.3e}")
    assert p >= 50.0
    # odd sizes: crop + pad of a non-multiple input (configs with stripe_groups need square padded inputs: the reference
    # itself crashes otherwise, SURVEY.md Appendix D.2)
    if any(g is not None for g in cfg["stripe_groups"]):
        return
    xo = x[..., : x.shape[-2] - 3, : x.shape[-1] - 5].contiguous()
    m.set_precision("auto")
    a = m(xo)
    m.set_precision("fp32")
    b = m(xo)
    assert a.shape == b.shape
    assert (-10 * torch.log10(((a - b) ** 2).mean())).item() >= 50.0


def test_cuda_graph_replay_matches_eager(pkg, oracle, device):
    """GRL.use_cuda_graph: the captured graph of the tensor-core forward replays bit-identically to the eager launch
    sequence, for new inputs of the captured shape, a second shape gets its own graph, and the caller may mutate the
    result in place (engines/base.py:113) without touching the graph's static buffers."""
    cfg = pkg.configs.grl_config("base", "sr", 4, 64)
    m = build(pkg, oracle, cfg, device, "fp16", style="init", seed=3)
    x1 = oracle.synth_input((2, 3, 64, 64), seed=5).to(device)
    x2 = oracle.synth_input((2, 3, 64, 64), seed=6).to(device)
    e1, e2 = m(x1).clone(), m(x2).clone()
    m.use_cuda_graph = True
    g1 = m(x1)
    g1_copy = g1.clone()
    g1.clamp_(0, 0.1)  # in-place mutation by the caller
    g2 = m(x2)
    g1b = m(x1)
    assert torch.equal(g1_copy, e1) and torch.equal(g2, e2) and torch.equal(g1b, e1)
    x3 = oracle.synth_input((1, 3, 64, 128), seed=7).to(device)  # another shape: another graph
    g3 = m(x3)
    m.use_cuda_graph = False
    assert torch.equal(g3, m(x3)) and len(m._graphs) == 2
    m.load_state_dict(oracle.synth_state_dict(cfg, seed=4, style="init"), strict=False)
    assert len(m._graphs) == 0  # new weights: stale graphs are dropped
