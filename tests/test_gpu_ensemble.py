"""x8 self-ensemble on the GPU: the gather / merge kernels bit-exact against torch rot90 / flip, GRL(self_ensemble=True)
against the unmodified reference's stored ensemble outputs (tests/golden/ensemble_*.npz) and against a Python loop of
8 plain forwards of the same module, CUDA-graph replay, and tiled inference."""
import pytest
import torch

from engine_oracle import augment, forward_tile, merge_reference
from support import build, ensemble_cases, loop_ensemble

pytestmark = pytest.mark.gpu
GATE = 1e-3  # fp32, BASELINE.json


@pytest.mark.parametrize("C", [1, 3, 6])
@pytest.mark.parametrize("H,W", [(37, 70), (5, 3), (33, 33)])
def test_gather_kernel_bit_exact(pkg, device, C, H, W):
    from grl_image_restoration_b200 import functional as K

    x = torch.randn(2, C, H, W, generator=torch.Generator().manual_seed(C * 100 + H)).to(device)
    for group in (0, 1):
        v = K.ens_gather(x, group)
        ref = torch.cat([augment(x, 2 * i + group) for i in range(4)])
        assert v.shape == ref.shape and torch.equal(v, ref), group


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("Hs,Ws", [(74, 140), (3, 5), (64, 64)])
def test_merge_kernel_bit_exact(pkg, device, C, Hs, Ws):
    from grl_image_restoration_b200 import functional as K

    B = 2
    g = torch.Generator().manual_seed(Hs * 7 + C)
    ya = torch.randn(4 * B, C, Hs, Ws, generator=g).to(device)
    yb = torch.randn(4 * B, C, Ws, Hs, generator=g).to(device)
    outs = [(ya if m % 2 == 0 else yb)[(m // 2) * B:(m // 2 + 1) * B] for m in range(8)]
    y = K.ens_merge(ya, yb, B)
    assert y.shape == (B, C, Hs, Ws) and torch.equal(y, merge_reference(outs))
    if Hs == Ws:  # both groups as the two halves of one tensor
        both = torch.cat([ya, yb])
        assert torch.equal(K.ens_merge(both[: 4 * B], both[4 * B:], B), y)


@pytest.mark.parametrize("name", ["micro_cab_x2", "micro_dn"])
def test_self_ensemble_fp32_vs_reference(pkg, oracle, golden_loader, device, name):
    c = ensemble_cases()[name]
    g = golden_loader(f"ensemble_{name}.npz")
    m = build(pkg, oracle, c["cfg"], device, "fp32", style="init", self_ensemble=True)
    x = g["input"].to(device)
    y = m(x)
    assert y.dtype == x.dtype and y.device == x.device and y.is_contiguous()
    err = (y.cpu() - g["merged"]).abs().max().item()
    print(f"{name}: x8 fp32 max-abs vs reference = {err:.3e}")
    assert y.shape == g["merged"].shape and err <= GATE
    assert torch.equal(x.cpu(), g["input"])  # input untouched


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("name", ["micro_cab_x2", "micro_dn"])
def test_self_ensemble_16bit_psnr_gate(pkg, oracle, golden_loader, device, name, precision):
    """The gate of the 16-bit end-to-end tests: |PSNR(cand, GT) - PSNR(ref, GT)| <= 0.01 dB, PSNR(cand, ref) >= 56 dB
    with fp16 operands (40 dB with bf16)."""
    c = ensemble_cases()[name]
    g = golden_loader(f"ensemble_{name}.npz")
    m = build(pkg, oracle, c["cfg"], device, precision, style="init", self_ensemble=True)
    assert m.precision == precision
    y = m(g["input"].to(device)).cpu()
    ref = g["merged"]
    assert y.shape == ref.shape and torch.isfinite(y).all()
    s = c["cfg"]["upscale"]
    b = s if s > 1 else 0
    gt = torch.rand(ref.shape, generator=torch.Generator().manual_seed(9))
    d_psnr = abs(oracle.psnr(y, gt, b).mean().item() - oracle.psnr(ref, gt, b).mean().item())
    p_cr = (-10 * torch.log10(((y - ref) ** 2).mean())).item()
    print(f"{name} x8 [{precision}]: max-abs {(y - ref).abs().max().item():.3e}  PSNR(cand, ref) {p_cr:.1f} dB  "
          f"|dPSNR vs GT| {d_psnr:.4f} dB")
    assert d_psnr <= 0.01
    assert p_cr >= (56.0 if precision == "fp16" else 40.0)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("hw", [(28, 44), (32, 32)])
def test_self_ensemble_equals_loop_of_plain_forwards(pkg, oracle, device, precision, hw):
    """Non-square (two view batches) and square (one shared view batch) inputs, 2 images each."""
    cfg = pkg.configs.micro_config()
    m = build(pkg, oracle, cfg, device, precision, style="init", self_ensemble=True)
    x = oracle.synth_input((2, 3, *hw), seed=21).to(device)
    ref = loop_ensemble(m, x)
    for mb in (1, 16):
        m.ensemble_max_batch = mb
        y = m(x)
        err = (y - ref).abs().max().item()
        print(f"{precision} {hw} ensemble_max_batch={mb}: max-abs vs loop of 8 plain forwards = {err:.3e}")
        assert y.shape == ref.shape and err <= 1e-6


def test_self_ensemble_off_is_the_plain_forward(pkg, oracle, device):
    cfg = pkg.configs.micro_config()
    x = oracle.synth_input((2, 3, 28, 44), seed=3).to(device)
    for precision in ("fp32", "fp16"):
        plain = build(pkg, oracle, cfg, device, precision, style="init")
        off = build(pkg, oracle, cfg, device, precision, style="init", self_ensemble=False)
        assert torch.equal(plain(x), off(x))
        off.self_ensemble = True
        assert not torch.equal(plain(x), off(x))


def test_self_ensemble_cuda_graph_matches_eager(pkg, oracle, device):
    """Each view chunk shape gets its own captured graph (3 + 3 + 2 views here); gather and merge run outside the graphs.
    The result is a fresh tensor: mutating it leaves the next call untouched."""
    cfg = pkg.configs.micro_config()
    m = build(pkg, oracle, cfg, device, "fp16", style="init", self_ensemble=True)
    m.ensemble_max_batch = 3
    x1 = oracle.synth_input((1, 3, 32, 32), seed=5).to(device)
    x2 = oracle.synth_input((1, 3, 32, 32), seed=6).to(device)
    e1, e2 = m(x1).clone(), m(x2).clone()
    m.use_cuda_graph = True
    g1 = m(x1)
    g1_copy = g1.clone()
    g1.clamp_(0, 0.1)
    g2 = m(x2)
    assert torch.equal(g1_copy, e1) and torch.equal(g2, e2) and torch.equal(m(x1), e1)
    assert len(m._graphs) == 2


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-3), ("fp16", 2e-2)])
def test_forward_tile_ensembles_every_tile(pkg, oracle, device, precision, tol):
    from grl_image_restoration_b200 import tiling

    cfg = pkg.configs.micro_config(img_size=32, upscale=2)
    sd = oracle.synth_state_dict(cfg, seed=0, style="init")
    m = build(pkg, oracle, cfg, device, precision, style="init", self_ensemble=True)
    x = oracle.synth_input((2, 3, 40, 56), seed=11)

    def x8_oracle(t):
        with torch.no_grad():
            return merge_reference([oracle.grl_forward(sd, cfg, augment(t, mode).contiguous()) for mode in range(8)])

    ref = forward_tile(x8_oracle, x, 32, 8, 2)
    y = tiling.forward_tile(m, x.to(device), 32, 8, max_batch=5).cpu()
    err = (y - ref).abs().max().item()
    print(f"forward_tile x8 [{precision}]: max-abs vs per-tile x8 reference loop = {err:.3e}")
    assert y.shape == ref.shape == (2, 3, 80, 112) and err <= tol
