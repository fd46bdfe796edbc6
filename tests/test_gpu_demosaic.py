"""Demosaicking on the GPU: the standalone kernel and the fused tensor-core head bit-exact against the library's host
closed form and the unfused path; GRL(input_format="rggb") against GRL on the demosaiced image (bit for bit) and against
the unmodified reference's dm pipeline (tests/golden/dm_*.npz); CUDA graphs, the x8 ensemble and tiled inference."""
import pytest
import torch

from support import dm_model

pytestmark = pytest.mark.gpu
NAMES = ["b2_40x56", "zero_pad_4x4", "odd_18x26"]


def pair(pkg, oracle, device, precision, **kw):
    return dm_model(pkg, oracle, device, precision, **kw), dm_model(pkg, oracle, device, precision, "rgb", **kw)


@pytest.mark.parametrize("h,w", [(2, 2), (5, 3), (9, 13), (16, 33), (40, 70), (33, 8)])
def test_kernel_bit_exact_vs_host(pkg, device, h, w):
    """Tiles with partial rows and columns, images smaller than one tile, signed values outside [0, 1]."""
    from grl_image_restoration_b200 import functional as K

    x = torch.randn(2, 4, h, w, generator=torch.Generator().manual_seed(h * 97 + w)) * 2
    y = K.demosaic(x.to(device))
    assert y.shape == (2, 3, 2 * h, 2 * w) and y.is_contiguous()
    assert torch.equal(y.cpu(), K.demosaic_host(x))


@pytest.mark.parametrize("name", NAMES)
def test_kernel_bit_exact_on_golden_inputs(pkg, golden_loader, device, name):
    from grl_image_restoration_b200 import functional as K

    cfa4 = golden_loader(f"dm_{name}.npz")["cfa4"]
    assert torch.equal(K.demosaic(cfa4.to(device)).cpu(), K.demosaic_host(cfa4))


def test_demosaic_rejects_bad_input(pkg, device):
    from grl_image_restoration_b200 import functional as K

    with pytest.raises(ValueError, match=r"\(B, 4, h, w\)"):
        K.demosaic(torch.rand(1, 3, 4, 4, device=device))
    with pytest.raises(ValueError, match="h, w >= 2"):
        K.demosaic(torch.rand(1, 4, 1, 4, device=device))
    with pytest.raises(RuntimeError, match="float32"):
        K.demosaic(torch.rand(1, 4, 4, 4, device=device, dtype=torch.float64))


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("h,w,Hp,Wp", [(20, 28, 64, 64), (2, 2, 32, 32), (9, 13, 32, 32), (8, 8, 16, 16), (5, 7, 10, 14)])
def test_fused_head_bit_exact_vs_demosaic_then_head(pkg, device, fmt, h, w, Hp, Wp):
    """grl_tc_head_pack_rggb == grl_tc_head_pack(demosaic(cfa4)), 16-bit operands and the fp32 copy: reflect padding,
    the zero fallback (pad > image), no padding, and padding of exactly the image size minus one."""
    from grl_image_restoration_b200 import functional as K, tc

    cfa4 = torch.rand(2, 4, h, w, generator=torch.Generator().manual_seed(h + 31 * w)).to(device)
    mean = [0.4488, 0.4371, 0.4040]
    a16, a32 = tc.head_pack_rggb(cfa4, Hp, Wp, mean, 1.0, 64, fmt, want_f32=True)
    b16, b32 = tc.head_pack(K.demosaic(cfa4), Hp, Wp, mean, 1.0, 64, fmt, want_f32=True)
    assert torch.equal(a16.view(torch.int16), b16.view(torch.int16)) and torch.equal(a32, b32)
    c16, c32 = tc.head_pack_rggb(cfa4, Hp, Wp, mean, 1.0, 64, fmt)
    assert c32 is None and torch.equal(c16.view(torch.int16), a16.view(torch.int16))


@pytest.mark.parametrize("precision", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_rggb_forward_equals_forward_of_demosaiced(pkg, oracle, golden_loader, device, precision, name):
    from grl_image_restoration_b200 import functional as K

    m_bayer, m_rgb = pair(pkg, oracle, device, precision)
    cfa4 = golden_loader(f"dm_{name}.npz")["cfa4"].to(device)
    y = m_bayer(cfa4)
    ref = m_rgb(K.demosaic(cfa4))
    err = (y - ref).abs().max().item()
    print(f"{name} [{precision}]: rggb forward vs forward(demosaic) max-abs {err:.1e}")
    assert y.shape == ref.shape == (cfa4.shape[0], 3, 2 * cfa4.shape[2], 2 * cfa4.shape[3]) and err == 0.0


@pytest.mark.parametrize("name", NAMES)
def test_rggb_fp32_vs_reference(pkg, oracle, golden_loader, device, name):
    g = golden_loader(f"dm_{name}.npz")
    m = dm_model(pkg, oracle, device, "fp32")
    y = m(g["cfa4"].to(device)).cpu()
    err = (y - g["output"]).abs().max().item()
    print(f"{name}: rggb fp32 max-abs vs reference dm pipeline = {err:.3e}")
    assert y.shape == g["output"].shape and err <= 1e-3


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_rggb_16bit_psnr_gate(pkg, oracle, golden_loader, device, name, precision):
    """The gate of the 16-bit end-to-end tests: |PSNR(cand, GT) - PSNR(ref, GT)| <= 0.01 dB, PSNR(cand, ref) >= 56 dB
    with fp16 operands (40 dB with bf16)."""
    g = golden_loader(f"dm_{name}.npz")
    m = dm_model(pkg, oracle, device, precision)
    assert m.precision == precision
    y = m(g["cfa4"].to(device)).cpu()
    ref = g["output"]
    assert y.shape == ref.shape and torch.isfinite(y).all()
    gt = torch.rand(ref.shape, generator=torch.Generator().manual_seed(9))
    d_psnr = abs(oracle.psnr(y, gt).mean().item() - oracle.psnr(ref, gt).mean().item())
    p_cr = (-10 * torch.log10(((y - ref) ** 2).mean())).item()
    print(f"{name} rggb [{precision}]: max-abs {(y - ref).abs().max().item():.3e}  PSNR(cand, ref) {p_cr:.1f} dB  "
          f"|dPSNR vs GT| {d_psnr:.4f} dB")
    assert d_psnr <= 0.01
    assert p_cr >= (56.0 if precision == "fp16" else 40.0)


def test_rggb_cuda_graph_matches_eager(pkg, oracle, golden_loader, device):
    """The fused head is captured with the network; the graph key carries the input format, so the same module replays
    a packed input and an RGB input of the same batch from different graphs."""
    from grl_image_restoration_b200 import functional as K

    m = dm_model(pkg, oracle, device, "fp16")
    x1 = golden_loader("dm_b2_40x56.npz")["cfa4"].to(device)
    x2 = x1.flip(-1).contiguous()
    e1, e2 = m(x1).clone(), m(x2).clone()
    rgb = K.demosaic(x1)
    e_rgb = m.forward_rgb(rgb).clone()
    m.use_cuda_graph = True
    g1 = m(x1)
    g1_copy = g1.clone()
    g1.zero_()
    g2 = m(x2)
    assert torch.equal(g1_copy, e1) and torch.equal(g2, e2) and torch.equal(m(x1), e1)
    assert torch.equal(m.forward_rgb(rgb), e_rgb)
    assert sorted(k[-1] for k in m._graphs) == ["rgb", "rggb"]


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_rggb_self_ensemble_is_ensemble_of_demosaiced(pkg, oracle, golden_loader, device, precision):
    from grl_image_restoration_b200 import functional as K

    m_bayer, m_rgb = pair(pkg, oracle, device, precision, self_ensemble=True)
    cfa4 = golden_loader("dm_b2_40x56.npz")["cfa4"].to(device)
    y = m_bayer(cfa4)
    assert torch.equal(y, m_rgb(K.demosaic(cfa4)))
    m_bayer.self_ensemble = False
    assert not torch.equal(m_bayer(cfa4), y)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_rggb_forward_tile_demosaics_the_whole_frame(pkg, oracle, golden_loader, device, precision):
    """forward_tile of packed planes == forward_tile of the demosaiced frame; demosaicing tile by tile would not be."""
    from grl_image_restoration_b200 import functional as K, tiling

    m_bayer, m_rgb = pair(pkg, oracle, device, precision)
    cfa4 = golden_loader("dm_b2_40x56.npz")["cfa4"].to(device)
    rgb = K.demosaic(cfa4)
    y = tiling.forward_tile(m_bayer, cfa4, 32, 8, max_batch=3)
    ref = tiling.forward_tile(m_rgb, rgb, 32, 8, max_batch=3)
    assert y.shape == ref.shape == (2, 3, 40, 56) and torch.equal(y, ref)
    y_sh = tiling.forward_tile_sharded(m_bayer, cfa4, 32, 8, max_batch=3)  # no process group: forward_tile
    assert torch.equal(y_sh, ref)
    per_tile = tiling.forward_tile(lambda p: m_rgb(K.demosaic(p.contiguous())), cfa4, 16, 4, scale=2, max_batch=3)
    assert per_tile.shape == ref.shape and not torch.equal(per_tile, ref)


def test_rggb_rejects_other_shapes(pkg, oracle, device):
    m = dm_model(pkg, oracle, device, "fp16")
    for bad in ((1, 3, 8, 8), (1, 4, 1, 8), (4, 8, 8)):
        with pytest.raises(ValueError, match=r"\(B, 4, h, w\)"):
            m(torch.rand(*bad, device=device))
