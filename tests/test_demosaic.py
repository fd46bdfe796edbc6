"""Demosaicking, host side: the oracle restatement of dm_matlab and the library's closed form (grl_demosaic.h through
grl_demosaic_host) against the unmodified reference's stored outputs (tests/golden/dm_*.npz, oracle/make_golden_dm.py)
and against a float64 evaluation, with a derived bound; mutation controls that the bound must catch; the module surface.

Gate: an fp32 response of <= 11 exact-weight products is within gamma_11 * sum|w_i m_i| of the exact value whatever the
summation order (dm_oracle.dm_matlab_bound), so two fp32 evaluations are within twice that of each other."""
import pytest
import torch
import torch.nn.functional as F

import dm_oracle  # oracle/dm_oracle.py (conftest puts oracle/ on sys.path)
from support import dm_cases

NAMES = ["b2_40x56", "zero_pad_4x4", "odd_18x26"]


def ulp32(v):
    """fp32 ulp of float64 values (the spacing at |v|; the smallest normal's for 0)."""
    a = v.abs().to(torch.float32).clamp_min(torch.finfo(torch.float32).tiny)
    return (torch.nextafter(a, torch.tensor(float("inf"))) - a).to(torch.float64)


def within(cand, ref, bound):
    return bool(((cand.double() - ref.double()).abs() <= bound).all())


def pad_to(cfg, H, W):
    p = max(cfg["window_size"], *[s for s in cfg["stripe_size"] if s])
    return (H + p - 1) // p * p, (W + p - 1) // p * p


def head_reference(rgb, Hp, Wp):
    """check_image_size of the demosaiced image (grl.py:479-489): reflect, or zeros when the pad exceeds the image."""
    H, W = rgb.shape[2:]
    try:
        return F.pad(rgb, (0, Wp - W, 0, Hp - H), "reflect")
    except BaseException:
        return F.pad(rgb, (0, Wp - W, 0, Hp - H), "constant")


def head_padded_coordinate(cfa4, Hp, Wp):
    """Mutation of the fused head: the demosaic evaluated at the PADDED coordinate, on the mosaic reflect-padded to
    (Hp, Wp), instead of at the source pixel the padding maps it to.  (Only the colour phase from the padded coordinate
    would change nothing: reflecting about an edge of even length, 2 (H - 1) - y, keeps every index's parity.)"""
    B, _, h, w = cfa4.shape
    cfa = torch.zeros(B, 1, 2 * h, 2 * w, dtype=torch.float64)
    for i, (py, px) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        cfa[:, 0, py::2, px::2] = cfa4[:, i].double()
    big = F.pad(cfa, (0, Wp - 2 * w, 0, Hp - 2 * h), "reflect")
    planes = torch.stack([big[:, 0, py::2, px::2] for py, px in ((0, 0), (0, 1), (1, 0), (1, 1))], 1)
    return dm_oracle.dm_matlab(planes, torch.float64)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_reference_dm_matlab(golden_loader, name):
    g = golden_loader(f"dm_{name}.npz")
    cfa4, ref = g["cfa4"], g["rgb"]
    assert torch.equal(cfa4, torch.round(cfa4 * 255) / 255)  # uint8 mosaics / 255
    mine = dm_oracle.dm_matlab(cfa4)
    assert mine.dtype == torch.float32 and mine.shape == ref.shape
    bound = dm_oracle.dm_matlab_bound(cfa4)
    print(f"{name}: oracle fp32 vs reference max-abs {(mine - ref).abs().max().item():.3e}")
    assert within(mine, ref, 2 * bound)
    assert within(dm_oracle.dm_matlab(cfa4, torch.float64), ref, bound)


@pytest.mark.parametrize("name", NAMES)
def test_host_closed_form_vs_float64_and_reference(pkg, golden_loader, name):
    from grl_image_restoration_b200 import functional as K

    g = golden_loader(f"dm_{name}.npz")
    cfa4 = g["cfa4"]
    host = K.demosaic_host(cfa4)
    exact = dm_oracle.dm_matlab(cfa4, torch.float64)
    bound = dm_oracle.dm_matlab_bound(cfa4)
    err = (host.double() - exact).abs()
    print(f"{name}: host vs float64 max-abs {err.max().item():.3e}, worst {(err / ulp32(exact)).max().item():.2f} fp32 ulp; "
          f"vs reference max-abs {(host - g['rgb']).abs().max().item():.3e}")
    assert host.shape == g["rgb"].shape
    assert within(host, exact, bound)
    assert within(host, g["rgb"], 2 * bound)
    # raw mosaic sites are copies
    for c, (py, px), i in ((0, (0, 0), 0), (1, (0, 1), 1), (1, (1, 0), 2), (2, (1, 1), 3)):
        assert torch.equal(host[:, c, py::2, px::2], cfa4[:, i])


@pytest.mark.parametrize("h,w", [(2, 2), (2, 7), (5, 3), (16, 33)])
def test_host_closed_form_random_shapes(pkg, h, w):
    """Signed inputs outside [0, 1] and odd sizes, including the smallest legal one (2 x 2 quads)."""
    from grl_image_restoration_b200 import functional as K

    cfa4 = torch.randn(2, 4, h, w, generator=torch.Generator().manual_seed(h * 100 + w)) * 3
    host = K.demosaic_host(cfa4)
    assert host.shape == (2, 3, 2 * h, 2 * w)
    assert within(host, dm_oracle.dm_matlab(cfa4, torch.float64), dm_oracle.dm_matlab_bound(cfa4))


@pytest.mark.parametrize("mutation", ["swap_krbg", "zero_pad", "grbg"])
@pytest.mark.parametrize("name", NAMES)
def test_demosaic_mutations_fail_the_gate(golden_loader, name, mutation):
    g = golden_loader(f"dm_{name}.npz")
    cfa4 = g["cfa4"]
    bad = dm_oracle.dm_matlab(cfa4, torch.float64, mutation=mutation)
    assert not within(bad, g["rgb"], 2 * dm_oracle.dm_matlab_bound(cfa4)), mutation


@pytest.mark.parametrize("name", ["b2_40x56", "odd_18x26"])
def test_head_padded_coordinate_mutation_fails_the_gate(golden_loader, name):
    """The fused head's contract on the reflect-padded cases, in float64: the padded input is check_image_size of the
    demosaiced image.  The control passes the gate, the mutation does not."""
    c = dm_cases()
    g = golden_loader(f"dm_{name}.npz")
    cfa4, ref = g["cfa4"], g["rgb"]
    Hp, Wp = pad_to(c["cfg"], *ref.shape[2:])
    assert Hp > ref.shape[2] and Wp > ref.shape[3]
    gate = 2 * head_reference(dm_oracle.dm_matlab_bound(cfa4), Hp, Wp)
    want = head_reference(ref, Hp, Wp)
    assert within(head_reference(dm_oracle.dm_matlab(cfa4, torch.float64), Hp, Wp), want, gate)
    assert not within(head_padded_coordinate(cfa4, Hp, Wp), want, gate)


def test_demosaic_host_rejects_bad_arguments(pkg):
    from grl_image_restoration_b200 import capi

    assert capi.lib().grl_demosaic_host(None, 1, 2, 2, None) == -1
    assert b"demosaic_host" in capi.lib().grl_last_error()
    x = torch.zeros(1, 4, 1, 3)
    out = torch.zeros(1, 3, 2, 6)
    assert capi.lib().grl_demosaic_host(x.data_ptr(), 1, 1, 3, out.data_ptr()) == -1


def test_demosaic_entries_in_header_and_library(pkg):
    from grl_image_restoration_b200 import capi

    names = set(capi.header_symbols())
    for n in ("grl_demosaic_host", "grl_demosaic_f32", "grl_tc_head_pack_rggb", "grl_tc_head_pack"):
        assert n in names and n in capi._SIGNATURES and hasattr(capi.lib(), n)
    assert capi.ABI_VERSION == 6 and capi.lib().grl_abi_version() == 6


def test_input_format_flag(pkg):
    cfg = pkg.configs.grl_config("small", "dm", img_size=64)
    m = pkg.GRL(**cfg)
    assert m.input_format == "rgb"
    m2 = pkg.GRL(input_format="rggb", **cfg)
    assert m2.input_format == "rggb"
    assert m.state_dict().keys() == m2.state_dict().keys()
    with pytest.raises(ValueError, match="input_format"):
        pkg.GRL(input_format="bayer", **cfg)
    with pytest.raises(ValueError, match="in_channels"):
        pkg.GRL(input_format="rggb", **dict(pkg.configs.micro_config(in_channels=1, upsampler="", upscale=1)))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m2(torch.rand(1, 4, 8, 8))


def test_gemm_launches_of_packed_input_match_the_demosaiced_shape(pkg):
    from grl_image_restoration_b200 import tc

    cfg = pkg.configs.grl_config("small", "dm", img_size=64)
    rgb = pkg.GRL(precision="fp16", **cfg)
    bayer = pkg.GRL(precision="fp16", input_format="rggb", **cfg)
    a, b = tc.gemm_launches(rgb, (2, 3, 40, 56)), tc.gemm_launches(bayer, (2, 4, 20, 28))
    assert len(a) == len(b) > 0 and [repr(x) for x in a] == [repr(x) for x in b]
