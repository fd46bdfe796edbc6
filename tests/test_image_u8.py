"""8-bit images, host side: the closed forms of csrc/grl_image_u8.h through the library's host expansions
(grl_u8_to_f32_host, grl_f32_to_u8_host) against NumPy's and torch's own formulas on every 8-bit value and on the special
values of the float side; argument checks that need no GPU."""
import numpy as np
import pytest
import torch


def all_bytes():
    return torch.arange(256, dtype=torch.uint8).reshape(1, 1, 256, 1)


def torch_round8(v):
    """tensor_round (utils/utils_image.py:30-33) times 255, in fp32 on the CPU."""
    return (v.clamp(0, 1) * 255).round()


def test_unit_is_numpy_ieee_division_and_round8_inverts_it(pkg):
    from grl_image_restoration_b200 import functional as K

    unit = K.u8_to_f32_host(all_bytes()).reshape(-1)
    want = np.arange(256, dtype=np.float32) / np.float32(255)
    assert np.array_equal(unit.numpy(), want)
    assert torch.equal(unit, all_bytes().reshape(-1).float().div(255))  # to_tensor on the CPU
    # round8(k / 255) == k: why an 8-bit image and u8_to_f32 of it have the same metrics bit for bit
    back = K.f32_to_u8_host(unit.reshape(1, 1, 1, 256)).reshape(-1)
    assert torch.equal(back, torch.arange(256, dtype=torch.uint8))


def test_round8_matches_torch_on_ties_zeros_range_and_infinities(pkg):
    from grl_image_restoration_b200 import functional as K

    k = torch.arange(255, dtype=torch.float32)
    ties = (k + 0.5) / 255
    tiny = torch.finfo(torch.float32).tiny
    special = torch.tensor([0.0, -0.0, -tiny, tiny, -1e-8, -3.0, 1.0, 1.0000001, 1.5, 2.0, 1e30, -1e30, 255.0,
                            float("inf"), float("-inf")])
    g = torch.Generator().manual_seed(0)
    spread = torch.cat([torch.rand(4096, generator=g), torch.randn(4096, generator=g) * 2])
    v = torch.cat([ties, special, spread])
    got = K.f32_to_u8_host(v.reshape(1, 1, 1, -1)).reshape(-1)
    assert got.dtype == torch.uint8
    assert torch.equal(got.float(), torch_round8(v))
    # the ties really are ties in fp32 for some k, and they go to the even neighbour like torch.round
    exact = (ties * 255) == k + 0.5
    assert exact.any()
    assert torch.equal(got[:255][exact].long() % 2, torch.zeros(int(exact.sum()), dtype=torch.long))


def test_nan_gives_zero(pkg):
    from grl_image_restoration_b200 import functional as K

    v = torch.tensor([float("nan"), -float("nan"), 0.5, float("nan")]).reshape(1, 1, 2, 2)
    assert K.f32_to_u8_host(v).reshape(-1).tolist() == [0, 0, 128, 0]


@pytest.mark.parametrize("B,C,H,W", [(1, 1, 1, 1), (2, 3, 5, 7), (1, 6, 3, 2)])
def test_host_layouts_are_hwc_and_chw(pkg, B, C, H, W):
    from grl_image_restoration_b200 import functional as K

    img = torch.randint(0, 256, (B, H, W, C), dtype=torch.uint8, generator=torch.Generator().manual_seed(B * C + H))
    planes = K.u8_to_f32_host(img)
    assert planes.shape == (B, C, H, W)
    assert torch.equal(planes, img.permute(0, 3, 1, 2).float().div(255))
    assert torch.equal(K.f32_to_u8_host(planes), img)


def test_host_entry_points_reject_bad_arguments(pkg):
    from grl_image_restoration_b200 import capi

    assert capi.lib().grl_u8_to_f32_host(None, 1, 1, 1, 3, None) == -1
    assert b"u8_to_f32_host" in capi.lib().grl_last_error()
    x = torch.zeros(4)
    y = torch.zeros(4, dtype=torch.uint8)
    assert capi.lib().grl_f32_to_u8_host(x.data_ptr(), 1, 0, 2, 2, y.data_ptr()) == -1
    assert b"f32_to_u8_host" in capi.lib().grl_last_error()


def test_device_entry_points_validate_before_launching(pkg):
    """Shape checks come before any device work, so they hold on a machine without a GPU."""
    from grl_image_restoration_b200 import capi

    L = capi.lib()
    p = 16  # a non-NULL address that is never dereferenced: every call below is refused first
    assert L.grl_u8_to_f32(p, 1, 4, 4, 9, p, None) == -1
    assert b"C must be 1..8" in L.grl_last_error()
    assert L.grl_f32_to_u8(p, 1, 0, 4, 4, p, None) == -1
    assert L.grl_u8_to_f32(None, 1, 4, 4, 3, p, None) == -1
    assert b"null" in L.grl_last_error()
    assert L.grl_psnrb_u8(p, p, 1, 8, 8, 3, p, 1 << 20, p, None, None) == -1
    assert b"16 x 16" in L.grl_last_error()
    assert L.grl_ssim_u8(p, p, 1, 32, 32, 4, 0, p, 1 << 20, p, None, None, None, None) == -1
    assert b"C == 1 or 3" in L.grl_last_error()
    assert L.grl_niqe_luma_u8(p, 1, 96, 96, 1, 0, p, None) == -1
    assert b"C == 3" in L.grl_last_error()


def test_forward_u8_refuses_packed_bayer_models(pkg):
    from grl_image_restoration_b200 import tiling

    cfg = pkg.configs.grl_config("small", "dm", img_size=64)
    m = pkg.GRL(input_format="rggb", **cfg)
    img = torch.zeros(1, 8, 8, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="Bayer"):
        m.forward_u8(img)
    with pytest.raises(ValueError, match="Bayer"):
        tiling.forward_tile_u8(m, img, 8, 0)


def test_u8_surface_needs_cuda_tensors(pkg):
    from grl_image_restoration_b200 import functional as K, metrics

    img = torch.zeros(1, 16, 16, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA"):
        K.u8_to_f32(img)
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.psnr_fused(img, img)
    with pytest.raises(RuntimeError, match="CUDA"):
        pkg.GRL(**pkg.configs.micro_config()).forward_u8(img)
