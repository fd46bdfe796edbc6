"""8-bit images on the GPU: the conversion kernels (csrc/image_u8.cu) bit-exact against the torch formulas of the
datasets' to_tensor and the validation step's tensor_round; GRL.forward_u8 and tiling.forward_tile_u8 equal to the torch
composition around forward_rgb / forward_tile element for element; every metric on 8-bit images equal to the same
metric on u8_to_f32 of them, bit for bit.

The reference side of every k / 255 below is computed on the CPU, where the datasets' to_tensor runs: torch on a CUDA
tensor divides by a Python scalar as a multiply by its reciprocal, which is 1 ulp off the division for 126 of the 256
bytes (the metrics do not see it: both round back to the same byte)."""
import os

import numpy as np
import pytest
import torch

from engine_oracle import to_tensor
from support import micro, round8_ref, same_bits

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def random_u8(shape, seed, device):
    img = torch.randint(0, 256, shape, dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))
    ends = torch.tensor([255, 0], dtype=torch.uint8)
    img.view(-1)[: min(2, img.numel())] = ends[: min(2, img.numel())]
    return img.to(device)


SIZES = [(1, 1), (17, 33), (257, 130)]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("C", [1, 3, 6])
@pytest.mark.parametrize("H,W", SIZES)
def test_u8_to_f32_bit_exact(pkg, device, B, C, H, W):
    from grl_image_restoration_b200 import functional as K

    img = random_u8((B, H, W, C), B * 1000 + C * 100 + H, device)
    y = K.u8_to_f32(img)
    assert y.dtype == torch.float32 and y.shape == (B, C, H, W) and y.is_contiguous()
    assert torch.equal(y.cpu(), to_tensor(img))
    # a non-contiguous input is read as its values
    assert torch.equal(K.u8_to_f32(img.transpose(1, 2).contiguous().transpose(1, 2)), y)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("C", [1, 3, 6])
@pytest.mark.parametrize("H,W", SIZES)
def test_f32_to_u8_bit_exact(pkg, device, B, C, H, W):
    from grl_image_restoration_b200 import functional as K

    g = torch.Generator().manual_seed(B * 1000 + C * 100 + W)
    v = torch.rand(B, C, H, W, generator=g) * 1.4 - 0.2
    flat = v.view(-1)
    k = torch.arange(255, dtype=torch.float32)
    special = torch.cat([(k + 0.5) / 255, torch.tensor([0.0, -0.0, 1.0, 1.0000001, -1e-8, 1e30, -1e30, float("inf"),
                                                        float("-inf"), float("nan")])])
    n = min(flat.numel(), special.numel())
    flat[:n] = special[:n]
    out = K.f32_to_u8(v.to(device))
    assert out.dtype == torch.uint8 and out.shape == (B, H, W, C) and out.is_contiguous()
    out = out.cpu()
    nan = v.isnan().permute(0, 2, 3, 1)
    want = round8_ref(v)
    assert torch.equal(out[~nan], want[~nan])
    assert (out[nan] == 0).all()
    # round trip
    img = random_u8((B, H, W, C), W, device)
    assert torch.equal(K.f32_to_u8(K.u8_to_f32(img)), img)


def test_conversions_reject_bad_input(pkg, device):
    from grl_image_restoration_b200 import functional as K

    with pytest.raises(RuntimeError, match="uint8"):
        K.u8_to_f32(torch.zeros(1, 4, 4, 3, device=device))
    with pytest.raises(RuntimeError, match="1 <= C <= 8"):
        K.u8_to_f32(torch.zeros(1, 4, 4, 9, dtype=torch.uint8, device=device))
    with pytest.raises(RuntimeError, match="float32"):
        K.f32_to_u8(torch.zeros(1, 3, 4, 4, dtype=torch.uint8, device=device))
    with pytest.raises(RuntimeError, match="1 <= C <= 8"):
        K.f32_to_u8(torch.zeros(1, 3, 4, device=device))


# input (B, H, W) of an upscaling, a denoising and the grayscale micro config of tests/golden/cases.json
INPUTS = {"micro_cab_x2": (2, 24, 40), "micro_pad_dn": (1, 24, 40), "micro_gray": (1, 24, 24)}


@pytest.mark.parametrize("name", list(INPUTS))
@pytest.mark.parametrize("precision,ensemble,graph", [("fp32", False, False), ("fp32", True, False), ("fp16", False, False),
                                                      ("fp16", True, False), ("fp16", False, True)])
def test_forward_u8_equals_torch_composition(pkg, oracle, device, name, precision, ensemble, graph):
    m = micro(pkg, oracle, name, device, precision, self_ensemble=ensemble)
    m.use_cuda_graph = graph
    B, H, W = INPUTS[name]
    img = random_u8((B, H, W, m.in_channels), list(INPUTS).index(name), device)
    out = m.forward_u8(img)
    s = m.upscale
    assert out.dtype == torch.uint8 and out.shape == (B, H * s, W * s, m.out_channels) and out.is_contiguous()
    want = round8_ref(m.forward_rgb(to_tensor(img).to(device)))
    assert torch.equal(out, want)
    if graph:
        assert m._graphs, "the forward must have replayed a captured graph"
        assert torch.equal(m.forward_u8(img), want)
    with pytest.raises(ValueError, match="uint8 images"):
        m.forward_u8(img[..., :0])


def test_forward_tile_u8_equals_torch_composition(pkg, oracle, device):
    from grl_image_restoration_b200 import tiling

    m = micro(pkg, oracle, "micro_cab_x2", device, "fp16")
    img = random_u8((2, 40, 56, 3), 7, device)
    out = tiling.forward_tile_u8(m, img, 32, 8, max_batch=5)
    want = round8_ref(tiling.forward_tile(m, to_tensor(img).to(device), 32, 8, max_batch=5))
    assert out.shape == (2, 80, 112, 3) and out.dtype == torch.uint8
    assert torch.equal(out, want)


def pair(shape_hwc, seed, device):
    """Two related 8-bit images (a restoration and its target) and their k / 255 planes from u8_to_f32."""
    from grl_image_restoration_b200 import functional as K

    b = random_u8(shape_hwc, seed, device)
    noise = torch.randint(-12, 13, shape_hwc, generator=torch.Generator().manual_seed(seed + 1)).to(device)
    a = (b.short() + noise).clamp(0, 255).byte()
    return a, b, K.u8_to_f32(a), K.u8_to_f32(b)


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("shape,border", [((2, 67, 93), 0), ((2, 67, 93), 4), ((1, 128, 128), 2)])
def test_psnr_and_ssim_u8_equal_f32(pkg, device, C, shape, border):
    from grl_image_restoration_b200 import metrics

    a, b, fa, fb = pair(shape + (C,), C * 10 + border, device)
    for fn in (metrics.psnr_fused, metrics.ssim_fused):
        u8, f32 = fn(a, b, border), fn(fa, fb, border)
        assert torch.equal(u8[0], f32[0]) and torch.equal(u8[1], f32[1]), fn.__name__
    vu, vf = metrics.validation_metrics_fused(a, b, scale=border, is_sr=border > 0), \
        metrics.validation_metrics_fused(fa, fb, scale=border, is_sr=border > 0)
    assert vu.keys() == vf.keys() and all(torch.equal(vu[k], vf[k]) for k in vu)


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("shape", [(2, 37, 51), (1, 32, 48), (3, 16, 23)])
def test_psnrb_u8_equals_f32(pkg, device, C, shape):
    from grl_image_restoration_b200 import metrics

    a, b, fa, fb = pair(shape + (C,), C * 100 + shape[1], device)
    u8, f32 = metrics.psnrb_fused(a, b), metrics.psnrb_fused(fa, fb)
    assert torch.equal(u8[0], f32[0]) and torch.equal(u8[1], f32[1])


@pytest.mark.parametrize("shape,border", [((2, 200, 230), 0), ((1, 205, 300), 4)])
def test_niqe_u8_equals_f32(pkg, device, shape, border):
    from grl_image_restoration_b200 import metrics

    params = dict(np.load(os.path.join(GOLD, "niqe_pris_params.npz")))
    a, _, fa, _ = pair(shape + (3,), shape[1] + border, device)
    same_bits(metrics.niqe_features(a, params, border), metrics.niqe_features(fa, params, border))
    same_bits(metrics.niqe(a, params, border), metrics.niqe(fa, params, border))
    su, sf = metrics.niqe_stages(a, params, border), metrics.niqe_stages(fa, params, border)
    for k in sf:
        same_bits(su[k], sf[k])


def test_metrics_refuse_mixed_dtypes_and_bad_shapes(pkg, device):
    from grl_image_restoration_b200 import metrics

    a, b, fa, fb = pair((1, 32, 32, 3), 3, device)
    params = dict(np.load(os.path.join(GOLD, "niqe_pris_params.npz")))
    for fn in (metrics.psnr_fused, metrics.ssim_fused, metrics.psnrb_fused):
        with pytest.raises(RuntimeError, match="two uint8 images or two float"):
            fn(a, fb)
        with pytest.raises(RuntimeError, match="two uint8 images or two float"):
            fn(fa, b)
        with pytest.raises(RuntimeError, match="one shape"):
            fn(a, b[:, :16])
    with pytest.raises(RuntimeError, match="two uint8 images or two float"):
        metrics.validation_metrics_fused(a, fb)
    four = torch.zeros(1, 32, 32, 4, dtype=torch.uint8, device=device)
    with pytest.raises(RuntimeError, match="C == 1 or 3"):
        metrics.ssim_fused(four, four)
    with pytest.raises(RuntimeError, match="C == 1 or 3"):
        metrics.psnrb_fused(four, four)
    with pytest.raises(RuntimeError, match="RGB"):
        metrics.niqe(torch.zeros(1, 3, 128, 128, dtype=torch.uint8, device=device), params)
    with pytest.raises(RuntimeError, match="96 x 96"):
        metrics.niqe(torch.zeros(1, 90, 128, 3, dtype=torch.uint8, device=device), params)
