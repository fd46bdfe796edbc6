"""The fused SSIM kernel (ssim_tile_kernel in csrc/metric.cu behind grl_ssim_f32) stage by stage: its map against the
host computation of the same closed form (grl_ssim_host) bit for bit, its scores against the host's, the reference's
(tests/golden/ssim.npz) and the torch-op definition metrics.ssim, and metrics.validation_metrics_fused against
metrics.validation_metrics."""
import os

import numpy as np
import pytest
import torch
from torch.utils._pytree import tree_leaves
from torch.utils._python_dispatch import TorchDispatchMode

from metric_cases import SSIM_CASES, SSIM_GOLDEN, SSIM_SCORE_GATE, golden_pair, golden_scores, host_ssim

pytestmark = pytest.mark.gpu
METRICS_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz")


def device_ssim(a, b, border=0):
    """grl_ssim_f32 with both map outputs on contiguous CUDA fp32 images -> (ssim_rgb, ssim_y, map_rgb, map_y)."""
    from grl_image_restoration_b200 import capi

    B, C, H, W = a.shape
    h, w = H - 2 * border, W - 2 * border
    f64 = dict(device=a.device, dtype=torch.float64)
    ws = torch.empty(max(capi.lib().grl_ssim_workspace(B, C, H, W, border) // 8, 1), **f64)
    out, m, my = torch.empty(2, B, **f64), torch.full((B, C, h, w), -1.0, **f64), torch.full((B, 1, h, w), -1.0, **f64)
    capi.check(capi.lib().grl_ssim_f32(capi.ptr(a), capi.ptr(b), B, C, H, W, border, capi.ptr(ws), ws.numel() * 8,
                                       capi.ptr(out[0]), capi.ptr(out[1]), capi.ptr(m), capi.ptr(my) if C == 3 else None,
                                       capi.stream()))
    return out[0], out[1], m, my


@pytest.mark.parametrize("case", SSIM_CASES)
def test_kernel_against_host_and_reference(pkg, device, case):
    from grl_image_restoration_b200 import metrics

    g = np.load(SSIM_GOLDEN)
    restored, target = golden_pair(g, case)
    border = int(g[f"{case}_border"])
    hs, hsy, hm, hmy = host_ssim(restored, target, border, maps=True)
    a, b = restored.to(device), target.to(device)
    keep = a.clone()
    s, sy, m, my = device_ssim(a, b, border)
    assert torch.equal(a, keep), "the metric must not modify the images it is given"
    assert m.cpu().numpy().tobytes() == hm.tobytes(), "SSIM map differs from the host computation of the same closed form"
    if restored.shape[1] == 3:
        assert my.cpu().numpy().tobytes() == hmy.tobytes()
    assert np.abs(s.cpu().numpy() - hs).max() <= 1e-13 and np.abs(sy.cpu().numpy() - hsy).max() <= 1e-13
    want, want_y = golden_scores(g, case)
    assert np.abs(s.cpu().numpy() - want).max() <= SSIM_SCORE_GATE and np.abs(sy.cpu().numpy() - want_y).max() <= SSIM_SCORE_GATE
    f, fy = metrics.ssim_fused(a, b, border)  # the public call: same kernel, no map output
    assert torch.equal(f, s) and torch.equal(fy, sy)
    if restored.shape[1] == 1:
        assert torch.equal(fy, f)


@pytest.mark.parametrize("shape,border", [((2, 3, 16, 16), 0), ((3, 3, 67, 45), 0), ((2, 1, 40, 33), 2), ((2, 3, 256, 256), 4),
                                          ((1, 3, 1024, 1024), 4), ((1, 3, 2040, 1356), 0), ((1, 1, 1356, 2040), 0)])
def test_fused_ssim_vs_torch_ops(pkg, device, shape, border):
    from grl_image_restoration_b200 import metrics

    g = torch.Generator().manual_seed(21)
    b = torch.rand(shape, generator=g).to(device)
    a = (b + 0.1 * torch.randn(shape, generator=g).to(device)) * 1.2 - 0.1  # values outside [0, 1] exercise the clamp
    s, sy = metrics.ssim_fused(a, b, border)
    assert s.dtype == torch.float64 and s.shape == (shape[0],)
    # the torch-op definition on the CPU: its fp32 convolutions do not depend on the device library's math mode there
    assert (s.cpu() - metrics.ssim(a.cpu(), b.cpu(), border)).abs().max().item() <= SSIM_SCORE_GATE
    if shape[1] == 3:
        assert (sy.cpu() - metrics.ssim(a.cpu(), b.cpu(), border, "y")).abs().max().item() <= SSIM_SCORE_GATE
    else:
        assert torch.equal(sy, s)
    s2, sy2 = metrics.ssim_fused(a, b, border)
    assert torch.equal(s, s2) and torch.equal(sy, sy2)  # fixed summation order: bit-identical run to run
    for i in range(shape[0]):  # an image scores the same alone and in a batch
        si, syi = metrics.ssim_fused(a[i:i + 1], b[i:i + 1], border)
        assert torch.equal(si, s[i:i + 1]) and torch.equal(syi, sy[i:i + 1])
    same, same_y = metrics.ssim_fused(b, b.clone(), border)
    assert (same == 1.0).all() and (same_y == 1.0).all()


def test_input_conversion(pkg, device):
    """Non-contiguous and fp16 inputs are converted as psnrb_fused converts them, and left untouched."""
    from grl_image_restoration_b200 import metrics

    g = torch.Generator().manual_seed(22)
    b = torch.rand(2, 3, 48, 40, generator=g).to(device)
    a = (b + 0.05 * torch.randn(2, 3, 48, 40, generator=g).to(device)).clamp(0, 1)
    want = metrics.ssim_fused(a, b, 2)
    nc_a = a.permute(0, 1, 3, 2).contiguous().permute(0, 1, 3, 2)
    assert not nc_a.is_contiguous()
    got = metrics.ssim_fused(nc_a, b, 2)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    ha, hb = a.half(), b.half()
    keep = ha.clone()
    got = metrics.ssim_fused(ha, hb, 2)
    want = metrics.ssim_fused(ha.float(), hb.float(), 2)
    assert torch.equal(ha, keep) and torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    with pytest.raises(RuntimeError, match="one shape"):
        metrics.ssim_fused(a, b[:, :, :-1], 0)
    with pytest.raises(RuntimeError, match="C == 1 or 3"):
        metrics.ssim_fused(a[:, :2], b[:, :2], 0)
    with pytest.raises(RuntimeError, match="border"):
        metrics.ssim_fused(a, b, 20)


@pytest.mark.parametrize("case,is_sr", [("sr_x4", True), ("dn", False)])
def test_validation_metrics_fused(pkg, device, case, is_sr):
    from grl_image_restoration_b200 import metrics

    g = np.load(METRICS_GOLDEN)
    restored, target = torch.from_numpy(g[f"{case}_restored"]).to(device), torch.from_numpy(g[f"{case}_target"]).to(device)
    scale = int(g[f"{case}_border"]) or 1
    got = metrics.validation_metrics_fused(restored, target, scale=scale, is_sr=is_sr)
    want = metrics.validation_metrics(restored.cpu(), target.cpu(), scale=scale, is_sr=is_sr)  # the torch-op definitions
    assert list(got) == list(want)
    for name, tol in (("psnr", 1e-4), ("psnr_y", 1e-4), ("ssim", SSIM_SCORE_GATE), ("ssim_y", SSIM_SCORE_GATE)):
        assert got[name].shape == want[name].shape
        assert (got[name].double().cpu() - want[name].double()).abs().max().item() <= tol, name
        assert (got[name].double().cpu() - torch.from_numpy(g[f"{case}_{name}"]).double()).abs().max().item() <= tol, name


class Recorder:
    """Stands in for capi.lib(): records the name of every entry point called, forwards every call to the library."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*args):
            self.calls.append(name)
            return fn(*args)

        return call


class ImageOps(TorchDispatchMode):
    """Records every torch operator that takes one of the watched tensors' storage as an argument."""

    def __init__(self, *watched):
        super().__init__()
        self.ptrs, self.ops = {t.untyped_storage().data_ptr() for t in watched}, []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        flat = tree_leaves((args, kwargs or {}))
        if any(isinstance(t, torch.Tensor) and t.untyped_storage().data_ptr() in self.ptrs for t in flat):
            self.ops.append(str(func))
        return func(*args, **(kwargs or {}))


def test_validation_metrics_fused_is_two_library_calls(pkg, device, monkeypatch):
    """The C-ABI calls of validation_metrics_fused are the two kernels' entry points and the workspace query, four kernel
    launches in all, and no torch operator touches either image."""
    from grl_image_restoration_b200 import capi, metrics

    g = torch.Generator().manual_seed(23)
    a, b = torch.rand(2, 3, 64, 48, generator=g).to(device), torch.rand(2, 3, 64, 48, generator=g).to(device)
    lib = capi.lib()
    rec = Recorder(lib)
    monkeypatch.setattr(capi, "lib", lambda: rec)
    before = lib.grl_launch_count()
    with ImageOps(a, b) as ops:
        out = metrics.validation_metrics_fused(a, b, scale=4, is_sr=True)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert rec.calls == ["grl_psnr_f32", "grl_ssim_workspace", "grl_ssim_f32"]
    assert lib.grl_launch_count() - before == 4  # psnr_sse + psnr_finalize, ssim_tile + ssim_finalize
    assert ops.ops == [], ops.ops
    assert sorted(out) == ["psnr", "psnr_y", "ssim", "ssim_y"]
