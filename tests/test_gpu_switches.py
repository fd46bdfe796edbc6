"""The anchor_proj_type / anchor_one_stage / conv_type switches on the GPU: the anchor gather and max pooling bit for
bit; every GEMM / conv launch the switches add or change, from tc.gemm_launches and modules.f32_launches of each
switched micro architecture, against float64 through the launch-path gates of test_gpu_tc_gemm.py and
test_gpu_f32_paths.py; and switched networks against the reference's goldens (fp32 <= 1e-3 max-abs; fp16 / bf16 by
PSNR), with their routed biases, tiled, list and CUDA-graph forwards."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import f32_cases as F32
import gemm_cases as G
import grl_oracle as O
import switch_cases as sw
from support import bound_ratio
from engine_oracle import forward_tile

pytestmark = pytest.mark.gpu

CASES = sw.switch_cases()["cases"]
VALID = [n for n, c in CASES.items() if c["valid"]]


def _load(name):
    z = np.load(os.path.join(sw.GOLD, f"switches_{name}.npz"))
    return torch.from_numpy(z["x"]), torch.from_numpy(z["y"])


def _model(pkg, oracle, name, device, precision):
    c = CASES[name]
    shapes = {k: list(v.shape) for k, v in pkg.GRL(**c["kwargs"]).state_dict().items()
              if k.split("_")[0] not in ("table", "index", "mask")}
    m = pkg.GRL(**c["kwargs"])
    m.load_state_dict(sw.synth_state_dict(oracle, c["kwargs"], shapes), strict=False)
    m = m.to(device).eval()
    m.set_precision(precision)
    return m


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("k,stride,pad,row_major", [(3, 2, 1, True), (5, 4, 2, True), (2, 2, 0, False), (4, 3, 2, True)])
def test_anchor_gather_bit_exact(pkg, device, dtype, k, stride, pad, row_major):
    from grl_image_restoration_b200 import functional as K

    B, H, W, C, ld = 2, 13, 11, 5, 8
    x = torch.randn(B, H, W, ld, device=device).to(dtype)
    Ho, Wo = K.gather_size(H, W, k, stride, pad)
    ldy = k * k * C + 7
    got = K.anchor_gather(x, C, k, stride, pad, row_major, ldy)
    cols = F.unfold(x[..., :C].permute(0, 3, 1, 2).double(), k, padding=pad, stride=stride).view(B, C, k, k, -1)
    cols = (cols.permute(0, 4, 2, 3, 1) if row_major else cols.permute(0, 4, 3, 2, 1)).reshape(B * Ho * Wo, k * k * C)
    want = torch.zeros(B * Ho * Wo, ldy, dtype=dtype, device=device)
    want[:, : k * k * C] = cols.to(dtype)
    assert got.dtype == dtype and torch.equal(got.view(torch.int16 if dtype != torch.float32 else torch.int32),
                                              want.view(torch.int16 if dtype != torch.float32 else torch.int32))
    # PatchMerging's order by plain indexing (mixed_attn_block.py:702-706)
    if (k, stride, pad, row_major) == (2, 2, 0, False):
        u = x[:, : 2 * Ho, : 2 * Wo, :C]
        ref = torch.cat([u[:, 0::2, 0::2], u[:, 1::2, 0::2], u[:, 0::2, 1::2], u[:, 1::2, 1::2]], -1)
        assert torch.equal(got[:, : 4 * C].reshape(B, Ho, Wo, 4 * C), ref)


@pytest.mark.parametrize("df", [1, 2, 4])
def test_maxpool_bit_exact(pkg, device, df):
    from grl_image_restoration_b200 import functional as K, tc

    B, H, W, C = 2, 16, 24, 36
    x = torch.randn(B, H, W, C, device=device)
    got = K.pool(x, df, "maxpool")
    want = F.max_pool2d(x.permute(0, 3, 1, 2), df, df).permute(0, 2, 3, 1)
    assert torch.equal(got, want)
    for fmt in (0, 1):
        x16 = tc.pack_rows(x, 64, fmt)
        out = torch.empty(B, H // df, W // df, 64, device=device, dtype=tc.DTYPE[fmt])
        tc.maxpool16(x16, out, df)
        assert torch.equal(out, tc.pack_rows(want.contiguous(), 64, fmt))  # max of the rounded == rounded max


@pytest.mark.parametrize("name", VALID)
def test_fp32_network_matches_reference(pkg, oracle, device, name):
    x, y = _load(name)
    m = _model(pkg, oracle, name, device, "fp32")
    got = m(x.to(device)).cpu()
    err = (got - y).abs().max().item()
    print(f"\n[switches fp32] {name}: max |out - reference| = {err:.3e}")
    assert err <= 1e-3


# the launches the switches add or change: the anchor projections (every stage) and the stage / body convs
SWITCHED = re.compile(r"(^stage0\.block0\.anchor(\.\d+)?$)|(^stage0\.conv(\.\d)?$)|(^conv_after_body(\.\d)?$)")
LISTING_SHAPE = (1, 3, 27, 21)


def _listing_model(pkg, name, precision):
    m = pkg.GRL(**CASES[name]["kwargs"])
    m.set_precision(precision)
    return m


@pytest.mark.parametrize("fmt", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", VALID)
def test_switched_gemm_launches(pkg, device, name, fmt):
    """Each distinct tensor-core GEMM / conv launch of the switched layers (anchor stages with a gathered K and the
    bias or QKV epilogue, 1x1 / per-pixel Linear stage convs with residual and fp32 rows, the 3conv convs at the padded
    C/4 width): gemm_cases' operands, buffer checks and gates against grl_oracle.gemm_launch_reference."""
    from grl_image_restoration_b200 import tc

    if tc.capi.lib().grl_device_ok() != 1:
        pytest.skip("wgmma path needs sm_90")
    seen = {}
    for ln in tc.gemm_launches(_listing_model(pkg, name, "fp16"), LISTING_SHAPE):
        if SWITCHED.match(ln.name):
            a = ln.args
            seen.setdefault((G.path(ln), a["kpad"], a["npad"], a["taps"]), ln)
    assert seen
    for i, ln in enumerate(seen.values()):
        run = G.instantiate(tc, ln, fmt, device, seed=1000 + 10 * VALID.index(name) + i)
        assert run.sig == G.path(ln)
        q = tc.gemm_path(ln)
        tc.gemm(**run.kw)
        torch.cuda.synchronize()
        G.check_buffers(tc, run, fmt, q.epi_mode)
        got = {k: v for k, (v, _) in run.bufs.items()}
        o = dict(run.ops)
        ref = O.gemm_launch_reference(o.pop("x"), o.pop("w"), o.pop("bias"), bn=q.bn, **o)
        res = G.evaluate(tc, run, got, ref, fmt)
        print(f"\n[{tc.DTYPE[fmt]}] {name} {ln.name} kpad {ln.args['kpad']} npad {ln.args['npad']} epi {ln.args['epi']}: "
              f"{ {k: v[0] for k, v in res.items()} }")
        assert all(ok for _, ok in res.values()), (ln.name, res)


@pytest.mark.parametrize("name", VALID)
def test_switched_f32_launches(pkg, device, name):
    """Each distinct fp32 GEMM / conv launch of the switched layers (the gathered anchor GEMMs, PatchMerging's without
    bias; the 1x1 / Linear stage convs with residual; the 3conv convs) against float64, inside f32_cases.gemm_bound."""
    from grl_image_restoration_b200 import functional as K, modules

    seen = {}
    for g in modules.f32_launches(_listing_model(pkg, name, "fp32"), LISTING_SHAPE):
        if SWITCHED.match(g.name):
            seen.setdefault((F32.gemm_path(g), g.K, g.N), g)
    assert seen
    Bn, Hc, Wc, M = 2, 13, 21, 200
    for i, c in enumerate(seen.values()):
        gen = torch.Generator().manual_seed(2000 + 10 * VALID.index(name) + i)
        cin = c.K // 9 if c.conv else c.K
        rows = Bn * Hc * Wc if c.conv else M
        x = torch.randn(rows, cin, generator=gen) * torch.exp2(torch.rand(rows, 1, generator=gen) * 3 - 2)
        w = torch.randn(c.N, c.K, generator=gen) * c.K ** -0.5
        b = torch.randn(c.N, generator=gen) * 0.5 if c.bias else None
        r = torch.randn(rows, c.N, generator=gen) if c.res else None
        x, w = x.to(device), w.to(device)
        b = None if b is None else b.to(device)
        r = None if r is None else r.to(device)
        if c.conv:
            xi = x.view(Bn, Hc, Wc, cin)
            got = K.conv3x3(xi, w, b, c.act, c.slope, None if r is None else r.view(Bn, Hc, Wc, c.N)).view(rows, c.N)
            A = F32.im2col(xi.double())
        else:
            got = K.linear(x, w, b, c.act, c.slope, r)
            A = x.double()
        torch.cuda.synchronize()
        b64 = torch.zeros(c.N, device=device, dtype=torch.float64) if b is None else b.double()
        r64 = None if r is None else r.double()
        y64 = O.gemm_launch_reference(A, w.double(), b64, act=c.act, slope=c.slope, n_res=c.N, res=r64)["y"]
        bound, _ = F32.gemm_bound(A, w.double(), b64, c.act, c.slope, r64)
        ratio = bound_ratio(got, y64, bound)
        print(f"\n[fp32 gemm] {name} {c.name} K {c.K} N {c.N} act {c.act} bias {c.bias} res {c.res}: "
              f"worst error / bound {ratio:.3f}")
        assert ratio <= 1.0, (c, ratio)


# parameters whose loss the routed goldens must notice: new Linear biases (zero in the "init" style) and conv biases
ROUTED = {
    "linear": ("conv_after_body.bias", "layers.0.conv.bias"),
    "maxpool_df2": ("layers.0.blocks.1.attn.anchor.body.0.reduction.bias",),
    "conv2d_ms_df4": ("layers.0.blocks.2.attn.anchor.body.1.bias",),
    "3conv": ("layers.0.conv.2.bias",),
}


@pytest.mark.parametrize("name", list(ROUTED))
def test_routed_biases_reach_the_output(pkg, oracle, device, name):
    """Zeroing one switched bias moves the fp32 output off the golden by more than the 1e-3 gate."""
    x, y = _load(name)
    for pname in ROUTED[name]:
        m = _model(pkg, oracle, name, device, "fp32")
        with torch.no_grad():
            m.get_parameter(pname).zero_()
        err = (m(x.to(device)).cpu() - y).abs().max().item()
        print(f"\n[routed] {name}: {pname} zeroed -> max |out - reference| = {err:.3e}")
        assert err > 1e-3, pname


def _psnr(a, b):
    return (-10 * torch.log10(((a - b) ** 2).mean())).item()


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("name", VALID)
def test_tensor_core_network_matches_reference(pkg, oracle, device, name, precision):
    """PSNR of the tensor-core output against the reference's, peak 1.  On an H100 these routed micro networks measured
    79.9-93.9 dB with fp16 operands and 62.8-76.0 dB with bf16; the gates keep about 5 dB of that margin."""
    x, y = _load(name)
    m = _model(pkg, oracle, name, device, precision)
    got = m(x.to(device)).cpu()
    p = _psnr(got, y)
    print(f"\n[switches {precision}] {name}: PSNR vs reference {p:.2f} dB")
    assert p >= (75.0 if precision == "fp16" else 58.0)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_tile_list_and_graph_forwards_agree(pkg, oracle, device, precision):
    from grl_image_restoration_b200 import tiling

    m = _model(pkg, oracle, "conv2d_ms_df4_3conv", device, precision)
    g = torch.Generator().manual_seed(5)
    imgs = [torch.rand(3, h, w, generator=g).to(device) for h, w in ((27, 21), (32, 40), (27, 21))]
    plain = [m(i[None])[0] for i in imgs]
    for a, b in zip(m.forward_list(imgs), plain):
        assert torch.equal(a, b)
    x = imgs[1][None]
    tiled = tiling.forward_tile(m, x, 16, 4, max_batch=5)
    seq = forward_tile(lambda t: m(t).cpu(), x, 16, 4, m.upscale)
    torch.testing.assert_close(tiled.cpu(), seq, rtol=0, atol=1e-5 if precision == "fp32" else 2e-3)
    if precision != "fp32":
        m.use_cuda_graph = True
        for _ in range(3):
            assert torch.equal(m(x), plain[1][None])
