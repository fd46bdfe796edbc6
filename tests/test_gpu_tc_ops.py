"""bf16 tensor-core operators (wgmma GEMM / implicit-GEMM conv) vs fp32 references evaluated on
the same bf16-rounded operands.  Tolerances are bf16-sized: these tests prove descriptor / layout / addressing
correctness (a wrong swizzle or index gives O(1) errors), the PSNR gate of the whole network is in
test_gpu_model_bf16.py."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rnd(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale


def bf(t, fmt=0):
    """Round to the 16-bit operand format under test (0 = fp16, 1 = bf16)."""
    return t.to(torch.bfloat16 if fmt else torch.float16).float()


# Both operand loaders behind grl_tc_attn are production code and are exercised by the same tests: 5 = TMA boxes of the
# token tensors (default; geometries without boxes, tails and dense V are gathered), 0 = cp.async row gathers for every
# geometry.
ATTN_VARIANTS = [5, 0]


@pytest.fixture(scope="module", params=ATTN_VARIANTS, ids=lambda v: "attn" if v is None else f"attn{v}")
def tc(pkg, device, request):
    from grl_image_restoration_b200 import capi, tc as T

    if capi.lib().grl_device_ok() != 1:
        pytest.skip("wgmma path needs sm_90")
    if request.param is None:
        yield T
        return
    prev = capi.lib().grl_tc_attn_variant(request.param)
    yield T
    capi.lib().grl_tc_attn_variant(prev)


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("M,K,N,act", [(128, 64, 64, 0), (1000, 180, 360, 1), (257, 192, 540, 0), (4096, 360, 180, 0),
                                       (130, 64, 30, 2)])
def test_gemm_bias_act(tc, device, M, K, N, act, fmt):
    x, w, b = rnd((M, K), 1), rnd((N, K), 2, K ** -0.5), rnd((N,), 3)
    kpad, npad = tc.round_up(K, 64), tc.round_up(N, 64)
    ref = F.linear(bf(x, fmt), bf(w, fmt), b)
    ref = F.gelu(ref) if act == 1 else (F.leaky_relu(ref, 0.2) if act == 2 else ref)
    x16 = tc.pack_rows(x.to(device), kpad, fmt)
    w16 = tc._pad_matrix(w.to(device), npad, kpad, fmt=fmt)
    bp = tc._pad_vector(b.to(device), npad)
    o16 = torch.empty(M, npad, device=device, dtype=tc.DTYPE[fmt])
    o32 = torch.empty(M, N, device=device, dtype=torch.float32)
    tc.gemm(x16, w16, bp, M=M, kpad=kpad, npad=npad, n_store=npad, n_real=N, out_bf16=o16, out_f32=o32, act=act, slope=0.2)
    err = (o32.cpu() - ref).abs().max().item()
    assert err <= 2e-3 * max(1.0, ref.abs().max().item()), err
    assert (o16.cpu().float()[:, :N] - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
    assert o16.cpu().float()[:, N:].abs().max().item() == 0 if npad > N else True


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("B,H,W,Cin,Cout,act", [(1, 16, 32, 64, 64, 0), (2, 24, 40, 180, 45, 1), (1, 8, 16, 45, 180, 0),
                                                (1, 37, 19, 36, 36, 2), (1, 64, 64, 180, 180, 0)])
def test_conv3x3_tc(tc, device, B, H, W, Cin, Cout, act, fmt):
    x, w, b = rnd((B, Cin, H, W), 5), rnd((Cout, Cin, 3, 3), 6, (9 * Cin) ** -0.5), rnd((Cout,), 7)
    r = rnd((B, H, W, Cout), 8)
    ref = F.conv2d(bf(x, fmt), bf(w, fmt), b, padding=1)
    ref = F.gelu(ref) if act == 1 else (F.leaky_relu(ref, 0.01) if act == 2 else ref)
    ref = ref.permute(0, 2, 3, 1) + r
    cin_pad, npad = tc.round_up(Cin, 64), tc.round_up(Cout, 64)
    conv = torch.nn.Conv2d(Cin, Cout, 3, 1, 1)
    conv.weight.data.copy_(w), conv.bias.data.copy_(b)
    conv = conv.to(device)
    wp, bp = tc.pack_conv(conv, cin_pad, npad, fmt)
    x16 = tc.pack_rows(x.permute(0, 2, 3, 1).contiguous().to(device), cin_pad, fmt)
    o32 = torch.empty(B, H, W, Cout, device=device, dtype=torch.float32)
    o16 = torch.empty(B, H, W, npad, device=device, dtype=tc.DTYPE[fmt])
    tc.conv3x3(x16, wp, bp, cin_pad, npad, n_store=npad, n_real=Cout, act=act, slope=0.01, out_bf16=o16, out_f32=o32,
               res_f32=r.to(device))
    err = (o32.cpu() - ref).abs().max().item()
    assert err <= 3e-3 * max(1.0, ref.abs().max().item()), err
    assert (o16.cpu().float()[..., :Cout] - ref).abs().max().item() <= 3e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("fmt", [0, 1])
def test_gemm_qkv_epilogue(tc, device, fmt):
    M, K, slots = 300, 180, 6
    x, w, b = rnd((M, K), 11), rnd((slots * 30, K), 12, K ** -0.5), rnd((slots * 30,), 13)
    scale = torch.tensor([14.4, 1.0, 0.0, 3.3, 1.0, 0.0])
    rmap = [s * 32 + e for s in range(slots) for e in range(30)]
    w16 = tc._pad_matrix(w.to(device), slots * 32, 192, row_map=rmap, fmt=fmt)
    bp = tc._pad_vector(b.to(device), slots * 32, rmap)
    out = torch.empty(M, slots * 32, device=device, dtype=tc.DTYPE[fmt])
    tc.gemm(tc.pack_rows(x.to(device), 192, fmt), w16, bp, M=M, kpad=192, npad=slots * 32, epi=tc.EPI_QKV,
            n_store=slots * 32, out_bf16=out, slot_scale=scale.to(device))
    y = F.linear(bf(x, fmt), bf(w, fmt), b).view(M, slots, 30)
    ref = torch.where(scale.view(1, slots, 1) > 0, F.normalize(y, dim=-1) * scale.view(1, slots, 1), y)
    got = out.cpu().float().view(M, slots, 32)
    assert got[..., 30:].abs().max().item() == 0
    assert (got[..., :30] - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("C,cab", [(180, True), (64, False), (128, False), (36, True)])
def test_gemm_layernorm_epilogue(tc, device, C, cab, fmt):
    M, K, L = 515, 192, 103
    x, w, b = rnd((M, K), 21), rnd((C, K), 22, K ** -0.5), rnd((C,), 23)
    res, g, be = rnd((M, C), 24), rnd((C,), 25) + 1.0, rnd((C,), 26)
    cy, gate = rnd((M, C), 27), torch.sigmoid(rnd((M // L, C), 28))
    n_ln = 64 if C <= 64 else 128 if C <= 128 else 192
    cpad = tc.round_up(C, 64)
    ref = res + 0.5 * F.layer_norm(F.linear(bf(x, fmt), bf(w, fmt), b), (C,), g, be, 1e-5)
    kw = {}
    if cab:
        cy16 = tc.pack_rows(cy.to(device), cpad, fmt)
        ref = ref + bf(cy, fmt) * gate.repeat_interleave(L, 0)
        kw = dict(cab_y=cy16, cab_gate=gate.to(device))
    o32 = torch.empty(M, C, device=device, dtype=torch.float32)
    o16 = torch.empty(M, cpad, device=device, dtype=tc.DTYPE[fmt])
    tc.gemm(tc.pack_rows(x.to(device), K, fmt), tc._pad_matrix(w.to(device), n_ln, K, fmt=fmt), tc._pad_vector(b.to(device), n_ln), M=M,
            kpad=K, npad=n_ln, epi=tc.EPI_LN, n_store=n_ln, n_real=C, out_bf16=o16, out_f32=o32, res_f32=res.to(device),
            C=C, gamma=g.to(device), beta=be.to(device), eps=1e-5, res_scale=0.5, L=L, **kw)
    assert (o32.cpu() - ref).abs().max().item() <= 5e-3
    # the 16-bit copy adds its own rounding: half an ulp of bf16 (8 significant bits) is up to 2^-8 |ref|, which the fp16
    # bound of 5e-2 does not cover at |ref| > 12
    tol16 = 5e-2 if fmt == 0 else 5e-2 + 2.0 ** -8 * ref.abs().max().item()
    assert (o16.cpu().float()[:, :C] - ref).abs().max().item() <= tol16
    if cpad > C:
        assert o16.cpu().float()[:, C:].abs().max().item() == 0
