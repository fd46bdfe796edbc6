"""Host logic of the tensor-core path (no GPU): the one-time weight packing of tc.py, checked by emulating in fp32 torch what
the kernels do with the packed operands -- the slot layout of the QKV GEMM, the ones-column of the value slots, the K-index map
of the output projection, the im2col order of the 3x3 convs and the PixelShuffle store pattern of grl_tc_gemm (ps_r) --
against the plain nn.Module arithmetic of the reference (mixed_attn_block_efficient.py:358-381, upsample.py:6-30)."""
import pytest
import torch
import torch.nn.functional as F

from support import build


@pytest.fixture(scope="module")
def tc(pkg):
    from grl_image_restoration_b200 import tc as _tc

    return _tc


def _block(pkg, oracle, **kw):
    model = build(pkg, oracle, pkg.configs.micro_config(**kw), "cpu", "fp32", style="spread", seed=3)
    return model, model.layers[0].blocks[0]


@pytest.mark.parametrize("embed_dim,heads", [(36, 2), (60, 3), (64, 1)])
def test_qkv_slot_packing(pkg, oracle, tc, embed_dim, heads):
    """x @ w_qkv^T + b_qkv read back slot by slot == the reference's qkv linear in its (half, q|k|v, head, e) order; pad
    columns are zero except the ones-column of every value slot when head_dim < 32."""
    _, blk = _block(pkg, oracle, embed_dim=embed_dim, heads=heads)
    plan = tc.BlockPlan(blk, fmt=0)
    C, c = blk.dim, blk.dim // 2
    d = c // heads
    x = torch.randn(50, C)
    xp = F.pad(x, (0, plan.cpad - C))
    y = xp @ plan.w_qkv.float().t() + plan.b_qkv  # (50, nslots * 32) as the GEMM writes it (before normalise / scale)
    w16 = blk.attn.qkv.body.weight.half().float()  # operands are rounded to fp16 by the packer
    ref = x @ w16.t() + blk.attn.qkv.body.bias     # (50, 3C): [window q k v | stripe q k v], each (head, e)
    assert plan.nslots == 6 * heads and y.shape[1] == plan.nslots * tc.SLOT
    y = y.view(50, plan.nslots, tc.SLOT)
    src = 0
    for half in range(2):
        for t in range(3):
            for head in range(heads):
                slot = half * 3 * heads + t * heads + head
                torch.testing.assert_close(y[:, slot, :d], ref[:, src:src + d], rtol=1e-5, atol=1e-5)
                pad = y[:, slot, d:]
                if d < tc.SLOT:
                    if t == 2:  # value slot: the last column is the ones-column (softmax denominator out of P V)
                        assert torch.equal(pad[:, -1], torch.ones(50)) and not pad[:, :-1].any()
                    else:
                        assert not pad.any()
                src += d
    assert src == 3 * C
    assert plan.ones_w == (d < tc.SLOT) and plan.ones_s == (d < tc.SLOT)


@pytest.mark.parametrize("embed_dim,heads", [(36, 2), (60, 3)])
def test_proj_reads_the_slot_layout(pkg, oracle, tc, embed_dim, heads):
    """The attention kernels write head h of the window (stripe) half into slot h (heads + h); w_proj's K index map makes
    `slots @ w_proj^T` equal the reference's proj(cat(window heads, stripe heads)) (mixed_attn_block_efficient.py:376-381)."""
    _, blk = _block(pkg, oracle, embed_dim=embed_dim, heads=heads)
    plan = tc.BlockPlan(blk, fmt=0)
    C, c = blk.dim, blk.dim // 2
    d = c // heads
    o = torch.randn(40, 2 * heads, d)                     # per-head attention outputs, window heads first
    slots = torch.zeros(40, plan.k_proj)
    for h in range(2 * heads):
        slots[:, h * tc.SLOT:h * tc.SLOT + d] = o[:, h]
        if d < tc.SLOT:
            slots[:, h * tc.SLOT + tc.SLOT - 1] = 1.0      # the normalised ones-column the kernel leaves there: weight must be 0
    y = slots @ plan.w_proj.float().t() + plan.b_proj
    ref = o.reshape(40, C) @ blk.attn.proj.weight.half().float().t() + blk.attn.proj.bias
    torch.testing.assert_close(y[:, :C], ref, rtol=1e-5, atol=1e-5)
    assert not y[:, C:].any()  # LayerNorm tile pad columns


def _conv_emulation(x, wpack, bias, cin_pad):
    """What the implicit-GEMM conv computes: for every pixel, K = (tap, channel) with tap = ky * 3 + kx and zero padding
    outside the image (TMA OOB fill).  x (B, H, W, cin_pad) channels-last -> (B, H, W, npad)."""
    B, H, W, _ = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    cols = torch.cat([xp[:, ky:ky + H, kx:kx + W, :] for ky in range(3) for kx in range(3)], dim=-1)  # (B,H,W,9*cin_pad)
    return cols @ wpack.float().t() + bias


def test_conv_im2col_order(pkg, tc):
    conv = torch.nn.Conv2d(5, 7, 3, 1, 1)
    with torch.no_grad():
        conv.weight.copy_(conv.weight.half().float())
    w, b = tc.pack_conv(conv, 64, 32, fmt=0)
    assert w.shape == (32, 9 * 64) and b.shape == (32,)
    x = torch.randn(2, 6, 9, 5)
    y = _conv_emulation(F.pad(x, (0, 59)), w, b, 64)
    ref = conv(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    torch.testing.assert_close(y[..., :7], ref, rtol=1e-5, atol=1e-5)
    assert not y[..., 7:].any()


@pytest.mark.parametrize("r", [2, 3, 4])
def test_pixelshuffle_store_pattern(pkg, tc, r):
    """pack_conv(ps_r=r) + the store of gemm_tc.cu (column n' = q * Cq + c of pixel (y, x) goes to pixel (y r + q / r,
    x r + q % r), channel c) == nn.PixelShuffle(r)(conv(x)) (upsample.py:6-30)."""
    cq = 8
    conv = torch.nn.Conv2d(6, cq * r * r, 3, 1, 1)
    with torch.no_grad():
        conv.weight.copy_(conv.weight.half().float())
    npad = tc.round_up(cq * r * r, 32)
    w, b = tc.pack_conv(conv, 64, npad, fmt=0, ps_r=r)
    x = torch.randn(2, 5, 4, 6)
    y = _conv_emulation(F.pad(x, (0, 58)), w, b, 64)[..., :cq * r * r]  # (B, H, W, r^2 * Cq), n' = q * Cq + c
    B, H, W = 2, 5, 4
    out = torch.zeros(B, H * r, W * r, cq)
    for q in range(r * r):
        out[:, q // r::r, q % r::r, :] = y[..., q * cq:(q + 1) * cq]
    ref = F.pixel_shuffle(conv(x.permute(0, 3, 1, 2)), r).permute(0, 2, 3, 1)
    torch.testing.assert_close(out, ref, rtol=1e-5, atol=1e-5)


def test_anchor_projection_packing(pkg, oracle, tc):
    """Anchor reduction weights land at row head * 32 + e (one slot per stripe head); mixed_attn_block.py:714-736."""
    _, blk = _block(pkg, oracle, embed_dim=36, heads=2)
    plan = tc.BlockPlan(blk, fmt=0)
    red = blk.attn.anchor.body[0].reduction
    hs, ds = 2, red.weight.shape[0] // 2
    x = torch.randn(30, blk.dim)
    y = F.pad(x, (0, plan.cpad - blk.dim)) @ plan.w_anc.float().t() + plan.b_anc
    ref = x @ red.weight.half().float().t() + red.bias
    for h in range(hs):
        torch.testing.assert_close(y[:, h * tc.SLOT:h * tc.SLOT + ds], ref[:, h * ds:(h + 1) * ds], rtol=1e-5, atol=1e-5)
        assert not y[:, h * tc.SLOT + ds:(h + 1) * tc.SLOT].any()
