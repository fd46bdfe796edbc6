"""Exact contracts of the small kernels around the tensor-core GEMM and attention: operand packing, the fused network
head, anchor pooling, the CAB channel gate, the per-block attention constants (slot scales, 4-copy bias table) and the
two store patterns of the conv epilogue (PixelShuffle, NCHW tail).  Every kernel is compared with a plain torch /
float64 reference of the same operation; the two store tests compare the fused store with the plain store of the same
launch, since only the destination address differs.  Shapes are deliberately not multiples of the tiles (conv tiles are
8 x 16 pixels, row tiles 128) and every test runs both 16-bit operand formats (fmt 0 = fp16, 1 = bf16)."""
import math

import pytest
import torch
import torch.nn.functional as F

from grl_oracle import LN100_F32, channel_gate_reference, to16
from support import FMTS, same_bits

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # fp32 unit roundoff
GRL_ERR_WORKSPACE = -3


@pytest.fixture(scope="module")
def tc(pkg, device):
    from grl_image_restoration_b200 import capi, tc as T

    if capi.lib().grl_device_ok() != 1:
        pytest.skip("wgmma path needs sm_90")
    return T


def capi():
    from grl_image_restoration_b200 import capi as C

    return C


def dt(fmt):
    return torch.bfloat16 if fmt else torch.float16


def ulp16(x, fmt):
    """One unit in the last place of the 16-bit format at |x| (subnormal floor included)."""
    mant, emin = (8, -126) if fmt else (11, -14)
    e = torch.floor(torch.log2(x.abs().double().clamp_min(2.0 ** emin)))
    return torch.pow(2.0, e - (mant - 1))


def edge_values(fmt):
    """fp32 inputs at the edges of the 16-bit conversion: signed zeros, subnormals of the target format, exact
    round-to-nearest-even ties (built from bit patterns) on both sides of an even / odd neighbour, values above the fp16
    maximum, infinities and NaN."""
    g = torch.Generator().manual_seed(5)
    vals = [0.0, -0.0, 1.0, -1.0, 65504.0, -65504.0, 65519.0, 65520.0, -65520.0, 65536.0, 1e5, -3e38, 3.4e38,
            float("inf"), float("-inf"), float("nan")]
    out = [torch.tensor(vals)]
    if fmt == 0:
        # fp16 subnormals k 2^-24 and ties (k + 1/2) 2^-24, normals and the ties between them
        k = torch.randint(1, 1024, (64,), generator=g).double()
        out += [k * 2.0 ** -24, -(k + 0.5) * 2.0 ** -24, (k + 0.5) * 2.0 ** -24, torch.tensor([2.0 ** -25, 2.0 ** -26])]
        bits = torch.randint(0x0400, 0x7BFF, (256,), generator=g, dtype=torch.int32).to(torch.int16)
        lo = bits.view(torch.float16).double()
        hi = (bits + 1).view(torch.float16).double()
        out += [(lo + hi) / 2, -(lo + hi) / 2, torch.tensor([65504.0 + 8.0, 65504.0 + 16.0])]  # 65512 is the tie to inf
    else:
        # bf16 subnormals are fp32 subnormals with 16 zero low bits; ties have low bits 0x8000
        hi16 = torch.randint(1, 0x7F7F, (256,), generator=g, dtype=torch.int32)
        sub16 = torch.randint(1, 0x0080, (64,), generator=g, dtype=torch.int32)
        for h in (hi16, sub16):
            for low in (0x0000, 0x8000, 0x7FFF, 0x8001):
                b = (h << 16) | low
                f = b.view(torch.float32).double()
                out += [f, -f]
    return torch.cat([o.double() for o in out]).float()


@pytest.mark.parametrize("fmt", FMTS)
def test_pack16_edge_values_bit_exact(tc, device, fmt):
    """grl_tc_pack16: fp32 -> 16-bit is round-to-nearest-even, bit-exact against torch.  fp16 saturates (+-inf and
    everything >= 65520 in magnitude become +-65504, DESIGN.md); NaN stays NaN, which is what the PTX ISA specifies for
    cvt.rn.satfinite (and for the bf16 convert).  Zeros fill [C, Cpad)."""
    v = edge_values(fmt)
    C, Cpad = 40, 64
    M = (v.numel() + C - 1) // C
    x = torch.zeros(M * C)
    x[: v.numel()] = v
    x = x.view(M, C)
    y = tc.pack_rows(x.to(device), Cpad, fmt).cpu()
    same_bits(y[:, :C], to16(x, fmt))
    assert not y[:, C:].float().any() and not torch.signbit(y[:, C:].float()).any()
    if fmt == 0:
        yf = y.float()
        assert yf[~torch.isnan(yf)].abs().max().item() == 65504.0  # never inf
    assert torch.isnan(y[:, :C].float()).sum().item() == torch.isnan(x).sum().item() == 1


@pytest.mark.parametrize("fmt", FMTS)
def test_pack16_strided_source_and_empty(tc, device, fmt):
    """A strided fp32 source (ldx > C) packs row by row; a ragged row count (M not a multiple of 128) and M = 0 work."""
    M, C, ldx, Cpad = 301, 36, 50, 64
    src = torch.randn(M, ldx, generator=torch.Generator().manual_seed(3)) * 300.0
    src_d = src.to(device)
    y = torch.full((M, Cpad), float("nan"), device=device, dtype=dt(fmt))
    C_ = capi()
    C_.check(C_.lib().grl_tc_pack16(C_.ptr(src_d), ldx, C_.ptr(y), M, C, Cpad, fmt, C_.stream()))
    y = y.cpu()
    same_bits(y[:, :C], to16(src[:, :C], fmt))
    assert not y[:, C:].float().any()
    e = tc.pack_rows(torch.empty(0, C, device=device), Cpad, fmt)
    torch.cuda.synchronize()
    assert e.shape == (0, Cpad)


@pytest.mark.parametrize("fmt", FMTS)
def test_unpack16_every_bit_pattern(tc, device, fmt):
    """grl_tc_unpack16: 16-bit -> fp32 is exact for every one of the 65536 bit patterns (zeros, subnormals, infinities,
    NaN), reading columns [x_off, x_off + C) of rows of pitch ldx into rows of pitch ldy; the columns of y past C and the
    rows past M are not written."""
    allbits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    C, ldx, x_off, ldy = 100, 136, 24, 112
    M = allbits.numel() // C + 1  # 656 rows: not a multiple of anything the kernel tiles by
    x = torch.zeros(M, ldx, dtype=torch.int16)
    flat = torch.zeros(M * C, dtype=torch.int16)
    flat[: allbits.numel()] = allbits
    x[:, x_off:x_off + C] = flat.view(M, C)
    x16 = x.view(dt(fmt)).to(device)
    y = torch.full((M + 1, ldy), 7.0, device=device)
    C_ = capi()
    C_.check(C_.lib().grl_tc_unpack16(C_.ptr(x16), ldx, x_off, C_.ptr(y), ldy, M, C, fmt, C_.stream()))
    y = y.cpu()
    same_bits(y[:M, :C], x[:, x_off:x_off + C].view(dt(fmt)).float())
    assert (y[:M, C:] == 7.0).all() and (y[M:] == 7.0).all()
    assert tc.unpack_rows(torch.empty(0, 64, device=device, dtype=dt(fmt)), 8).shape == (0, 8)


HEAD = [  # B, Cin, H, W, Hp, Wp: no pad | reflect | zero (pad >= size in H) | zero (pad >= size in W only)
    (2, 3, 16, 24, 16, 24), (2, 3, 13, 21, 16, 24), (2, 1, 5, 21, 16, 24), (3, 4, 13, 5, 16, 16), (2, 3, 9, 9, 12, 18),
]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("per_channel", [False, True])
@pytest.mark.parametrize("B,Cin,H,W,Hp,Wp", HEAD)
def test_head_pack_bit_exact(tc, device, B, Cin, H, W, Hp, Wp, per_channel, fmt):
    """grl_tc_head_pack = check_image_size + normalise + bchw -> channels-last + pack, bit-exact: reflect padding on the
    bottom / right (F.pad "reflect") when the pad is smaller than the image in both dimensions, else zero padding of the
    RAW image (torch raises for that reflect pad, and the reference then pads with zeros); then (x - mean) * img_range
    in fp32 (y32, want_f32) and its 16-bit rounding (y16) with channels [Cin, Cpad) zero."""
    g = torch.Generator().manual_seed(B * 100 + H)
    x = torch.rand(B, Cin, H, W, generator=g) * 1.3 - 0.1
    mean = [0.4488, 0.4371, 0.4040, 0.5][:Cin] if per_channel else [0.45]
    rng = 255.0 if per_channel else 1.7
    pad = (0, Wp - W, 0, Hp - H)
    reflect = Hp - H < H and Wp - W < W
    xp = F.pad(x, pad, "reflect") if reflect else F.pad(x, pad, "constant", 0.0)
    m = torch.tensor(mean * Cin if len(mean) == 1 else mean).view(1, Cin, 1, 1)
    ref32 = ((xp - m) * rng).permute(0, 2, 3, 1).contiguous()
    for want_f32 in (False, True):
        for cpad in (8, 64):
            y16, y32 = tc.head_pack(x.to(device), Hp, Wp, mean, rng, cpad, fmt, want_f32=want_f32)
            y16 = y16.cpu()
            same_bits(y16[..., :Cin], to16(ref32, fmt))
            assert not y16[..., Cin:].float().any()
            if want_f32:
                same_bits(y32.cpu(), ref32)
            else:
                assert y32 is None


def _avgpool(tc, x16, df, fmt):
    B, H, W, Cp = x16.shape
    y = torch.empty(B, H // df, W // df, Cp, device=x16.device, dtype=x16.dtype)
    C_ = capi()
    C_.check(C_.lib().grl_tc_avgpool16(C_.ptr(x16), C_.ptr(y), B, H, W, Cp, df, fmt, C_.stream()))
    return y.cpu()


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("Cpad", [64, 192])
@pytest.mark.parametrize("df", [1, 2, 3, 4])
def test_avgpool16(tc, device, df, Cpad, fmt):
    """grl_tc_avgpool16 (the anchor pooling): fp32 sum of the df x df 16-bit inputs, times fp32(1 / df^2), rounded once
    to 16 bits.  The inputs keep magnitudes in [2^-6, 4) (or 0), so the fp32 sum of <= 16 of them is exact; the result is
    then the float64 mean rounded once -- bit-exact for df in {1, 2, 4} (1 / df^2 is a power of two), within one 16-bit
    ulp for df = 3 (1/9 is rounded to fp32 first)."""
    B, H, W = 2, 12, 36
    g = torch.Generator().manual_seed(df * 7 + Cpad)
    x = (torch.randn(B, H, W, Cpad, generator=g) * 1.2).clamp(-3.99, 3.99)
    x = torch.where(x.abs() < 2.0 ** -6, torch.zeros_like(x), x)
    x16 = to16(x, fmt)
    got = _avgpool(tc, x16.to(device), df, fmt)
    mean = x16.double().view(B, H // df, df, W // df, df, Cpad).mean(dim=(2, 4))
    ref = mean.float().to(dt(fmt))  # mean is a sum of <= 16 values with a 22-bit span: fp32-exact, one rounding to 16 bits
    if df != 3:
        same_bits(got, ref)
    else:
        assert ((got.double() - mean).abs() <= ulp16(mean, fmt)).all()


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("C", [36, 180])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("L", [1, 511, 512, 513, 4103])
def test_tc_channel_gate(tc, device, L, B, C, fmt):
    """grl_tc_channel_gate: channel means of the 16-bit CAB features (B, L, ld = cpad > C) in deterministic chunks of
    kPoolRowsTc = 512 rows, then the squeeze-excite MLP, against float64.  Columns [C, cpad) hold 1e3 and must not leak.

    Bound.  A chunk is a sequential fp32 sum of <= 512 terms and the chunks are summed sequentially, so
    |fl(sum) - sum| <= (511 + chunks - 1) u sum|y|; the division by L adds u |mean|:  |dmean_c| <= (512 + chunks) u mean|y_c|
    (u = 2^-24).  The hidden unit h_r = relu(sum_c w1 mean_c + b1) (C + 1 fp32 fma / add) gets
    |dh_r| <= sum_c |w1_rc| |dmean_c| + (C + 1) u (sum_c |w1_rc mean_c| + |b1_r|), the logit s_c likewise with R and w2, and
    sigmoid' <= 1/4 plus ~4 u for expf / add / divide.  The test allows twice that first-order bound."""
    R = C // 18
    cpad = tc.round_up(C, 64)
    g = torch.Generator().manual_seed(L + 10 * B + C + 1000 * fmt)
    y = torch.randn(B, L, C, generator=g) * 2.0 + 0.3
    y16 = torch.full((B, L, cpad), 1e3).to(dt(fmt))
    y16[..., :C] = y.to(dt(fmt))
    w1, b1 = torch.randn(R, C, generator=g) / C ** 0.5, torch.randn(R, generator=g) * 0.1
    w2, b2 = torch.randn(C, R, generator=g) / R ** 0.5, torch.randn(C, generator=g) * 0.1
    ref, m, h = channel_gate_reference(y16[..., :C].float(), w1, b1, w2, b2)
    chunks = (L + 511) // 512
    dm = (512 + chunks) * U * y16[..., :C].double().abs().mean(1)
    dh = dm @ w1.double().abs().T + (C + 1) * U * (m.abs() @ w1.double().abs().T + b1.double().abs())
    ds = dh @ w2.double().abs().T + (R + 1) * U * (h.abs() @ w2.double().abs().T + b2.double().abs())
    bound = 2 * (ds / 4 + 4 * U * ref)
    lib, C_ = capi().lib(), capi()
    d = lambda t: t.contiguous().to(device)  # noqa: E731
    yd, w1d, b1d, w2d, b2d = d(y16), d(w1), d(b1), d(w2), d(b2)
    nbytes = lib.grl_tc_channel_gate_workspace(B, L, C)
    assert nbytes == 4 * B * chunks * C
    ws = torch.empty(nbytes // 4, device=device)
    gate = torch.full((B, C), -1.0, device=device)
    C_.check(lib.grl_tc_channel_gate(C_.ptr(yd), cpad, fmt, B, L, C, C_.ptr(w1d), C_.ptr(b1d), C_.ptr(w2d), C_.ptr(b2d), R,
                                     C_.ptr(gate), C_.ptr(ws), nbytes, C_.stream()))
    err = (gate.cpu().double() - ref).abs()
    assert (err <= bound).all(), f"max err {err.max().item():.3e}, bound there {bound.view(-1)[err.argmax()].item():.3e}"
    # host validation: a workspace one float short is refused before any launch
    rc = lib.grl_tc_channel_gate(C_.ptr(yd), cpad, fmt, B, L, C, C_.ptr(w1d), C_.ptr(b1d), C_.ptr(w2d), C_.ptr(b2d), R,
                                 C_.ptr(gate), C_.ptr(ws), nbytes - 4, C_.stream())
    assert rc == GRL_ERR_WORKSPACE


@pytest.mark.parametrize("hw,hs", [(1, 1), (2, 2), (3, 3), (8, 8), (2, 5)])
def test_slot_scale_layout(tc, device, hw, hs):
    """grl_tc_slot_scale: the per-slot scale vector of the packed QKV GEMM, in slot order
    [win q | win k | win v | stripe q | stripe k | stripe v] x heads:
      win q    = exp(min(ls_w, ln 100)) log2 e,   win k = 1,   win v = 0 (value slots are not normalised);
      stripe q = exp(min(ls_s2, ln 100)) log2 e   -- pass 2 (mixed_attn_block_efficient.py:259) is q against the anchors
                                                      under attn_transform2;
      stripe k = exp(min(ls_s1, ln 100)) log2 e   -- pass 1 (:257) is the anchors against k under attn_transform1, and
                                                      the scale of that pass sits on its keys (the anchors carry 1);
      stripe v = 0.
    ln 100 is the fp32 constant of the kernel.  Per-head logit scales below, at and above it make a swapped pair, a
    per-head misorder or a missing clamp visible.  rtol: expf is within 2 ulp (CUDA programming guide, 4 u relative), plus
    the fp32 rounding of log2 e and of the product: 6 u, u = 2^-24."""
    g = torch.Generator().manual_seed(hw * 10 + hs)

    def draw(h, below):
        v = math.log(5.0) + (math.log(150.0) - math.log(5.0)) * torch.rand(h, generator=g)
        if h >= 2:
            v[0], v[1] = LN100_F32, below  # at and below the clamp
        if h >= 3:
            v[2] = 5.3  # above it
        return v.float()

    lw, l1, l2 = draw(hw, 2.1), draw(hs, 2.3), draw(hs, 2.5)
    out = torch.full((3 * hw + 3 * hs,), float("nan"), device=device)
    C_ = capi()
    lwd, l1d, l2d = lw.view(hw, 1, 1).to(device), l1.view(hs, 1, 1).to(device), l2.view(hs, 1, 1).to(device)
    C_.check(C_.lib().grl_tc_slot_scale(C_.ptr(lwd), C_.ptr(l1d), C_.ptr(l2d), hw, hs, C_.ptr(out), C_.stream()))
    sc = lambda ls: torch.exp(ls.double().clamp(max=LN100_F32)) * (1 / math.log(2.0))  # noqa: E731
    ref = torch.cat([sc(lw), torch.ones(hw, dtype=torch.float64), torch.zeros(hw, dtype=torch.float64),
                     sc(l2), sc(l1), torch.zeros(hs, dtype=torch.float64)])
    got = out.cpu().double()
    exact = ref.eq(0) | ref.eq(1)
    assert torch.equal(got[exact], ref[exact])
    rel = ((got - ref).abs() / ref)[~exact]
    assert rel.max().item() <= 6 * U, rel.max().item()


def _bias_geoms():
    rows = []
    for ws in (8, 16, 32, 36):
        rows.append((f"window{ws}", (2 * ws - 1) ** 2))
    for (sh, sw), df in (((64, 64), 2), ((48, 96), 4), ((72, 144), 4)):
        rows.append((f"stripe{sh}x{sw}_df{df}", (sh + sh // df - 1) * (sw + sw // df - 1)))
    return rows


@pytest.mark.parametrize("heads", [1, 3, 8])
@pytest.mark.parametrize("name,rows", _bias_geoms(), ids=[n for n, _ in _bias_geoms()])
def test_bias_table4(tc, device, name, rows, heads):
    """grl_tc_bias_table4 (the attention kernel's relative-position bias): copy c of head h holds
    16 sigmoid(W2 relu(W1 t + b1)) log2 e at [c, c + rows) of the (heads, 4, rows_pad) table -- the shifted copies the
    attention kernel reads with aligned loads -- and every other entry of the zero-initialised buffer stays exactly 0.

    Bound (float64 reference, u = 2^-24): the hidden unit is two fp32 fma, |dh_k| <= 2 u (|w1_k0 t0| + |w1_k1 t1| +
    |b1_k|); the logit is 512 sequential fma, |da| <= 512 u sum_k |w2_k h_k| + sum_k |w2_k| |dh_k|; then
    d(16 sigmoid(a)) = 16 sigmoid(a) (1 - sigmoid(a)) da, plus ~6 u relative for expf, add, divide and the two products.
    The test allows twice that."""
    hidden = 512
    g = torch.Generator().manual_seed(rows + heads)
    t = (torch.rand(rows, 2, generator=g) * 16 - 8)
    w1 = torch.randn(hidden, 2, generator=g) * 0.7
    b1 = torch.randn(hidden, generator=g) * 0.5
    w2 = torch.randn(heads, hidden, generator=g) * 0.15
    rows_pad = tc.bias_rows_pad(rows)
    out = torch.zeros(heads, 4, rows_pad, device=device)
    C_ = capi()
    d = lambda x: x.contiguous().to(device)  # noqa: E731
    td, w1d, b1d, w2d = d(t), d(w1), d(b1), d(w2)
    C_.check(C_.lib().grl_tc_bias_table4(C_.ptr(td), rows, C_.ptr(w1d), C_.ptr(b1d), C_.ptr(w2d), hidden, heads, tc.LOG2E,
                                         rows_pad, C_.ptr(out), C_.stream()))
    out = out.cpu().double()
    pre = t.double() @ w1.double().T + b1.double()
    h = torch.relu(pre)
    a = h @ w2.double().T  # (rows, heads)
    sg = torch.sigmoid(a)
    ref = (16 * sg * tc.LOG2E).T  # (heads, rows)
    dh = 2 * U * (t.double().abs() @ w1.double().abs().T + b1.double().abs())
    da = hidden * U * (h @ w2.double().abs().T) + dh @ w2.double().abs().T
    bound = 2 * (16 * tc.LOG2E * sg * (1 - sg) * da + 6 * U * 16 * tc.LOG2E * sg).T
    mask = torch.zeros_like(out, dtype=torch.bool)
    for c in range(4):
        err = (out[:, c, c:c + rows] - ref).abs()
        assert (err <= bound).all(), f"copy {c}: max err {err.max().item():.3e}"
        mask[:, c, c:c + rows] = True
    assert not out[~mask].any(), "entries outside the four shifted copies were written"


def _conv(device, Cin, Cout, seed):
    g = torch.Generator().manual_seed(seed)
    conv = torch.nn.Conv2d(Cin, Cout, 3, 1, 1)
    conv.weight.data.copy_(torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5)
    conv.bias.data.copy_(torch.randn(Cout, generator=g) * 0.3)
    return conv.to(device)


def _x16(tc, device, B, Cin, H, W, seed, fmt):
    x = torch.randn(B, Cin, H, W, generator=torch.Generator().manual_seed(seed))
    return x, tc.pack_rows(x.permute(0, 2, 3, 1).contiguous().to(device), tc.round_up(Cin, 64), fmt)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("Cq", [8, 64])
@pytest.mark.parametrize("r", [2, 3])
def test_pixelshuffle_store_bitwise(tc, device, r, Cq, fmt):
    """The conv epilogue's PixelShuffle store (ps_r = r, weights packed with pack_conv(..., ps_r=r)) writes exactly the
    values of the plain 16-bit store of the same packed conv, rearranged by PixelShuffle: column q Cq + c of pixel (y, x)
    goes to channel c of pixel (y r + q // r, x r + q % r).  Bitwise, since only the store address differs.  A loose
    check against F.pixel_shuffle(F.conv2d(...)) catches packing errors."""
    B, Cin, H, W = 2, 48, 13, 21
    Cout = Cq * r * r
    conv = _conv(device, Cin, Cout, 100 + r + Cq)
    x, x16 = _x16(tc, device, B, Cin, H, W, 200 + r + Cq, fmt)
    cin_pad, npad = 64, tc.round_up(Cout, 64)
    wp, bp = tc.pack_conv(conv, cin_pad, npad, fmt, ps_r=r)
    fused = torch.full((B, H * r, W * r, Cq), float("nan"), device=device, dtype=dt(fmt))
    tc.conv3x3(x16, wp, bp, cin_pad, npad, n_store=Cout, n_real=Cout, out_bf16=fused, ps_r=r)
    plain = torch.full((B, H, W, npad), float("nan"), device=device, dtype=dt(fmt))
    tc.conv3x3(x16, wp, bp, cin_pad, npad, n_store=npad, n_real=Cout, out_bf16=plain)
    fused, plain = fused.cpu(), plain.cpu()
    shuffled = plain[..., :Cout].reshape(B, H, W, r, r, Cq).permute(0, 1, 3, 2, 4, 5).reshape(B, H * r, W * r, Cq)
    same_bits(fused, shuffled)
    ref = F.pixel_shuffle(F.conv2d(x.to(dt(fmt)).float(), conv.weight.detach().cpu().to(dt(fmt)).float(),
                                   conv.bias.detach().cpu(), padding=1), r).permute(0, 2, 3, 1)
    assert (fused.float() - ref).abs().max().item() <= 3e-2 * max(1.0, ref.abs().max().item())


# (r, out channels, input residual): every head's tail; the residual exists only on the no-upsampler tail (r = 1)
TAILS = [(r, oc, False) for r in (1, 2, 3, 4) for oc in (1, 3)] + [(1, 1, True), (1, 3, True)]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("r,oc,with_res", TAILS)
def test_nchw_tail_store(tc, device, r, oc, with_res, fmt):
    """The network's last conv writes (B, oc, Hc, Wc) fp32 planes from its epilogue: PixelShuffle(r) when r > 1, the crop
    to Hc x Wc, x * post_scale + post_shift[c] as one fmaf, and with the input residual (the no-upsampler tail,
    tc.forward) the fp32 residual added before it.  Reference: the same conv with a plain fp32 store,
    rearranged and cropped in torch, then scale and shift in float64 rounded to fp32 -- within 1 fp32 ulp (the fmaf's
    single rounding).  The output is a view into a NaN-filled buffer with a guard region after it: no in-crop value may
    stay NaN, and no tile past the crop may write outside it."""
    B, Cin, H, W = 2, 64, 13, 21
    Cout = oc * r * r
    Hc, Wc = H * r - 3, W * r - 3  # neither a multiple of the 8 x 16 tile nor of r
    conv = _conv(device, Cin, Cout, 300 + r + oc)
    x, x16 = _x16(tc, device, B, Cin, H, W, 400 + r + oc, fmt)
    npad = 64
    wp, bp = tc.pack_conv(conv, 64, npad, fmt)
    res = torch.randn(B, H, W, Cout, generator=torch.Generator().manual_seed(5)).to(device) if with_res else None
    scale, shift = 1.0 / 255.0, [0.4488, -0.4371, 0.404, 0.0][:oc]
    ref32 = torch.empty(B, H, W, Cout, device=device)
    tc.conv3x3(x16, wp, bp, 64, npad, n_store=npad, n_real=Cout, out_f32=ref32, res_f32=res)
    n = B * oc * Hc * Wc
    buf = torch.full((n + 4096,), float("nan"), device=device)
    out = buf[:n].view(B, oc, Hc, Wc)
    tc.conv3x3(x16, wp, bp, 64, npad, n_store=npad, n_real=Cout, res_f32=res, out_nchw=out, nchw_r=r, post_scale=scale,
               post_shift=shift)
    buf = buf.cpu()
    assert torch.isnan(buf[n:]).all(), "a tile past the crop wrote outside the output"
    got = buf[:n].view(B, oc, Hc, Wc)
    assert not torch.isnan(got).any(), "an in-crop pixel was not written"
    t = ref32.cpu().permute(0, 3, 1, 2)
    t = F.pixel_shuffle(t, r) if r > 1 else t
    t = t[:, :, :Hc, :Wc].double()
    ref = (t * torch.tensor(scale, dtype=torch.float32).double() +
           torch.tensor(shift, dtype=torch.float32).double().view(1, oc, 1, 1)).float()
    ulp = torch.nextafter(ref.abs(), torch.tensor(float("inf"))) - ref.abs()
    err = (got - ref).abs()
    assert (err <= ulp).all(), f"max err {err.max().item():.3e}"
