"""CPU oracle for the GRL forward hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` leg may
import this file.  The product path (grl-image-restoration_b200/) never does; it fails loudly when
its CUDA library is missing.

What this is: a functional (state_dict in, tensors out) restatement, in plain CPU PyTorch fp32 ops,
of the reference's algorithm for the path named by BASELINE.json.  The reference is Python/ATen,
so the arithmetic below is issued through the same ATen CPU primitives (matmul, conv2d, softmax,
layer_norm) in the same order as the reference; every function cites the reference file:line it
follows (paths relative to /root/reference).  It deliberately MATERIALISES the (N1 x N2) attention
maps, the int64 relative-position index and the -100 shift masks the way the reference does, so it
is also the honest CPU baseline (`cpu_baseline.kind == "port"`).

Parity pinning: oracle/make_golden.py imports the UNMODIFIED reference in the build container and
(a) asserts this file reproduces it (tables / indices / masks bit-exact, module and model outputs
to <= 2e-6), (b) writes tests/golden/*.npz which tests/test_oracle_golden.py replays anywhere.
"""
from math import log, prod

import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# configuration helpers
# --------------------------------------------------------------------------------------

_DEFAULTS = dict(  # models/networks/grl.py:220-256 (constructor defaults)
    img_size=64,
    in_channels=3,
    out_channels=None,
    embed_dim=96,
    upscale=2,
    img_range=1.0,
    upsampler="",
    depths=[6, 6, 6, 6, 6, 6],
    num_heads_window=[3, 3, 3, 3, 3, 3],
    num_heads_stripe=[3, 3, 3, 3, 3, 3],
    window_size=8,
    stripe_size=[8, 8],
    stripe_groups=[None, None],
    stripe_shift=False,
    mlp_ratio=4.0,
    anchor_window_down_factor=1,
    local_connection=False,
    init_method="n",
)


def full_config(cfg):
    out = dict(_DEFAULTS)
    out.update(cfg)
    out["out_channels"] = out["out_channels"] or out["in_channels"]
    return out


def pair(v):
    return tuple(v) if isinstance(v, (list, tuple)) else (v, v)


def stripe_info(stripe_size, stripe_groups, stripe_shift, resolution):
    """models/common/mixed_attn_block_efficient.py:61-70."""
    sizes, shifts = [], []
    for s, g, d in zip(stripe_size, stripe_groups, resolution):
        if g is None:
            sizes.append(s)
            shifts.append(s // 2 if stripe_shift else 0)
        else:
            sizes.append(d // g)
            shifts.append(0 if g == 1 else d // (g * 2))
    return sizes, shifts


def pad_size(cfg):
    """models/networks/grl.py:273-276."""
    c = full_config(cfg)
    ms = max(0 if s is None else s for s in c["stripe_size"])
    mg = max(0 if s is None else s for s in c["stripe_groups"]) * c["anchor_window_down_factor"]
    return max(c["window_size"], ms, mg)


# --------------------------------------------------------------------------------------
# partition / geometry (models/common/ops.py)
# --------------------------------------------------------------------------------------


def partition(x, ws):
    """ops.py:36-54: (B,H,W,C) -> (B*nW, wh, ww, C), windows ordered row-major."""
    B, H, W, C = x.shape
    x = x.reshape(B, H // ws[0], ws[0], W // ws[1], ws[1], C)
    return x.permute(0, 1, 3, 2, 4, 5).reshape(-1, ws[0], ws[1], C)


def unpartition(w, ws, size):
    """ops.py:57-73."""
    H, W = size
    nh, nw = H // ws[0], W // ws[1]
    B = w.shape[0] // (nh * nw)
    x = w.reshape(B, nh, nw, ws[0], ws[1], -1)
    return x.permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, -1)


def region_ids(resolution, ws, shift):
    """ops.py:76-99 (_fill_window): 9-region id image by *sequential slice assignment*, then
    partitioned into per-window id vectors (nW, wh*ww).  The python-slice semantics for a zero
    shift (slice(-w, -0) is empty, slice(-0, None) is everything) are kept on purpose."""
    img = torch.zeros((1, resolution[0], resolution[1], 1))
    hs = (slice(0, -ws[0]), slice(-ws[0], -shift[0]), slice(-shift[0], None))
    wsl = (slice(0, -ws[1]), slice(-ws[1], -shift[1]), slice(-shift[1], None))
    n = 0
    for a in hs:
        for b in wsl:
            img[:, a, b, :] = n
            n += 1
    return partition(img, ws).reshape(-1, ws[0] * ws[1])


def shift_mask(resolution, ws, shift, df=1, window_to_anchor=True):
    """ops.py:112-157 (calculate_mask == calculate_mask_all with df=1): 0 / -100 masks."""
    ares = [s // df for s in resolution]
    aws = [s // df for s in ws]
    ash = [s // df for s in shift]
    idw = region_ids(resolution, ws, shift)
    ida = region_ids(ares, aws, ash)
    diff = idw.unsqueeze(2) - ida.unsqueeze(1) if window_to_anchor else ida.unsqueeze(2) - idw.unsqueeze(1)
    return torch.where(diff != 0, torch.full_like(diff, -100.0), torch.zeros_like(diff))


def coords_table(ws, df=1):
    """ops.py:225-271 with pretrained size (0,0): log-spaced relative coordinate table
    (1, wh+awh-1, ww+aww-1, 2)."""
    aws = [w // df for w in ws]
    hi = [w1 - 1 - (w1 - w2) // 2 for w1, w2 in zip(ws, aws)]
    lo = [-(w2 - 1) - (w1 - w2) // 2 for w1, w2 in zip(ws, aws)]
    ch = torch.arange(lo[0], hi[0] + 1, dtype=torch.float32)
    cw = torch.arange(lo[1], hi[1] + 1, dtype=torch.float32)
    t = torch.stack(torch.meshgrid([ch, cw], indexing="ij")).permute(1, 2, 0).contiguous().unsqueeze(0)
    t[..., 0] /= hi[0]
    t[..., 1] /= hi[1]
    t *= 8
    import numpy as np  # the reference divides by a numpy float64 scalar (ops.py:269)

    return torch.sign(t) * torch.log2(torch.abs(t) + 1.0) / np.log2(8)


def position_index(ws, df=1, window_to_anchor=True):
    """ops.py:352-375 + coords_diff_odd ops.py:308-316."""
    aws = [w // df for w in ws]

    def grid(n):
        a = torch.arange(0, n[0])
        b = torch.arange(0, n[1])
        return torch.stack(torch.meshgrid([a, b], indexing="ij")).flatten(1)

    cw, ca = grid(ws), grid(aws)
    width = aws[1] + ws[1] - 1
    if window_to_anchor:
        d = (cw[:, :, None] - ca[:, None, :]).permute(1, 2, 0).contiguous()
        off = [a - 1 for a in aws]
    else:
        d = (ca[:, :, None] - cw[:, None, :]).permute(1, 2, 0).contiguous()
        off = [w - 1 for w in ws]
    d[:, :, 0] += off[0]
    d[:, :, 1] += off[1]
    d[:, :, 0] *= width
    return d.sum(-1)


def table_index_mask(cfg, x_size):
    """models/networks/grl.py:386-429 (set_table_index_mask)."""
    c = full_config(cfg)
    ws = pair(c["window_size"])
    df = c["anchor_window_down_factor"]
    ss, sss = stripe_info(c["stripe_size"], c["stripe_groups"], True, x_size)
    r = lambda v: v[::-1]
    return {
        "table_w": coords_table(ws),
        "table_sh": coords_table(ss, df),
        "table_sv": coords_table(r(ss), df),
        "index_w": position_index(ws),
        "index_sh_a2w": position_index(ss, df, False),
        "index_sh_w2a": position_index(ss, df, True),
        "index_sv_a2w": position_index(r(ss), df, False),
        "index_sv_w2a": position_index(r(ss), df, True),
        "mask_w": shift_mask(x_size, ws, [w // 2 for w in ws]),
        "mask_sh_a2w": shift_mask(x_size, ss, sss, df, False),
        "mask_sh_w2a": shift_mask(x_size, ss, sss, df, True),
        "mask_sv_a2w": shift_mask(x_size, r(ss), r(sss), df, False),
        "mask_sv_w2a": shift_mask(x_size, r(ss), r(sss), df, True),
    }


# --------------------------------------------------------------------------------------
# attention
# --------------------------------------------------------------------------------------


def affine(sd, pre, attn, table, index, mask):
    """mixed_attn_block_efficient.py:36-58 + CPB_MLP mixed_attn_block.py:24-31."""
    B_, H, N1, N2 = attn.shape
    attn = attn * torch.clamp(sd[pre + "logit_scale"], max=log(1.0 / 0.01)).exp()
    t = F.linear(table, sd[pre + "cpb_mlp.0.weight"], sd[pre + "cpb_mlp.0.bias"])
    t = F.linear(torch.relu(t), sd[pre + "cpb_mlp.2.weight"]).view(-1, H)
    bias = t[index.view(-1)].view(N1, N2, -1).permute(2, 0, 1).contiguous()
    attn = attn + (16 * torch.sigmoid(bias)).unsqueeze(0)
    if mask is not None:
        nW = mask.shape[0]
        attn = (attn.view(B_ // nW, nW, H, N1, N2) + mask.unsqueeze(1).unsqueeze(0)).view(-1, H, N1, N2)
    return attn


def cosine_attention(sd, pre, q, k, v, table, index, mask, merge_heads=True):
    """mixed_attn_block_efficient.py:77-94 (Attention.attn)."""
    B_, H, _, d = q.shape
    a = F.normalize(q, dim=-1) @ F.normalize(k, dim=-1).transpose(-2, -1)
    a = torch.softmax(affine(sd, pre, a, table, index, mask), dim=-1)
    x = a @ v
    if merge_heads:
        x = x.transpose(1, 2).reshape(B_, -1, H * d)
    return x


# --------------------------------------------------------------------------------------
# the tensor-core attention kernel's algorithm (csrc/attn_tc.cu), in float64
# --------------------------------------------------------------------------------------

ATTN_KEY_TILE = 64   # keys per tile (attn_tc.cu: KT)
ATTN_Q_TILE = 128    # query rows per CTA (kQT); a partial last tile is padded
ATTN_WARP_ROWS = 32  # rows that share one lazy-rescale decision
ATTN_TAU = 8.0       # attn_tc.cuh: kTau
LOG2E = 1.4426950408889634


def lazy_softmax_emulate(x, v, dtype, mutation=None):
    """The attention kernel's softmax on log2-domain scores x (..., R, N), R a multiple of 32, and values v (..., N, d).

    Keys go in tiles of 64, in order.  Each row keeps a reference m_ref: the first tile sets it to the tile maximum; after
    that it moves only when the tile maximum of some row of its warp (32 consecutive rows) exceeds it by more than
    ATTN_TAU, and then every row of that warp moves by delta = max(mx - m_ref, 0) and scales O and l by 2^-delta.
    P = exp2(x - m_ref) is rounded to `dtype`, O += P V and l += sum of the ROUNDED P (what the ones-column of V yields).
    Everything else is float64.  Returns (O / l, info) with info["rescales"] the warp rescales after the first tile and
    info["p_max"] the largest P.

    mutation imitates a kernel bug: "rescale_o_only" (l misses the rescale), "unrounded_denominator" (l sums the
    unrounded P)."""
    *lead, R, N = x.shape
    o = x.new_zeros(*lead, R, v.shape[-1])
    l = x.new_zeros(*lead, R)
    m_ref = None
    rescales, p_max = 0, 0.0
    for t, k0 in enumerate(range(0, N, ATTN_KEY_TILE)):
        xt = x[..., k0:k0 + ATTN_KEY_TILE]
        mx = xt.amax(-1)
        if t == 0:
            m_ref = mx.clone()
        else:
            warp = (mx - m_ref > ATTN_TAU).unflatten(-1, (R // ATTN_WARP_ROWS, ATTN_WARP_ROWS)).any(-1, keepdim=True)
            grow = warp.expand(*warp.shape[:-1], ATTN_WARP_ROWS).flatten(-2)
            n = int(warp.sum())
            if n:
                delta = torch.where(grow, (mx - m_ref).clamp_min(0.0), torch.zeros_like(mx))
                m_ref = m_ref + delta
                sc = torch.exp2(-delta)
                o = o * sc[..., None]
                if mutation != "rescale_o_only":
                    l = l * sc
                rescales += n
        p = torch.exp2(xt - m_ref[..., None])
        p16 = p.to(dtype).to(x.dtype)
        o = o + p16 @ v[..., k0:k0 + ATTN_KEY_TILE, :].to(x.dtype)
        l = l + (p if mutation == "unrounded_denominator" else p16).sum(-1)
        p_max = max(p_max, float(p.max()))
    return o / l[..., None], {"rescales": rescales, "p_max": p_max}


def attn_windows(tokens, grid, heads):
    """(B, H, W, heads * 32) token slots -> (B * nW, heads, wh * ww, 32) in the order the kernel walks a window:
    torch.roll by (-sh, -sw), then partition.  grid = (H, W, wh, ww, sh, sw)."""
    _, _, wh, ww, sh, sw = grid
    t = torch.roll(tokens, (-sh, -sw), (1, 2)) if sh or sw else tokens
    return partition(t, (wh, ww)).reshape(-1, wh * ww, heads, 32).transpose(1, 2)


def attn_pair_geometry(gq, gk, use_mask):
    """(index (Nq, Nk), mask (nW, Nq, Nk) of 0 / -100, or None) of one launch of the attention kernel.  Equal windows are
    window attention; otherwise the smaller window is the anchor window of a stripe pass (df = token / anchor window)."""
    if gq[2:4] == gk[2:4]:
        res, ws, sh, df, w2a = gq[:2], list(gq[2:4]), list(gq[4:6]), 1, True
    else:
        w2a = gq[2] > gk[2]  # the queries are the tokens: pass 2
        tg, ag = (gq, gk) if w2a else (gk, gq)
        df = tg[2] // ag[2]
        assert tg[3] // ag[3] == df and tg[0] // ag[0] == df
        res, ws, sh = tg[:2], list(tg[2:4]), list(tg[4:6])
    index = position_index(ws, df, w2a)
    mask = shift_mask(list(res), ws, sh, df, w2a) if use_mask else None
    return index, mask


def attn_launch_reference(q, k, v, table, index, mask, dtype, mutation=None, max_elems=1 << 25):
    """One launch of the attention kernel on gathered operands, in float64 on q's device.

    q (Bw, h, Nq, 32), k and v (Bw, h, Nk, 32): the 16-bit operand values (q carries exp(min(s, ln 100)) * log2 e);
    table (h, rows) bias in log2 units; index (Nq, Nk) into it; mask (nW, Nq, Nk) of 0 / -100 (window w uses mask[w % nW])
    or None.  Returns (exact, emulated, info), each output (Bw, h, Nq, 32) float64:
      exact:    softmax over the keys of 2^(S + bias + mask log2 e), times V;
      emulated: lazy_softmax_emulate of the same scores, rounded to `dtype`.  The query tile is padded to 128 rows the
                way the kernel pads it (zero Q, the bias and mask row of query 0): those rows share warp decisions.
    Windows are processed in chunks of at most max_elems scores."""
    f = torch.float64
    dev = q.device
    Bw, h, Nq, _ = q.shape
    Nk = k.shape[2]
    qp = -(-Nq // ATTN_Q_TILE) * ATTN_Q_TILE
    r = torch.arange(qp, device=dev)
    rows = torch.where(r < Nq, r, 0)
    bias = table.to(dev, f)[:, index.to(dev)[rows]]  # (h, qp, Nk)
    mlog = None if mask is None else mask.to(dev, f)[:, rows] * LOG2E
    exact, emul = torch.empty(Bw, h, Nq, 32, dtype=f, device=dev), torch.empty(Bw, h, Nq, 32, dtype=f, device=dev)
    info = {"rescales": 0, "p_max": 0.0}
    step = max(1, max_elems // (h * qp * Nk))
    for w0 in range(0, Bw, step):
        w1 = min(Bw, w0 + step)
        qq = torch.zeros(w1 - w0, h, qp, 32, dtype=f, device=dev)
        qq[:, :, :Nq] = q[w0:w1].to(f)
        vv = v[w0:w1].to(f)
        x = qq @ k[w0:w1].to(f).transpose(-1, -2) + bias
        if mlog is not None:
            x = x + mlog[torch.arange(w0, w1, device=dev) % mlog.shape[0]].unsqueeze(1)
        exact[w0:w1] = torch.softmax(x[:, :, :Nq] * log(2.0), dim=-1) @ vv
        o, inf = lazy_softmax_emulate(x, vv, dtype, mutation)
        emul[w0:w1] = o[:, :, :Nq].to(dtype).to(f)
        info["rescales"] += inf["rescales"]
        info["p_max"] = max(info["p_max"], inf["p_max"])
    return exact, emul, info


ATTN_F32_KEY_TILE = 32  # keys per online-softmax step of attn_f32_kernel (ops_f32.cu: kKT)


def attn_f32_reference(q, k, v, logit_scale, table, index, mask, mutation=None, max_elems=1 << 25):
    """One launch of the fp32 attention kernel (ops_f32.cu attn_f32_kernel) on gathered operands, in float64 on q's device.

    q (Bw, h, Nq, d), k and v (Bw, h, Nk, d) as stored (q and k un-normalised: the kernel normalises them with the
    F.normalize eps); logit_scale (h,) natural log, clamped at ln 100; table (h, rows) bias in natural units; index
    (Nq, Nk) into it; mask (nW, Nq, Nk) of 0 / -100 (window w uses mask[w % nW]) or None.  Returns (Bw, h, Nq, d).

    mutation imitates a kernel bug: "k_unnormalised", "scale_unclamped", "rescale_missing_l" (the running denominator
    is not rescaled when a later key tile of ATTN_F32_KEY_TILE keys raises the row maximum)."""
    f = torch.float64
    dev = q.device
    qn = F.normalize(q.to(f), dim=-1, eps=1e-12)
    kn = k.to(f) if mutation == "k_unnormalised" else F.normalize(k.to(f), dim=-1, eps=1e-12)
    ls = logit_scale.to(dev, f).reshape(-1)
    sc = torch.exp(ls if mutation == "scale_unclamped" else ls.clamp(max=log(100.0)))[:, None, None]
    bias = table.to(dev, f)[:, index.to(dev)]
    mk = None if mask is None else mask.to(dev, f)
    Bw, h, Nq, d = q.shape
    Nk = k.shape[2]
    out = torch.empty(Bw, h, Nq, d, dtype=f, device=dev)
    step = max(1, max_elems // (h * Nq * Nk))
    for w0 in range(0, Bw, step):
        w1 = min(Bw, w0 + step)
        x = qn[w0:w1] @ kn[w0:w1].transpose(-1, -2) * sc + bias
        if mk is not None:
            x = x + mk[torch.arange(w0, w1, device=dev) % mk.shape[0]].unsqueeze(1)
        vv = v[w0:w1].to(f)
        if mutation != "rescale_missing_l":
            out[w0:w1] = torch.softmax(x, dim=-1) @ vv
            continue
        m = torch.full(x.shape[:-1], -float("inf"), dtype=f, device=dev)
        l, o = torch.zeros_like(m), torch.zeros(*x.shape[:-1], d, dtype=f, device=dev)
        for k0 in range(0, Nk, ATTN_F32_KEY_TILE):
            xt = x[..., k0:k0 + ATTN_F32_KEY_TILE]
            mn = torch.maximum(m, xt.amax(-1))
            p = torch.exp(xt - mn[..., None])
            o = o * torch.exp(m - mn)[..., None] + p @ vv[..., k0:k0 + ATTN_F32_KEY_TILE, :]
            l = l + p.sum(-1)
            m = mn
        out[w0:w1] = o / l[..., None]
    return out


GEMM_TILE_M = 128       # accumulator rows per CTA of gemm_tc_kernel (kBM)
GEMM_CONV_PATCH = (8, 16)  # conv row tile: an 8 x 16 pixel patch (kTH, kTW)
GEMM_K_CHUNK = 64       # k per stage of the operand ring (kBK)
GELU_AS_ABS_ERR = 5e-7  # max |gelu_as - erf GELU| over fp32 inputs (tests/test_gpu_tc_gemm.py::test_gelu_as_bound)


def gelu_as_emulate(x):
    """gemm_tc.cu's gelu_as in numpy float32 with a correctly rounded reciprocal and exp2 (the hardware's .approx
    errors are not modelled) and fmaf as one rounding of the float64 result.  x: float32 ndarray."""
    import numpy as np

    f = np.float32

    def fma(a, b, c):
        return (a.astype(np.float64) * b + c).astype(f)

    z = np.abs(x) * f(0.70710678118654752440)
    t = (1.0 / fma(f(0.3275911), z, f(1.0)).astype(np.float64)).astype(f)
    e = np.exp2(((-z * z) * f(1.4426950408889634)).astype(np.float64)).astype(f)
    p = fma(f(1.061405429), t, f(-1.453152027))
    p = fma(p, t, f(1.421413741))
    p = fma(p, t, f(-0.284496736))
    p = fma(p, t, f(0.254829592))
    erf_abs = fma(-p * t, e, f(1.0))
    half_x = f(0.5) * x
    return fma(half_x, np.copysign(erf_abs, x), half_x)


def _gelu(v, tanh=False):
    if tanh:
        return 0.5 * v * (1 + torch.tanh((2 / torch.pi) ** 0.5 * (v + 0.044715 * v ** 3)))
    return 0.5 * v * (1 + torch.special.erf(v * 0.5 ** 0.5))


def gemm_launch_reference(x, w, bias, *, taps=1, epi=0, act=0, slope=0.0, n_res=0, res=None, slot_scale=None, gamma=None,
                          beta=None, eps=1e-5, res_scale=1.0, cab_y=None, cab_gate=None, L=1, ps_r=0, nchw_r=0, crop=None,
                          post_scale=1.0, post_shift=None, bn=None, mutation=None):
    """One grl_tc_gemm launch in float64 on x's device, from the 16-bit operand values (gemm_tc.cu; include/grl_b200.h).

    x: (M, K) rows, or (B, H, W, K) channels-last when taps == 9 (3 x 3 conv, zero padding); w (N, taps K) with
    k = tap K + c, tap = 3 dy + dx; bias (N,).  epi 0: act(acc + b) (act 1 = erf GELU, 2 = LeakyReLU(slope)) + res on the
    first n_res columns; epi 1: every 32-wide slot with slot_scale > 0 becomes (acc + b) scale / max(||acc + b||, 1e-12);
    epi 2: res + res_scale LayerNorm(acc + b) over the first C = len(gamma) columns (two-pass moments, biased variance)
    + cab_y cab_gate[row // L].  Returns {"y": (rows, N or C) in token order}, plus "ps" (B, H r, W r, N / r^2) for the
    PixelShuffle store (column n = q N / r^2 + c) and "nchw" (B, N / r^2, Hc, Wc) = y post_scale + post_shift[c] for the
    NCHW tail (torch channel order n = c r^2 + q), cropped to crop = (Hc, Wc).

    mutation imitates a kernel bug: "bias_tile_local" / "slot_scale_per_tile" (index by the column inside the bn-wide N
    tile), "drop_kchunk" (k chunk 4 of 64, the first that reuses a ring stage, is skipped), "taps_transposed" (dy <-> dx),
    "ln_unbiased" (variance over n - 1), "ln_no_eps", "ln_naive_fp32" (E[x^2] - E[x]^2 in float32),
    "cab_gate_per_tile" (every row takes the gate of its row tile's first row), "no_residual_last_tile" (the last row tile
    / pixel patch adds no residual), "gelu_tanh", "ps_swapped" (PixelShuffle store with q and c swapped)."""
    f = torch.float64
    dev = x.device
    x, w, bias = x.to(f), w.to(f).clone(), bias.to(f).clone()
    conv = taps == 9
    K = x.shape[-1]
    N = w.shape[0]
    if mutation == "drop_kchunk":
        w[:, 4 * GEMM_K_CHUNK:5 * GEMM_K_CHUNK] = 0
    if conv:
        B, H, W, _ = x.shape
        xp = F.pad(x, (0, 0, 1, 1, 1, 1))
        acc = torch.zeros(B, H, W, N, dtype=f, device=dev)
        for t in range(9):
            dy, dx = divmod(t, 3)
            if mutation == "taps_transposed":
                dy, dx = dx, dy
            acc += xp[:, dy:dy + H, dx:dx + W] @ w[:, t * K:(t + 1) * K].T
        acc = acc.reshape(-1, N)
        py, px = GEMM_CONV_PATCH
        yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
        tile = ((torch.arange(B, device=dev)[:, None, None] * -(-H // py) + yy // py) * -(-W // px) + xx // px).reshape(-1)
    else:
        acc = x @ w.T
        tile = torch.arange(acc.shape[0], device=dev) // GEMM_TILE_M
    cols = torch.arange(N, device=dev)
    if mutation == "bias_tile_local":
        bias = bias[cols % bn]
    v = acc + bias
    last = tile == tile.max()
    if res is not None:
        res = res.to(f).reshape(v.shape[0], -1).clone()
        if mutation == "no_residual_last_tile":
            res[last] = 0
    if epi == 0:
        if act == 1:
            v = _gelu(v, mutation == "gelu_tanh")
        elif act == 2:
            v = torch.where(v > 0, v, v * slope)
        if res is not None:
            v[:, :n_res] += res[:, :n_res]
    elif epi == 1:
        s = v.reshape(v.shape[0], -1, 32)
        sc = slot_scale.to(dev, f)
        if mutation == "slot_scale_per_tile":
            sc = sc[(cols[::32] % bn) // 32]
        nrm = s.pow(2).sum(-1, keepdim=True).sqrt().clamp_min(1e-12)
        v = torch.where(sc[None, :, None] > 0, s * sc[None, :, None] / nrm, s).reshape(v.shape)
    else:
        C = gamma.numel()
        u = v[:, :C]
        if mutation == "ln_naive_fp32":
            u32 = u.float()
            mean = u32.mean(-1, keepdim=True)
            var = (u32 * u32).mean(-1, keepdim=True) - mean * mean
            mean, var = mean.to(f), var.to(f)
        else:
            mean = u.mean(-1, keepdim=True)
            var = (u - mean).pow(2).sum(-1, keepdim=True) / (C - 1 if mutation == "ln_unbiased" else C)
        e = 0.0 if mutation == "ln_no_eps" else eps
        v = (u - mean) / torch.sqrt(var + e) * gamma.to(dev, f) + beta.to(dev, f)
        v = res[:, :C] + res_scale * v
        if cab_y is not None:
            rows = torch.arange(v.shape[0], device=dev)
            if mutation == "cab_gate_per_tile":
                rows = rows // GEMM_TILE_M * GEMM_TILE_M
            v = v + cab_y.to(f).reshape(v.shape[0], -1)[:, :C] * cab_gate.to(dev, f)[rows // L]
    out = {"y": v}
    if ps_r:
        r, Bi, Hi, Wi = ps_r, *x.shape[:3]
        if mutation == "ps_swapped":  # column n read as torch's c r^2 + q
            t = v.reshape(Bi, Hi, Wi, -1, r, r).permute(0, 1, 4, 2, 5, 3)
        else:
            t = v.reshape(Bi, Hi, Wi, r, r, -1).permute(0, 1, 3, 2, 4, 5)
        out["ps"] = t.reshape(Bi, Hi * r, Wi * r, -1)
    if nchw_r:
        r, Bi, Hi, Wi = nchw_r, *x.shape[:3]
        t = v[:, :n_res].reshape(Bi, Hi, Wi, -1, r, r).permute(0, 3, 1, 4, 2, 5).reshape(Bi, -1, Hi * r, Wi * r)
        t = t[:, :, :crop[0], :crop[1]] * post_scale
        out["nchw"] = t + torch.tensor(list(post_shift)[:t.shape[1]], dtype=f, device=dev)[None, :, None, None]
    return out


LN100_F32 = float(torch.tensor(log(100.0), dtype=torch.float32))  # the logit-scale clamp as the kernels hold it


def to16(x, fmt):
    """The 16-bit rounding contract of the pack kernels: round to nearest even; fp16 saturates at +-65504 (cvt.rn.satfinite,
    where torch's .half() would give inf), bf16 is torch's .bfloat16()."""
    x = x.float()
    return x.bfloat16() if fmt else x.clamp(-65504.0, 65504.0).half()


def channel_gate_reference(y, w1, b1, w2, b2):
    """float64 squeeze-excite of the CAB: sigmoid(W2 relu(W1 mean_L(y) + b1) + b2), y (B, L, C).  Returns the gate, the
    means and the hidden units."""
    m = y.double().mean(1)
    h = torch.relu(m @ w1.double().T + b1.double())
    return torch.sigmoid(h @ w2.double().T + b2.double()), m, h


U = 2.0 ** -24  # fp32 unit roundoff
L_LN = 100      # rows per image of the CAB gate in ln_reference / ln_bound: the boundary lies inside an 8-row block


def gamma(n):
    """gamma_n = n u / (1 - n u): the relative error bound of n fp32 roundings."""
    return n * U / (1 - n * U)


def ln_reference(u, gamma_, beta, eps, rs, x, cy, gate, mutation=None):
    """float64 LayerNorm residual of the fp32 kernels (K.ln_residual): LN(u) rs + x + cy gate[image of the row], with the
    images L_LN rows each.  `mutation` names a kernel bug whose effect to compute instead."""
    C = u.shape[1]
    if mutation == "naive fp32 E[x^2] - E[x]^2":
        u32 = u.float()
        mean32 = u32.mean(1, keepdim=True)
        mean, var = mean32.double(), ((u32 * u32).mean(1, keepdim=True) - mean32 * mean32).double()
    else:
        mean = u.mean(1, keepdim=True)
        var = (u - mean).pow(2).sum(1, keepdim=True) / (C - 1 if mutation == "n - 1 variance" else C)
    e = 0.0 if mutation == "no eps" else eps
    r = (u - mean) / torch.sqrt(var + e) * gamma_ + beta
    r = r * (1.0 if mutation == "res_scale dropped" else rs)
    if x is not None:
        r = r + x
    if cy is not None:
        rows = torch.arange(u.shape[0], device=u.device)
        if mutation == "CAB gate of the wrong image at the boundary":
            rows = rows // 8 * 8  # every row of an 8-row block takes the image of the block's first row
        r = r + cy * gate[rows // L_LN]
    return r


def ln_bound(u, gamma_, beta, eps, rs, x, cy, gate):
    """Per-element bound of ln_reference's fp32 kernel: two-pass moments over C, each a lane-strided sequential sum plus a
    5-level warp tree."""
    C = u.shape[1]
    ns = -(-C // 32) + 5
    mean = u.mean(1, keepdim=True)
    e_mean = gamma(ns) * u.abs().sum(1, keepdim=True) / C + U * mean.abs()
    d = u - mean
    var = d.pow(2).mean(1, keepdim=True)
    # the deviations carry the common mean error (its cross term sums to zero) and one rounding each
    e_var = e_mean ** 2 + (var + e_mean ** 2) * (gamma(ns) + 4 * U)
    rel_v = (e_var + U * (var + eps)) / (var + eps)
    rel_r = 0.5 * rel_v * (1 + rel_v) + 2.5 * U  # sqrt, reciprocal
    rstd = 1 / torch.sqrt(var + eps)
    n = d * rstd
    e_n = (e_mean + U * (d.abs() + e_mean)) * rstd + n.abs() * (rel_r + U)
    t = n * gamma_ + beta
    e = gamma_.abs() * e_n + U * ((n * gamma_).abs() + t.abs())
    r = t * rs
    e = abs(rs) * e + U * r.abs()
    if x is not None:
        r = r + x
        e = e + U * r.abs()
    if cy is not None:
        cg = cy * gate[torch.arange(u.shape[0], device=u.device) // L_LN]
        e = e + U * (cg.abs() + (r + cg).abs())
    return e * (1 + 1e-6)


def window_attention(sd, pre, qkv, x_size, ws, heads, shifted, table, index, mask):
    """mixed_attn_block_efficient.py:128-165."""
    H, W = x_size
    B, L, C = qkv.shape
    s = ws[0] // 2 if shifted else 0
    t = qkv.view(B, H, W, C)
    if s > 0:
        t = torch.roll(t, shifts=(-s, -s), dims=(1, 2))
    t = partition(t, ws).reshape(-1, prod(ws), C)
    B_, N, _ = t.shape
    t = t.reshape(B_, N, 3, heads, -1).permute(2, 0, 3, 1, 4)
    x = cosine_attention(sd, pre + "attn_transform.", t[0], t[1], t[2], table, index, mask)
    x = unpartition(x.view(-1, ws[0], ws[1], C // 3), ws, x_size)
    if s > 0:
        x = torch.roll(x, shifts=(s, s), dims=(1, 2))
    return x.reshape(B, L, C // 3)


def stripe_attention(sd, pre, qkv, anchor, x_size, stripe_size, stripe_groups, shifted, df, heads,
                     table, index_a2w, index_w2a, mask_a2w, mask_w2a):
    """mixed_attn_block_efficient.py:215-270."""
    H, W = x_size
    B, L, C = qkv.shape
    ss, sh = stripe_info(stripe_size, stripe_groups, shifted, x_size)
    ass, ash = [s // df for s in ss], [s // df for s in sh]
    t = qkv.view(B, H, W, C)
    if shifted:
        t = torch.roll(t, shifts=(-sh[0], -sh[1]), dims=(1, 2))
        anchor = torch.roll(anchor, shifts=(-ash[0], -ash[1]), dims=(1, 2))
    t = partition(t, ss).reshape(-1, prod(ss), C)
    a = partition(anchor, ass).reshape(-1, prod(ass), C // 3)
    B_, N1, _ = t.shape
    N2 = a.shape[1]
    t = t.reshape(B_, N1, 3, heads, -1).permute(2, 0, 3, 1, 4)
    a = a.reshape(B_, N2, heads, -1).permute(0, 2, 1, 3)
    x = cosine_attention(sd, pre + "attn_transform1.", a, t[1], t[2], table, index_a2w, mask_a2w, False)
    x = cosine_attention(sd, pre + "attn_transform2.", t[0], a, x, table, index_w2a, mask_w2a)
    x = unpartition(x.view(B_, ss[0], ss[1], C // 3), ss, x_size)
    if shifted:
        x = torch.roll(x, shifts=sh, dims=(1, 2))
    return x.reshape(B, H * W, C // 3)


def anchor_projection(sd, pre, x, x_size, df):
    """mixed_attn_block.py:714-736 (AnchorLinear, avgpool, one stage)."""
    B, L, C = x.shape
    t = x.transpose(1, 2).view(B, C, *x_size)
    t = F.avg_pool2d(t, df, df).flatten(2).transpose(1, 2)
    t = F.linear(t, sd[pre + "body.0.reduction.weight"], sd[pre + "body.0.reduction.bias"])
    return t.view(B, x_size[0] // df, x_size[1] // df, -1)


def block_tables(tim, stripe_type, win_shift, stripe_shift):
    """mixed_attn_block_efficient.py:510-537."""
    d = "sv" if stripe_type == "W" else "sh"
    return dict(
        table_w=tim["table_w"], index_w=tim["index_w"], mask_w=tim["mask_w"] if win_shift else None,
        table_s=tim["table_" + d], index_a2w=tim[f"index_{d}_a2w"], index_w2a=tim[f"index_{d}_w2a"],
        mask_a2w=tim[f"mask_{d}_a2w"] if stripe_shift else None,
        mask_w2a=tim[f"mask_{d}_w2a"] if stripe_shift else None,
    )


def mixed_attention(sd, pre, x, x_size, bc, t, taps=None):
    """mixed_attn_block_efficient.py:351-381.  `bc` = per-block settings from block_settings()."""
    B, L, C = x.shape
    qkv = F.linear(x, sd[pre + "qkv.body.weight"], sd[pre + "qkv.body.bias"])
    qkv_w, qkv_s = torch.split(qkv, C * 3 // 2, dim=-1)
    anchor = anchor_projection(sd, pre + "anchor.", x, x_size, bc["df"])
    xw = window_attention(sd, pre + "window_attn.", qkv_w, x_size, bc["ws"], bc["heads_w"], bc["win_shift"],
                          t["table_w"], t["index_w"], t["mask_w"])
    xs = stripe_attention(sd, pre + "stripe_attn.", qkv_s, anchor, x_size, bc["stripe_size"], bc["stripe_groups"],
                          bc["stripe_shift"], bc["df"], bc["heads_s"], t["table_s"], t["index_a2w"],
                          t["index_w2a"], t["mask_a2w"], t["mask_w2a"])
    out = F.linear(torch.cat([xw, xs], dim=-1), sd[pre + "proj.weight"], sd[pre + "proj.bias"])
    if taps is not None:
        taps.update(qkv=qkv, anchor=anchor, x_window=xw, x_stripe=xs, attn_out=out)
    return out


def cab(sd, pre, x, x_size):
    """mixed_attn_block.py:948-983 (CAB + ChannelAttention)."""
    B, L, C = x.shape
    t = x.transpose(1, 2).view(B, C, *x_size).contiguous()
    t = F.conv2d(t, sd[pre + "cab.0.weight"], sd[pre + "cab.0.bias"], padding=1)
    t = F.conv2d(F.gelu(t), sd[pre + "cab.2.weight"], sd[pre + "cab.2.bias"], padding=1)
    g = F.adaptive_avg_pool2d(t, 1)
    g = torch.relu(F.conv2d(g, sd[pre + "cab.3.attention.1.weight"], sd[pre + "cab.3.attention.1.bias"]))
    g = torch.sigmoid(F.conv2d(g, sd[pre + "cab.3.attention.3.weight"], sd[pre + "cab.3.attention.3.bias"]))
    return (t * g).flatten(2).transpose(1, 2)


def mlp(sd, pre, x):
    """swin_v1_block.py:37-43 (GELU = exact erf form)."""
    return F.linear(F.gelu(F.linear(x, sd[pre + "fc1.weight"], sd[pre + "fc1.bias"])),
                    sd[pre + "fc2.weight"], sd[pre + "fc2.bias"])


def layer_norm(sd, pre, x):
    return F.layer_norm(x, (x.shape[-1],), sd[pre + "weight"], sd[pre + "bias"], 1e-5)


def block_settings(cfg, stage, i):
    """models/networks/grl.py:104-132 (per-block schedule) + efficient.py:466-471 (W-type swap)."""
    c = full_config(cfg)
    stype = "H" if i % 2 == 0 else "W"
    ss, sg = list(c["stripe_size"]), list(c["stripe_groups"])
    if stype == "W":
        ss, sg = ss[::-1], sg[::-1]
    return dict(
        ws=pair(c["window_size"]), win_shift=(i % 2 == 0), stripe_type=stype,
        stripe_shift=(i % 4 in [2, 3]) if c["stripe_shift"] else False,
        stripe_size=ss, stripe_groups=sg, df=c["anchor_window_down_factor"],
        heads_w=c["num_heads_window"][stage], heads_s=c["num_heads_stripe"][stage],
        local_connection=c["local_connection"], res_scale=0.1 if c["init_method"] == "r" else 1.0,
    )


def transformer_block(sd, pre, x, x_size, bc, tim, taps=None):
    """mixed_attn_block_efficient.py:539-556 (post-norm residual block)."""
    t = block_tables(tim, bc["stripe_type"], bc["win_shift"], bc["stripe_shift"])
    a = layer_norm(sd, pre + "norm1.", mixed_attention(sd, pre + "attn.", x, x_size, bc, t, taps))
    if bc["local_connection"]:
        x = x + bc["res_scale"] * a + cab(sd, pre + "conv.", x, x_size)
    else:
        x = x + bc["res_scale"] * a
    if taps is not None:
        taps["after_attn"] = x
    x = x + bc["res_scale"] * layer_norm(sd, pre + "norm2.", mlp(sd, pre + "mlp.", x))
    return x


def transformer_stage(sd, cfg, stage, x, x_size, tim):
    """models/networks/grl.py:164-170."""
    c = full_config(cfg)
    pre = f"layers.{stage}."
    r = x
    for i in range(c["depths"][stage]):
        r = transformer_block(sd, f"{pre}blocks.{i}.", r, x_size, block_settings(cfg, stage, i), tim)
    B, L, C = r.shape
    t = r.transpose(1, 2).view(B, C, *x_size)
    t = F.conv2d(t, sd[pre + "conv.weight"], sd[pre + "conv.bias"], padding=1)
    return t.flatten(2).transpose(1, 2) + x


def forward_features(sd, cfg, x):
    """models/networks/grl.py:491-504."""
    c = full_config(cfg)
    x_size = (x.shape[2], x.shape[3])
    t = layer_norm(sd, "norm_start.", x.flatten(2).transpose(1, 2))
    tim = {k: v.to(x.device, x.dtype) if v.is_floating_point() else v.to(x.device)
           for k, v in table_index_mask(cfg, x_size).items()}
    for s in range(len(c["depths"])):
        t = transformer_stage(sd, cfg, s, t, x_size, tim)
    t = layer_norm(sd, "norm_end.", t)
    return t.transpose(1, 2).view(x.shape[0], -1, *x_size)


def grl_forward(sd, cfg, x):
    """models/networks/grl.py:479-551 (check_image_size + forward)."""
    c = full_config(cfg)
    conv = lambda n, t: F.conv2d(t, sd[n + ".weight"], sd[n + ".bias"], padding=1)
    H, W = x.shape[2:]
    p = pad_size(cfg)
    ph, pw = (p - H % p) % p, (p - W % p) % p
    try:
        x = F.pad(x, (0, pw, 0, ph), "reflect")
    except BaseException:
        x = F.pad(x, (0, pw, 0, ph), "constant")
    if c["in_channels"] == 3:
        mean = torch.tensor((0.4488, 0.4371, 0.4040), dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    else:
        mean = torch.zeros(1, 1, 1, 1, dtype=x.dtype, device=x.device)
    x = (x - mean) * c["img_range"]
    up = c["upsampler"]
    if up in ("pixelshuffle", "pixelshuffledirect", "nearest+conv"):
        x = conv("conv_first", x)
        x = conv("conv_after_body", forward_features(sd, cfg, x)) + x
        if up == "pixelshuffle":
            x = F.leaky_relu(conv("conv_before_upsample.0", x), 0.01)
            s = c["upscale"]
            if s & (s - 1) == 0:  # upsample.py:16-20
                n = 0
                while (1 << n) < s:
                    x = F.pixel_shuffle(conv(f"upsample.up.{2 * n}", x), 2)
                    n += 1
            elif s == 3:
                x = F.pixel_shuffle(conv("upsample.up.0", x), 3)
            else:
                raise ValueError(f"scale {s} is not supported")
            x = conv("conv_last", x)
        elif up == "pixelshuffledirect":
            x = F.pixel_shuffle(conv("upsample.up.0", x), c["upscale"])
        else:
            x = F.leaky_relu(conv("conv_before_upsample.0", x), 0.01)
            x = F.leaky_relu(conv("conv_up1", F.interpolate(x, scale_factor=2, mode="nearest")), 0.2)
            x = F.leaky_relu(conv("conv_up2", F.interpolate(x, scale_factor=2, mode="nearest")), 0.2)
            x = conv("conv_last", F.leaky_relu(conv("conv_hr", x), 0.2))
    else:
        first = conv("conv_first", x)
        res = conv("conv_after_body", forward_features(sd, cfg, first)) + first
        x = x + conv("conv_last", res) if c["in_channels"] == c["out_channels"] else conv("conv_last", res)
    x = x / c["img_range"] + mean
    return x[:, :, : H * c["upscale"], : W * c["upscale"]]


# --------------------------------------------------------------------------------------
# metric (the PSNR the reference's validation_step reports)
# --------------------------------------------------------------------------------------


def tensor_round(img, data_range=1.0):
    """utils/utils_image.py:30-33."""
    img = img.clamp(0.0, 1.0 * data_range)
    return (img * 255.0 / data_range).round() * data_range / 255.0


def psnr(restored, target, border=0):
    """utils/metrics/psnr.py:44-48 after tensor_round, with the SR border shave of engines/base.py:265-267."""
    a, b = tensor_round(restored), tensor_round(target)
    if border > 0:
        a, b = a[..., border:-border, border:-border], b[..., border:-border, border:-border]
    return -10 * (a - b).pow(2).mean([-3, -2, -1]).log10()


# --------------------------------------------------------------------------------------
# weights: parameter shapes (SURVEY.md Appendix C) and seeded synthetic state dicts
# --------------------------------------------------------------------------------------


def param_shapes(cfg):
    """Names/shapes of every parameter of models.networks.grl.GRL for `cfg` (Appendix C)."""
    c = full_config(cfg)
    C, cin, cout = c["embed_dim"], c["in_channels"], c["out_channels"]
    hid = int(C * c["mlp_ratio"])
    sh = {"conv_first.weight": (C, cin, 3, 3), "conv_first.bias": (C,)}
    for n in ("norm_start", "norm_end"):
        sh[n + ".weight"], sh[n + ".bias"] = (C,), (C,)
    for s, depth in enumerate(c["depths"]):
        for i in range(depth):
            p = f"layers.{s}.blocks.{i}."
            sh[p + "attn.qkv.body.weight"], sh[p + "attn.qkv.body.bias"] = (3 * C, C), (3 * C,)
            sh[p + "attn.anchor.body.0.reduction.weight"] = (C // 2, C)
            sh[p + "attn.anchor.body.0.reduction.bias"] = (C // 2,)
            for tr, h in (("window_attn.attn_transform", c["num_heads_window"][s]),
                          ("stripe_attn.attn_transform1", c["num_heads_stripe"][s]),
                          ("stripe_attn.attn_transform2", c["num_heads_stripe"][s])):
                q = f"{p}attn.{tr}."
                sh[q + "logit_scale"] = (h, 1, 1)
                sh[q + "cpb_mlp.0.weight"], sh[q + "cpb_mlp.0.bias"] = (512, 2), (512,)
                sh[q + "cpb_mlp.2.weight"] = (h, 512)
            sh[p + "attn.proj.weight"], sh[p + "attn.proj.bias"] = (C, C), (C,)
            for n in ("norm1", "norm2"):
                sh[p + n + ".weight"], sh[p + n + ".bias"] = (C,), (C,)
            if c["local_connection"]:
                sh[p + "conv.cab.0.weight"], sh[p + "conv.cab.0.bias"] = (C // 4, C, 3, 3), (C // 4,)
                sh[p + "conv.cab.2.weight"], sh[p + "conv.cab.2.bias"] = (C, C // 4, 3, 3), (C,)
                sh[p + "conv.cab.3.attention.1.weight"] = (C // 18, C, 1, 1)
                sh[p + "conv.cab.3.attention.1.bias"] = (C // 18,)
                sh[p + "conv.cab.3.attention.3.weight"] = (C, C // 18, 1, 1)
                sh[p + "conv.cab.3.attention.3.bias"] = (C,)
            sh[p + "mlp.fc1.weight"], sh[p + "mlp.fc1.bias"] = (hid, C), (hid,)
            sh[p + "mlp.fc2.weight"], sh[p + "mlp.fc2.bias"] = (C, hid), (C,)
        sh[f"layers.{s}.conv.weight"], sh[f"layers.{s}.conv.bias"] = (C, C, 3, 3), (C,)
    sh["conv_after_body.weight"], sh["conv_after_body.bias"] = (C, C, 3, 3), (C,)
    up, s = c["upsampler"], c["upscale"]
    if up == "pixelshuffle":
        sh["conv_before_upsample.0.weight"], sh["conv_before_upsample.0.bias"] = (64, C, 3, 3), (64,)
        if s & (s - 1) == 0:
            n = 0
            while (1 << n) < s:
                sh[f"upsample.up.{2 * n}.weight"], sh[f"upsample.up.{2 * n}.bias"] = (256, 64, 3, 3), (256,)
                n += 1
        else:
            sh["upsample.up.0.weight"], sh["upsample.up.0.bias"] = (576, 64, 3, 3), (576,)
        sh["conv_last.weight"], sh["conv_last.bias"] = (cout, 64, 3, 3), (cout,)
    elif up == "pixelshuffledirect":
        sh["upsample.up.0.weight"], sh["upsample.up.0.bias"] = (s * s * cout, C, 3, 3), (s * s * cout,)
    elif up == "nearest+conv":
        sh["conv_before_upsample.0.weight"], sh["conv_before_upsample.0.bias"] = (64, C, 3, 3), (64,)
        for n in ("conv_up1", "conv_up2", "conv_hr"):
            sh[n + ".weight"], sh[n + ".bias"] = (64, 64, 3, 3), (64,)
        sh["conv_last.weight"], sh["conv_last.bias"] = (cout, 64, 3, 3), (cout,)
    else:
        sh["conv_last.weight"], sh["conv_last.bias"] = (cout, C, 3, 3), (cout,)
    return sh


def synth_state_dict(cfg, seed=0, style="spread"):
    """Deterministic synthetic weights shared by reference, oracle and candidate (SURVEY.md 8c):
    one generator per parameter *name* (so the values do not depend on module construction order).
    style "spread" (default, used by every golden fixture): fan-in scaled weights, non-trivial biases / LayerNorm
    affine, and logit_scale spread over [ln 5, ln 150] so the clamp at ln 100 is exercised -- a deliberately harsh,
    near-chaotic network.  style "init": the distribution the reference's own constructor produces
    (grl.py:455-462: Linear ~ trunc_normal(std 0.02) with zero bias, LayerNorm identity, logit_scale = ln 10,
    Conv2d = PyTorch's default kaiming-uniform), i.e. what an untrained reference model computes.
    style "routed": "init" with every parameter that routes per head or per row made distinct, so that a swapped,
    misordered or dropped one changes the output: per-head logit_scale over [ln 5, ln 150] (a different draw for the
    window, stripe-1 and stripe-2 transforms), cpb_mlp weights as in "spread" plus a random cpb_mlp.0.bias, Linear
    biases ~ N(0, 0.02), LayerNorm weight 1 + 0.1 N and bias 0.02 N (cpb_mlp.0.bias: 0.1 N).  The overrides draw from a
    second per-name generator, so "init" and "spread" are unchanged."""
    import zlib

    if style not in ("spread", "init", "routed"):
        raise ValueError(f"unknown weight style {style!r}")
    sd = {}
    for name, shape in sorted(param_shapes(cfg).items()):
        g = torch.Generator().manual_seed((zlib.crc32(name.encode()) + 7919 * seed) % (2 ** 31))
        if style in ("init", "routed"):
            linear_bias = False
            if name.endswith("logit_scale"):
                v = torch.full(shape, log(10.0))
            elif ".norm" in name or name.startswith("norm_"):
                v = torch.ones(shape) if name.endswith("weight") else torch.zeros(shape)
            elif len(shape) == 4 or (name.endswith("bias") and (name.startswith("conv") or ".conv." in name
                                                                 or ".cab." in name or name.startswith("upsample"))):
                fan_in = prod(param_shapes(cfg)[name.replace(".bias", ".weight")][1:])
                bound = 1.0 / fan_in ** 0.5
                v = (torch.rand(shape, generator=g) * 2 - 1) * bound
            elif name.endswith("bias"):
                v = torch.zeros(shape)
                linear_bias = True
            else:
                v = torch.nn.init.trunc_normal_(torch.empty(shape), std=0.02, generator=g)
            if style == "routed":
                r = torch.Generator().manual_seed((zlib.crc32(name.encode()) + 7919 * seed + 104729) % (2 ** 31))
                if name.endswith("logit_scale"):
                    v = log(5.0) + (log(150.0) - log(5.0)) * torch.rand(shape, generator=r)
                elif "cpb_mlp" in name:
                    v = torch.randn(shape, generator=r) * (0.7 if name.endswith("0.weight") else
                                                           0.15 if name.endswith("2.weight") else 0.1)
                elif ".norm" in name or name.startswith("norm_"):
                    v = (1.0 + 0.1 * torch.randn(shape, generator=r)) if name.endswith("weight") else \
                        0.02 * torch.randn(shape, generator=r)
                elif linear_bias:
                    v = 0.02 * torch.randn(shape, generator=r)
            sd[name] = v.float()
            continue
        if name.endswith("logit_scale"):
            v = log(5.0) + (log(150.0) - log(5.0)) * torch.rand(shape, generator=g)
        elif ".norm" in name or name.startswith("norm_"):
            v = (1.0 + 0.2 * torch.randn(shape, generator=g)) if name.endswith("weight") else 0.1 * torch.randn(shape, generator=g)
        elif name.endswith("bias"):
            v = 0.05 * torch.randn(shape, generator=g)
        elif "cpb_mlp" in name:
            v = torch.randn(shape, generator=g) * (0.7 if name.endswith("0.weight") else 0.15)
        else:
            fan_in = prod(shape[1:])
            v = torch.randn(shape, generator=g) * (1.0 / fan_in) ** 0.5
        sd[name] = v.float()
    return sd


def synth_input(shape, seed=1234, noise_sigma=0.0):
    """SURVEY.md 8d: rand in [0,1]; denoise inputs add (sigma/255) randn, unclamped."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(shape, generator=g)
    if noise_sigma > 0:
        x = x + (noise_sigma / 255.0) * torch.randn(shape, generator=g)
    return x
