"""The tensor-core attention kernel (csrc/attn_tc.cu) on every launch path the released configs take, against a float64
emulation of its own algorithm (grl_oracle.attn_launch_reference).

A launch's path is its signature (`path`): the key-window template KW, whether the last query tile (128 rows) and key tile
(64 keys) are full, the TMA box widths of the query and key grids, dense V / dense output, the ones column and the shift
mask.  The image size does not enter it.  CASES and ZOO_CASES hold one minimal problem per signature, taken from the
first released (config, block, pass) that launches it: 2 x 2 windows of that pass's grid and B = 2 (an interior window, a
masked and wrapped boundary window and a batch offset), the config's heads and head_dim, in the packed production
layout.  test_released_attention_paths_have_cases (CPU) walks every block of every architecture of archs.architectures
through tc.attention_launches, the descriptors BlockPlan.run launches, and fails on a signature without a case.

The gate bounds |got - emulated| in ulps of the output format, taken at max(|emulated|, the row's rms).  The emulation
differs from the kernel only in the fp32 summation order of the wgmma products and in ex2.approx, so almost every element
agrees bit for bit; the rest are flipped roundings of one P or of the output (the fraction is printed).  Each case also reports |emulated - exact|,
the error the design accepts.  Mutation controls derived from the emulation (a kernel bug's effect, never an edited
kernel) must fail the gate wherever they apply.
"""
import math
from typing import NamedTuple

import pytest
import torch

import archs
import grl_oracle as O

ATTN_VARIANTS = [5, 0]  # grl_tc_attn_variant: 5 = TMA boxes where the geometry has them (default), 0 = cp.async gathers
B = 2
GATE_ULP = 6.0  # max |got - emulated| in output ulps: 2 x the worst unmutated case (3.0 ulp, H100 80GB HBM3 at 400 W)
GATE_CHAIN = 10.0  # both stripe passes against the chained emulation: 2 x the worst case (4.75 ulp, same card)


class AttnCase(NamedTuple):
    src: str      # the first released config / block that launches this path (or why an extra case exists)
    role: str     # "window", "stripe1" (anchors attend to the stripe's tokens), "stripe2" (tokens attend to anchors)
    win: tuple    # the token window of the pass: the attention window or the (oriented) stripe
    df: int       # anchor down factor (1 for window attention)
    shifted: bool
    heads: int
    d: int        # head_dim: < 32 runs the ones column
    grow: float = 0.0  # > 0: a bias that grows by `grow` log2 units per key row (the lazy-rescale path)


CASES = [
    AttnCase("tiny/sr/b0", "window", (32, 32), 1, True, 2, 16),
    AttnCase("tiny/sr/b0", "stripe1", (64, 64), 4, False, 2, 16),
    AttnCase("tiny/sr/b0", "stripe2", (64, 64), 4, False, 2, 16),
    AttnCase("tiny/sr/b1", "window", (32, 32), 1, False, 2, 16),
    AttnCase("tiny/sr/b2", "stripe1", (64, 64), 4, True, 2, 16),
    AttnCase("tiny/sr/b2", "stripe2", (64, 64), 4, True, 2, 16),
    AttnCase("tiny/dn/b0", "window", (16, 16), 1, True, 2, 16),
    AttnCase("tiny/dn/b0", "stripe1", (64, 128), 4, False, 2, 16),
    AttnCase("tiny/dn/b0", "stripe2", (64, 128), 4, False, 2, 16),
    AttnCase("tiny/dn/b1", "window", (16, 16), 1, False, 2, 16),
    AttnCase("tiny/dn/b2", "stripe1", (64, 128), 4, True, 2, 16),
    AttnCase("tiny/dn/b2", "stripe2", (64, 128), 4, True, 2, 16),
    AttnCase("tiny/deblur/b0", "window", (12, 12), 1, True, 2, 16),
    AttnCase("tiny/deblur/b0", "stripe1", (48, 96), 4, False, 2, 16),
    AttnCase("tiny/deblur/b0", "stripe2", (48, 96), 4, False, 2, 16),
    AttnCase("tiny/deblur/b1", "window", (12, 12), 1, False, 2, 16),
    AttnCase("tiny/deblur/b1", "stripe1", (96, 48), 4, False, 2, 16),
    AttnCase("tiny/deblur/b1", "stripe2", (96, 48), 4, False, 2, 16),
    AttnCase("tiny/deblur/b2", "stripe1", (48, 96), 4, True, 2, 16),
    AttnCase("tiny/deblur/b2", "stripe2", (48, 96), 4, True, 2, 16),
    AttnCase("tiny/deblur/b3", "stripe1", (96, 48), 4, True, 2, 16),
    AttnCase("tiny/deblur/b3", "stripe2", (96, 48), 4, True, 2, 16),
    AttnCase("tiny/jpeg/b1", "stripe1", (144, 72), 4, False, 2, 16),
    AttnCase("tiny/jpeg/b1", "stripe2", (144, 72), 4, False, 2, 16),
    AttnCase("tiny/jpeg/b3", "stripe1", (144, 72), 4, True, 2, 16),
    AttnCase("tiny/jpeg/b3", "stripe2", (144, 72), 4, True, 2, 16),
    AttnCase("tiny/dm/b0", "window", (8, 8), 1, True, 2, 16),
    AttnCase("tiny/dm/b0", "stripe1", (32, 32), 4, False, 2, 16),
    AttnCase("tiny/dm/b0", "stripe2", (32, 32), 4, False, 2, 16),
    AttnCase("tiny/dm/b1", "window", (8, 8), 1, False, 2, 16),
    AttnCase("tiny/dm/b2", "stripe1", (32, 32), 4, True, 2, 16),
    AttnCase("tiny/dm/b2", "stripe2", (32, 32), 4, True, 2, 16),
    AttnCase("small/sr/b0", "window", (32, 32), 1, True, 2, 32),
    AttnCase("small/sr/b0", "stripe1", (64, 64), 4, False, 2, 32),
    AttnCase("small/sr/b0", "stripe2", (64, 64), 4, False, 2, 32),
    AttnCase("small/sr/b1", "window", (32, 32), 1, False, 2, 32),
    AttnCase("small/sr/b2", "stripe1", (64, 64), 4, True, 2, 32),
    AttnCase("small/sr/b2", "stripe2", (64, 64), 4, True, 2, 32),
    AttnCase("small/dn/b0", "window", (16, 16), 1, True, 2, 32),
    AttnCase("small/dn/b0", "stripe1", (64, 128), 4, False, 2, 32),
    AttnCase("small/dn/b0", "stripe2", (64, 128), 4, False, 2, 32),
    AttnCase("small/dn/b1", "window", (16, 16), 1, False, 2, 32),
    AttnCase("small/dn/b2", "stripe1", (64, 128), 4, True, 2, 32),
    AttnCase("small/dn/b2", "stripe2", (64, 128), 4, True, 2, 32),
    AttnCase("small/deblur/b0", "window", (12, 12), 1, True, 2, 32),
    AttnCase("small/deblur/b0", "stripe1", (48, 96), 4, False, 2, 32),
    AttnCase("small/deblur/b0", "stripe2", (48, 96), 4, False, 2, 32),
    AttnCase("small/deblur/b1", "window", (12, 12), 1, False, 2, 32),
    AttnCase("small/deblur/b1", "stripe1", (96, 48), 4, False, 2, 32),
    AttnCase("small/deblur/b1", "stripe2", (96, 48), 4, False, 2, 32),
    AttnCase("small/deblur/b2", "stripe1", (48, 96), 4, True, 2, 32),
    AttnCase("small/deblur/b2", "stripe2", (48, 96), 4, True, 2, 32),
    AttnCase("small/deblur/b3", "stripe1", (96, 48), 4, True, 2, 32),
    AttnCase("small/deblur/b3", "stripe2", (96, 48), 4, True, 2, 32),
    AttnCase("small/jpeg/b1", "stripe1", (144, 72), 4, False, 2, 32),
    AttnCase("small/jpeg/b1", "stripe2", (144, 72), 4, False, 2, 32),
    AttnCase("small/jpeg/b3", "stripe1", (144, 72), 4, True, 2, 32),
    AttnCase("small/jpeg/b3", "stripe2", (144, 72), 4, True, 2, 32),
    AttnCase("small/dm/b0", "window", (8, 8), 1, True, 2, 32),
    AttnCase("small/dm/b0", "stripe1", (32, 32), 4, False, 2, 32),
    AttnCase("small/dm/b0", "stripe2", (32, 32), 4, False, 2, 32),
    AttnCase("small/dm/b1", "window", (8, 8), 1, False, 2, 32),
    AttnCase("small/dm/b2", "stripe1", (32, 32), 4, True, 2, 32),
    AttnCase("small/dm/b2", "stripe2", (32, 32), 4, True, 2, 32),
    AttnCase("base/sr/b0", "stripe1", (64, 64), 2, False, 3, 30),
    AttnCase("base/sr/b2", "stripe1", (64, 64), 2, True, 3, 30),
    AttnCase("base/sr/b2", "stripe2", (64, 64), 2, True, 3, 30),
    AttnCase("base/dn/b0", "stripe1", (64, 128), 2, False, 3, 30),
    AttnCase("base/dn/b0", "stripe2", (64, 128), 2, False, 3, 30),
    AttnCase("base/dn/b2", "stripe1", (64, 128), 2, True, 3, 30),
    AttnCase("base/dn/b2", "stripe2", (64, 128), 2, True, 3, 30),
]

EXTRAS = [
    AttnCase("extra: 8 heads, the kernel's limit", "window", (32, 32), 1, True, 8, 16),
    AttnCase("extra: 4x8 window, 32 keys in one partial tile", "window", (4, 8), 1, False, 2, 32),
    AttnCase("extra: 8x16 stripes, df 2", "stripe2", (8, 16), 2, True, 2, 32),
    AttnCase("extra: 64x64 stripes, df 2, head_dim 32", "stripe2", (64, 64), 2, True, 3, 32),
    AttnCase("extra: 32x16 stripes, df 4", "stripe2", (32, 16), 4, False, 2, 32),
    AttnCase("extra: 48x96 stripes, 1 head", "stripe2", (48, 96), 4, True, 1, 32),
    AttnCase("extra: lazy rescale, KW 32", "window", (32, 32), 1, False, 3, 32, 0.6),
    AttnCase("extra: lazy rescale, KW 32", "window", (32, 32), 1, True, 3, 30, 6.0),
    AttnCase("extra: lazy rescale, generic KW (jpeg window)", "window", (36, 36), 1, False, 3, 32, 0.6),
    AttnCase("extra: lazy rescale, generic KW (jpeg window)", "window", (36, 36), 1, True, 3, 30, 6.0),
]
# released paths outside the VARIANTS x TASKS grid of archs: GRL-Base blind SR's stripe pass 1 over 64 x 32 stripes
# with df 4 (16 x 8 anchor windows).  They come after EXTRAS because a case's seed is its index in the case list.
ZOO_CASES = [
    AttnCase("base/bsr/b1", "stripe1", (64, 32), 4, False, 3, 30),
    AttnCase("base/bsr/b3", "stripe1", (64, 32), 4, True, 3, 30),
]

# key-window widths with their own template instance in grl_tc_attn's switch (attn_tc.cu); any other width runs KW = 0
KW_TEMPLATES = (8, 16, 32, 64, 128)


def path(capi, ln):
    """Launch-path signature: (KW, last query tile full, last key tile full, box_q, box_k, v_dense, o_dense, ones_col,
    use_mask)."""
    box = capi.lib().grl_tc_attn_box_tokens
    nq, nk = ln.gq.wh * ln.gq.ww, ln.gk.wh * ln.gk.ww
    return (ln.gk.ww if ln.gk.ww in KW_TEMPLATES else 0, nq % 128 == 0, nk % 64 == 0, box(ln.gq), box(ln.gk),
            ln.v_dense, ln.o_dense, ln.ones_col, ln.use_mask)


def case_launch(case):
    """(x_size, launch descriptor) of a case: an image of 2 x 2 windows of the pass's grid."""
    from grl_image_restoration_b200 import geometry as G, tc

    wh, ww = case.win
    x_size = (2 * wh, 2 * ww)
    sh = (wh // 2, ww // 2) if case.shifted else (0, 0)
    tok = G.token_grid(x_size, case.win, sh)
    gq = gk = tok
    if case.role != "window":
        anc = G.anchor_grid(x_size, case.win, sh, case.df)
        gq, gk = (anc, tok) if case.role == "stripe1" else (tok, anc)
    return x_size, tc.attention_launch(case.role, gq, gk, case.heads, case.heads, case.heads * case.d, case.shifted)


def test_released_attention_paths_have_cases(pkg):
    """Every launch path of every block of every architecture of archs.architectures has a case, and every case of CASES
    and ZOO_CASES is a launched path."""
    from grl_image_restoration_b200 import capi, tc

    cases = [(path(capi, case_launch(c)[1]), c) for c in CASES + ZOO_CASES]
    assert len(dict(cases)) == len(cases), "two cases share a path"
    launched = [(path(capi, ln), f"{name} stage {si} block {bi} {ln.role}")
                for name, model, shape in archs.architectures(pkg, "fp16")
                for si, layer in enumerate(model.layers) for bi, blk in enumerate(layer.blocks)
                for ln in tc.attention_launches(blk, shape[2:])]
    archs.check_walk("tensor-core attention", launched, cases, [(path(capi, case_launch(c)[1]), c) for c in EXTRAS])


# ----------------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope="module", params=ATTN_VARIANTS, ids=lambda v: f"attn{v}")
def tc(pkg, device, request):
    from grl_image_restoration_b200 import capi, tc as T

    if capi.lib().grl_device_ok() != 1:
        pytest.skip("wgmma path needs sm_90")
    prev = capi.lib().grl_tc_attn_variant(request.param)
    yield T
    capi.lib().grl_tc_attn_variant(prev)


def grid_t(g):
    return (g.H, g.W, g.wh, g.ww, g.sh, g.sw)


def ulp(x, dtype):
    """Spacing of `dtype` at |x| (float64), subnormal spacing at the bottom."""
    fi = torch.finfo(dtype)
    e = torch.frexp(x.abs())[1]
    return torch.clamp(fi.eps * torch.exp2((e - 1).double()), min=fi.tiny * fi.eps)


def compare(got, emul, d, dtype):
    """(max |got - emul| in ulps at max(|emul|, row rms), fraction of elements that differ) over the d real columns."""
    g, e = got[..., :d].double(), emul[..., :d]
    rms = e.pow(2).mean(-1, keepdim=True).sqrt()
    diff = (g - e).abs()
    return float((diff / ulp(torch.maximum(e.abs(), rms), dtype)).max()), float((diff != 0).double().mean())


def fails_gate(stats):
    return stats[0] > GATE_ULP


def old_bound_catches(m, exact, d):
    """The bound of the operator tests this file replaces: max-abs 4e-2 * max(1, |ref|), mean 6e-3."""
    err = (m[..., :d] - exact[..., :d]).abs()
    return bool(err.max() > 4e-2 * max(1.0, float(exact[..., :d].abs().max())) or err.mean() > 6e-3)


def block_inputs(case, x_size, dtype, device, seed, batch=B):
    """Packed operands of one block, as the projection epilogues write them: qkv (B*L, 6*heads*32) in slot order
    [window q|k|v][stripe q|k|v] x head and anchor (B*La, heads*32).  q, k and anchors are L2-normalised over head_dim;
    window q, stripe q and stripe k carry exp(min(s, ln 100)) log2 e with a per-head s in [ln 5, ln 150]; with
    head_dim < 32 column 31 of every value slot is 1.  `batch` images of x_size."""
    h, d = case.heads, case.d
    H, W = x_size
    g = torch.Generator(device=device).manual_seed(seed)
    qkv = torch.zeros(batch * H * W, 6 * h, 32, device=device)
    qkv[..., :d] = torch.randn(batch * H * W, 6 * h, d, generator=g, device=device)
    for grp, scaled in ((0, True), (1, False), (3, True), (4, True)):
        s = math.log(5.0) + (math.log(150.0) - math.log(5.0)) * torch.rand(h, generator=g, device=device)
        scale = torch.exp(s.clamp(max=math.log(100.0))) * O.LOG2E if scaled else torch.ones(h, device=device)
        qkv[:, grp * h:(grp + 1) * h, :d] = torch.nn.functional.normalize(qkv[:, grp * h:(grp + 1) * h, :d], dim=-1) * scale[:, None]
    if d < 32:
        qkv[:, 2 * h:3 * h, 31] = 1.0
        qkv[:, 5 * h:6 * h, 31] = 1.0
    La = (H // case.df) * (W // case.df)
    anc = torch.zeros(batch * La, h, 32, device=device)
    anc[..., :d] = torch.nn.functional.normalize(torch.randn(batch * La, h, d, generator=g, device=device), dim=-1)
    return qkv.view(batch * H * W, -1).to(dtype), anc.view(batch * La, -1).to(dtype)


def cpb_table(ln, seed, grow=0.0):
    """(heads, rows) 16 sigmoid(MLP(coords)) log2 e of a random CPB-like MLP over the launch's relative coordinates.
    grow > 0 adds -grow * (query row - key row): the row maximum keeps outgrowing the lazy reference."""
    gq, gk = ln.gq, ln.gk
    tg = gq if gq.wh >= gk.wh else gk
    df = tg.wh // min(gq.wh, gk.wh)
    coords = O.coords_table([tg.wh, tg.ww], df).reshape(-1, 2).double()
    g = torch.Generator().manual_seed(seed)
    w1, b1 = torch.randn(512, 2, generator=g).double() * 0.7, torch.randn(512, generator=g).double() * 0.1
    w2 = torch.randn(ln.heads, 512, generator=g).double() * 0.15
    t = (16 * torch.sigmoid(torch.relu(coords @ w1.T + b1) @ w2.T) * O.LOG2E).T.float().contiguous()
    assert t.shape[1] == (gq.wh + gk.wh - 1) * (gq.ww + gk.ww - 1)
    if grow:
        dh = torch.arange(t.shape[1]) // (gq.ww + gk.ww - 1) - (gk.wh - 1)
        t = t * 0.25 - grow * dh.float()
    return t


def operand(buf, spec, grid, heads, batch=B):
    """(Bw, heads, N, 32) view of a launch operand of `batch` images, in the kernel's window order."""
    name, col = spec
    if name == "x1":
        return buf[name].view(-1, heads, grid.wh * grid.ww, 32)
    t = buf[name].view(batch, grid.H, grid.W, -1)[..., col:col + heads * 32]
    return O.attn_windows(t, grid_t(grid), heads)


def run(tc, ln, buf, table, batch=B):
    tc.attention(ln.gq, ln.gk, buf[ln.q[0]], ln.q[1], buf[ln.k[0]], ln.k[1], buf[ln.v[0]], ln.v[1], buf[ln.out[0]],
                 ln.out[1], batch, ln.heads, tc.shifted_copies(table.to(buf["qkv"].device)), ln.use_mask, v_dense=ln.v_dense,
                 o_dense=ln.o_dense, ones_col=ln.ones_col)


GATED = ("bias entry read from its neighbour", "shift mask missing for one region pair", "key box taken without the roll",
         "query box taken without the roll", "rescale applied to O only")
SENTINEL = -7.25
_REF = {}  # (case, fmt) -> float64 references, shared by both attention variants


def check_pads(got, ln, d, what):
    if d < 32:
        assert bool((got[..., d:31] == 0).all()), f"{what}: pad columns {d}..30 not zero"
        assert bool((got[..., 31] == (1.0 if ln.ones_col else 0.0)).all()), f"{what}: column 31"


def mutations(ref_fn, ln, q, k, v, table, index, mask, tokens, variant):
    """Mutation controls on the last window (batch 1, bottom-right: masked and wrapped): name -> emulated output."""
    from grl_image_restoration_b200 import capi

    out = {}
    w = q.shape[0] - 1
    qw, kw, vw = q[w:], k[w:], v[w:]
    mw = None if mask is None else mask[w % mask.shape[0]][None]
    # the relative position whose neighbour's entry moves the softmax most: max over pairs of p (1 - p) |2^delta - 1|
    tab = table.to(q.device, torch.float64)
    x = qw.double() @ kw.double().transpose(-1, -2) + tab[:, index]
    if mw is not None:
        x = x + mw.double() * O.LOG2E
    p = torch.softmax(x * math.log(2.0), dim=-1)
    nb = (index + 1).clamp(max=tab.shape[1] - 1)
    hit = (p * (1 - p) * (torch.exp2(tab[:, nb] - tab[:, index]) - 1).abs()).reshape(-1, index.numel()).amax(0).argmax()
    r = int(index.flatten()[hit])
    out["bias entry read from its neighbour"] = ref_fn(qw, kw, vw, torch.where(index == r, r + 1, index), mw)
    out["last key dropped"] = ref_fn(qw, kw[:, :, :-1], vw[:, :, :-1], index[:, :-1], None if mw is None else mw[..., :-1])
    if mw is not None:
        nW = mask.shape[0]
        rq = O.region_ids(grid_t(ln.gq)[:2], grid_t(ln.gq)[2:4], grid_t(ln.gq)[4:6])[w % nW]
        rk = O.region_ids(grid_t(ln.gk)[:2], grid_t(ln.gk)[2:4], grid_t(ln.gk)[4:6])[w % nW]
        i, j = (mw[0] != 0).nonzero()[0].tolist()
        pair = ((rq[:, None] == rq[i]) & (rk[None, :] == rk[j])).to(mw.device)
        out["shift mask missing for one region pair"] = ref_fn(qw, kw, vw, index, torch.where(pair, 0.0, mw))
    if variant == 5:
        box = capi.lib().grl_tc_attn_box_tokens
        bk, bq = box(ln.gk), box(ln.gq)
        gk, gq = grid_t(ln.gk), grid_t(ln.gq)
        if bk and k.shape[2] >= 64 and (gk[4] or gk[5]):
            j = k.shape[2] // 64 * 64 - bk  # the last box of the last full key tile
            k2, v2 = kw.clone(), vw.clone()
            k2[:, :, j:j + bk] = tokens("k", gk[:4] + (0, 0))[w:, :, j:j + bk]
            if not ln.v_dense:
                v2[:, :, j:j + bk] = tokens("v", gk[:4] + (0, 0))[w:, :, j:j + bk]
            out["key box taken without the roll"] = ref_fn(qw, k2, v2, index, mw)
        elif bq and q.shape[2] >= 128 and (gq[4] or gq[5]):
            q2 = qw.clone()
            q2[:, :, :bq] = tokens("q", gq[:4] + (0, 0))[w:, :, :bq]
            out["query box taken without the roll"] = ref_fn(q2, kw, vw, index, mw)
    resc = ref_fn(qw, kw, vw, index, mw, mutation="rescale_o_only")
    if resc[2]["rescales"]:
        out["rescale applied to O only"] = resc
    out["denominator from the unrounded P"] = ref_fn(qw, kw, vw, index, mw, mutation="unrounded_denominator")
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", CASES + EXTRAS + ZOO_CASES, ids=lambda c: f"{c.src.split(':')[0]}-{c.role}-{c.win[0]}x{c.win[1]}"
                         f"-df{c.df}-{'s' if c.shifted else 'u'}-h{c.heads}d{c.d}" + (f"-grow{c.grow}" if c.grow else ""))
def test_attention_path(tc, device, case, fmt):
    from grl_image_restoration_b200 import capi

    variant = capi.lib().grl_tc_attn_variant(-1)
    x_size, ln = case_launch(case)
    sig = path(capi, ln)
    if variant == 0 and case in CASES:  # without TMA the box fields do not matter: one run per remaining signature
        first = next(c for c in CASES if path(capi, case_launch(c)[1])[:3] + path(capi, case_launch(c)[1])[5:]
                     == sig[:3] + sig[5:] and (c.heads, c.d) == (case.heads, case.d))
        if first != case:
            pytest.skip(f"same cp.async path as {first.src} {first.role}")
    dtype = tc.DTYPE[fmt]
    seed = (CASES + EXTRAS + ZOO_CASES).index(case) * 2 + fmt
    H, W = x_size
    qkv, anc = block_inputs(case, x_size, dtype, device, seed)
    h, d = case.heads, case.d
    merged = torch.full((B * H * W, 2 * h * 32), SENTINEL, device=device, dtype=dtype)
    buf = {"qkv": qkv, "anchor": anc, "merged": merged}
    key = (case, fmt)

    def ref_fn(q, k, v, index, mask, mutation=None, table=None):
        return O.attn_launch_reference(q, k, v, table if table is not None else tables[ln.role], index, mask, dtype,
                                       mutation)

    tables = {}
    if case.role == "stripe2":  # pass 1 first: X1 is pass 2's value operand
        ln1 = tc.attention_launch("stripe1", ln.gk, ln.gq, h, h, h * d, case.shifted)
        anc_g = ln.gk
        nW = (anc_g.H // anc_g.wh) * (anc_g.W // anc_g.ww)
        buf["x1"] = torch.full((B * nW * h * anc_g.wh * anc_g.ww, 32), SENTINEL, device=device, dtype=dtype)
        tables["stripe1"] = cpb_table(ln1, seed + 1000)
        run(tc, ln1, buf, tables["stripe1"])
    tables[ln.role] = cpb_table(ln, seed, case.grow)
    if case.role == "stripe1":
        nW = (ln.gq.H // ln.gq.wh) * (ln.gq.W // ln.gq.ww)
        buf["x1"] = torch.full((B * nW * h * ln.gq.wh * ln.gq.ww, 32), SENTINEL, device=device, dtype=dtype)
    run(tc, ln, buf, tables[ln.role])
    torch.cuda.synchronize()

    index, mask = O.attn_pair_geometry(grid_t(ln.gq), grid_t(ln.gk), ln.use_mask)
    index, mask = index.to(device), None if mask is None else mask.to(device)
    q, k, v = (operand(buf, s, g, h) for s, g in ((ln.q, ln.gq), (ln.k, ln.gk), (ln.v, ln.gk)))
    got = operand(buf, ln.out, ln.gq, h)
    lines = []
    if case.role == "stripe2":
        x1 = buf["x1"].view(-1, h, ln.gk.wh * ln.gk.ww, 32)
        check_pads(x1, ln1, d, "X1")
        i1, m1 = O.attn_pair_geometry(grid_t(ln1.gq), grid_t(ln1.gk), ln1.use_mask)
        q1, k1, v1 = (operand(buf, s, g, h) for s, g in ((ln1.q, ln1.gq), (ln1.k, ln1.gk), (ln1.v, ln1.gk)))
        if key not in _REF:
            ex1, em1, _ = ref_fn(q1, k1, v1, i1.to(device), None if m1 is None else m1.to(device), table=tables["stripe1"])
            ex_c, em_c, _ = ref_fn(q, k, em1, index, mask)  # the chain with the emulated X1
            ex_c2, _, _ = ref_fn(q, k, ex1, index, mask)    # the chain of exact passes
            _REF[key] = {"p1": (ex1, em1), "chain": (ex_c2, em_c)}
        ex1, em1 = _REF[key]["p1"]
        s1 = compare(x1, em1, d, dtype)
        lines.append(f"  pass 1 (X1): {s1[0]:.2f} ulp, mismatch {s1[1]:.4f}")
        assert not fails_gate(s1), (case, "pass 1", s1)
    cached = _REF.get(key, {}).get("main")
    if cached is None or (case.role == "stripe2" and not torch.equal(cached[3], buf["x1"])):
        exact, emul, info = ref_fn(q, k, v, index, mask)
        _REF.setdefault(key, {})["main"] = (exact, emul, info, buf["x1"].clone() if case.role == "stripe2" else None)
    exact, emul, info, _ = _REF[key]["main"]
    stats = compare(got, emul, d, dtype)
    acc = float((emul - exact)[..., :d].abs().max())
    print(f"\n[attn{variant} {tc.DTYPE[fmt]}] {case.src} {case.role} {case.win} df{case.df} shifted={case.shifted} "
          f"h{h} d{d} grow={case.grow} path={sig}: |got-emulated| {stats[0]:.2f} ulp, mismatch {stats[1]:.4f}, "
          f"|emulated-exact| {acc:.2e}, rescales {info['rescales']}")
    if case.role == "stripe2":
        ex_c, em_c = _REF[key]["chain"]
        sc = compare(got, em_c, d, dtype)
        lines.append(f"  chain vs chained emulation: {sc[0]:.2f} ulp, mismatch {sc[1]:.4f}; chained |emulated-exact| "
                     f"{float((em_c - ex_c)[..., :d].abs().max()):.2e}")
        assert sc[0] <= GATE_CHAIN, (case, "chain", sc)
    print("\n".join(lines))
    check_pads(got, ln, d, "output")
    if ln.out[0] == "merged":  # the launch writes its own slots and nothing else
        rest = merged.view(B * H * W, 2, h * 32)[:, 1 - ln.out[1] // (h * 32)]
        assert bool((rest == SENTINEL).all()), "wrote outside its output slots"
    assert not fails_gate(stats), (case, stats)
    if case.grow:
        assert info["rescales"] > 0, "the lazy-rescale table did not move the reference"

    if variant != 5:
        return

    def tokens(which, grid):
        spec = {"q": ln.q, "k": ln.k, "v": ln.v}[which]
        t = buf[spec[0]].view(B, grid[0], grid[1], -1)[..., spec[1]:spec[1] + h * 32]
        return O.attn_windows(t, grid, h)

    muts = mutations(ref_fn, ln, q, k, v, tables[ln.role], index, mask, tokens, variant)
    w = got.shape[0] - 1
    for name, (m_exact, m_emul, _) in muts.items():
        ms = compare(got[w:], m_emul, d, dtype)
        print(f"  mutation '{name}': {ms[0]:.2f} ulp, mismatch {ms[1]:.4f} -> new gate "
              f"{'FAILS' if fails_gate(ms) else 'passes'}; old bound {'catches' if old_bound_catches(m_emul, exact[w:], d) else 'misses'} it")
    # The gate must see every mutation in GATED.  One dropped key can stay below one output ulp on stripe pass 1 (a key
    # among 1024-10368) and a denominator from the unrounded P is off by at most P's own rounding error (half an output
    # ulp), so those two are reported only.
    missed = [n for n, (_, m_emul, _) in muts.items() if n in GATED and not fails_gate(compare(got[w:], m_emul, d, dtype))]
    assert not missed, f"mutations the gate does not catch: {missed}"
