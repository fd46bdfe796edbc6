"""The launch-path cases of the tensor-core attention kernel (csrc/attn_tc.cu) and the machinery that runs and gates
them, shared by test_gpu_tc_attn.py (one small instance per path), test_gpu_tc_scale.py (the benchmark's sizes) and
test_gpu_tc_replay.py (real forwards).  A case's seed is its index in CASES + EXTRAS + ZOO_CASES."""
import math
from typing import NamedTuple

import torch

import grl_oracle as O
from support import grid_t, ulp

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


def compare(got, emul, d, dtype):
    """(max |got - emul| in ulps at max(|emul|, row rms), fraction of elements that differ) over the d real columns."""
    g, e = got[..., :d].double(), emul[..., :d]
    rms = e.pow(2).mean(-1, keepdim=True).sqrt()
    diff = (g - e).abs()
    return float((diff / ulp(torch.maximum(e.abs(), rms), dtype)).max()), float((diff != 0).double().mean())


def fails_gate(stats):
    return stats[0] > GATE_ULP


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


SENTINEL = -7.25


def check_pads(got, ln, d, what):
    if d < 32:
        assert bool((got[..., d:31] == 0).all()), f"{what}: pad columns {d}..30 not zero"
        assert bool((got[..., 31] == (1.0 if ln.ones_col else 0.0)).all()), f"{what}: column 31"
