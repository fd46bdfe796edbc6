"""The float64 references and derived bounds of the fp32 parity path's kernels (csrc/ops_f32.cu), shared by
test_gpu_f32_paths.py (one seeded instance per launch path) and test_gpu_f32_replay.py (real forwards).  The bounds and
gates are described in test_gpu_f32_paths.py."""
from typing import NamedTuple

import torch

import grl_oracle as O
from grl_oracle import U, gamma
from support import ulp

B = 2              # images of a launch-path case
ERFF_ULP = 2       # CUDA C++ Programming Guide, maximum ulp error of erff / expf (no fast math)
EXPF_ULP = 2
GATE_ATTN = 1695.0   # fp32 ulps at max(|ref|, row rms): 2 x the worst case, 847.2 (small/sr window; H100 80GB HBM3, 400 W)
GATE_CHAIN = 2165.0  # both stripe passes against the float64 chain: 2 x the worst case, 1082.3 (same card)
ACT_NONE, ACT_GELU, ACT_LEAKY = 0, 1, 2
POOL_ROWS = 256  # rows per partial sum of the channel gate (ops_f32.cu: kPoolRows)


def ulp_stats(got, ref):
    """max |got - ref| in fp32 ulps at max(|ref|, the row's rms) (rows: the last dimension)."""
    scale = torch.maximum(ref.abs(), ref.pow(2).mean(-1, keepdim=True).sqrt())
    return float(((got.double() - ref).abs() / ulp(scale, torch.float32)).nan_to_num(float("inf")).max())


def attn_ratio(got, ref, absref, nk, gate):
    """max |got - ref| / (gate fp32 ulps at max(|ref|, row rms) + gamma_(nk + nk / 32 + 2) (absref + |ref|)), absref the
    same pass on |v|.  The second term is the kernel's sequential sums over nk keys (numerator, denominator and one
    rescale per 32-key tile): it grows with the key count, and real operands whose v share one sign do not cancel it the
    way the zero-mean seeded operands that set the ulp gates do."""
    scale = torch.maximum(ref.abs(), ref.pow(2).mean(-1, keepdim=True).sqrt())
    acc = gamma(nk + nk // 32 + 2) * (absref + ref.abs())
    return float(((got.double() - ref).abs() / (gate * ulp(scale, torch.float32) + acc)).nan_to_num(float("inf")).max())


# ------------------------------------------------------------------------------------------------------- attention


def windows(t, g, heads):
    """(B, H, W, c) tokens -> (B nW, heads, wh ww, c / heads) in the kernel's window order (roll by -shift, then
    partition); g = (H, W, wh, ww, sh, sw)."""
    _, _, wh, ww, sh, sw = g
    t = torch.roll(t, (-sh, -sw), (1, 2)) if sh or sw else t
    return O.partition(t, (wh, ww)).reshape(-1, wh * ww, heads, t.shape[-1] // heads).transpose(1, 2)


def unwindows(o, g, nb):
    """Inverse of `windows`: (B nW, heads, wh ww, d) -> (B, H, W, heads d)."""
    H, W, wh, ww, sh, sw = g
    t = O.unpartition(o.transpose(1, 2).reshape(-1, wh, ww, o.shape[1] * o.shape[3]), (wh, ww), (H, W))
    assert t.shape[0] == nb
    return torch.roll(t, (sh, sw), (1, 2)) if sh or sw else t


class Pass(NamedTuple):
    """One attention launch on float64 operands: q, k (B, H, W, c) tokens; v tokens or, for stripe pass 2, the dense
    X1 (B nW, heads, Nk, d); o_dense: the launch writes dense X1 (stripe pass 1) instead of tokens."""
    gq: tuple
    gk: tuple
    q: torch.Tensor
    k: torch.Tensor
    v: torch.Tensor
    v_dense: bool
    o_dense: bool
    scale: torch.Tensor
    table: torch.Tensor
    use_mask: bool


def attn_ref(p, heads, mutation=None, index=None, mask=None, v=None, roll=True, drop_last_key=False, sel=None):
    """float64 reference of one pass in the kernel's window layout (B nW, heads, Nq, d).  roll=False: the kernel read
    and wrote the un-rolled grids.  sel: only these windows (indices into B nW), in that order."""
    gq, gk = (p.gq, p.gk) if roll else (p.gq[:4] + (0, 0), p.gk[:4] + (0, 0))
    if index is None or (mask is None and p.use_mask):
        i0, m0 = O.attn_pair_geometry(p.gq, p.gk, p.use_mask)
        index = i0 if index is None else index
        mask = m0 if mask is None else mask
    mask = mask if p.use_mask else None
    v = p.v if v is None else v
    q, k, vw = windows(p.q, gq, heads), windows(p.k, gk, heads), v if p.v_dense else windows(v, gk, heads)
    if sel is not None:
        q, k, vw = q[sel], k[sel], vw[sel]
        mask = None if mask is None else mask.to(sel.device)[sel % mask.shape[0]]
    if drop_last_key:
        k, vw, index, mask = k[:, :, :-1], vw[:, :, :-1], index[:, :-1], None if mask is None else mask[..., :-1]
    o = O.attn_f32_reference(q, k, vw, p.scale, p.table, index, mask, mutation)
    if not roll and not p.o_dense:  # written to the un-rolled token positions
        o = windows(unwindows(o, gq, B), p.gq, heads)
    return o


# ------------------------------------------------------------------------------------------------------------ GEMM


def im2col(x, transposed=False, wrap=False):
    """(B, H, W, Cin) -> (B H W, 9 Cin) with k = tap Cin + c, tap = 3 (dy + 1) + (dx + 1) (pack_conv_weight's order).
    Padding reads zero; wrap=True reads the flat neighbour m + dy W + dx instead (the previous row or image)."""
    Bn, H, W, C = x.shape
    flat = x.reshape(-1, C)
    M = flat.shape[0]
    m = torch.arange(M, device=x.device)
    yy, xx = (m // W) % H, m % W
    cols = []
    for t in range(9):
        dy, dx = divmod(t, 3)
        if transposed:
            dy, dx = dx, dy
        dy, dx = dy - 1, dx - 1
        src = m + dy * W + dx
        ok = (src >= 0) & (src < M) if wrap else (yy + dy >= 0) & (yy + dy < H) & (xx + dx >= 0) & (xx + dx < W)
        cols.append(torch.where(ok[:, None], flat[src.clamp(0, M - 1)], 0.0))
    return torch.cat(cols, 1)


def gemm_bound(A, w, b, act, slope, res):
    """Per-element bound on |kernel - float64| of act(A w^T + b) (+ res), for a sequential FMA chain over k."""
    return gemm_bound_of(A @ w.T + b, A.abs() @ w.abs().T, A.shape[1], act, slope, res)


def gemm_bound_of(v, absdot, K, act, slope, res):
    """gemm_bound from the pre-activation v = A w^T + b and absdot = |A| |w|^T (a conv gives both without im2col)."""
    e = gamma(K) * absdot
    e = e + U * (v.abs() + e)                                              # + bias
    if act == ACT_GELU:
        y = O._gelu(v)
        e = 1.13 * e + 0.5 * v.abs() * (ERFF_ULP * U + 3 * U) + U * y.abs()  # |GELU'| <= 1.13; erf term absolute
    elif act == ACT_LEAKY:
        y = torch.where(v > 0, v, v * slope)
        e = max(1.0, slope) * e + U * y.abs()
    else:
        y = v
    if res is not None:
        e = e + U * ((y + res).abs() + e)
    return e, v


# ------------------------------------------------------------------------------------------ channel gate, bias table


def gate_reference(y, w1, b1, w2, b2, mutation=None):
    L = y.shape[1]
    chunks = -(-L // POOL_ROWS)
    if mutation == "partial last chunk dropped":
        mean = y[:, :(chunks - 1) * POOL_ROWS].sum(1) / L
    elif mutation == "division by chunks x 256":
        mean = y.sum(1) / (chunks * POOL_ROWS)
    else:
        mean = y.mean(1)
    hpre = mean @ w1.T + b1
    h = hpre if mutation == "ReLU missing" else torch.relu(hpre)
    return torch.sigmoid(h @ w2.T + b2)


def gate_bound(y, w1, b1, w2, b2):
    L, C = y.shape[1], y.shape[2]
    R = w1.shape[0]
    mean = y.mean(1)
    e_mean = gamma(POOL_ROWS + -(-L // POOL_ROWS)) * y.abs().sum(1) / L + U * mean.abs()
    hpre = mean @ w1.T + b1
    e_h = e_mean @ w1.abs().T + gamma(-(-C // 32) + 5) * (mean.abs() @ w1.abs().T) + U * hpre.abs()
    h = torch.relu(hpre)
    s = h @ w2.T + b2
    e_s = e_h @ w2.abs().T + gamma(R) * (b2.abs() + h @ w2.abs().T)
    gt = torch.sigmoid(s)
    # below 2^-126 (s < -87.3) the gate is a subnormal rounded to 2^-149, or 0 where 1 + expf(-s) overflows (s < -88.7):
    # an absolute error of at most the gate itself and half a subnormal spacing
    tiny = torch.where(gt < 2.0 ** -126, gt + 2.0 ** -150, torch.zeros_like(gt))
    return gt * (1 - gt) * e_s + gt * (2 * EXPF_ULP * U * (1 - gt) + 2 * U) + tiny


def bias_table_bound(t, w1, b1, w2):
    """16 sigmoid(W2 relu(W1 t + b1)): two FMAs per hidden unit, a sequential FMA chain over them, expf."""
    hpre = t @ w1.T + b1
    e_h = gamma(2) * (t.abs() @ w1.abs().T + b1.abs())
    h = torch.relu(hpre)
    acc = h @ w2.T
    e_acc = e_h @ w2.abs().T + gamma(w1.shape[0]) * (h @ w2.abs().T)
    sg = torch.sigmoid(acc)
    return (16 * (sg * (1 - sg) * e_acc + sg * (2 * EXPF_ULP * U * (1 - sg) + 2 * U))).T, (16 * sg).T


# ------------------------------------------------------------------------------------------------ launch-path cases
# The signatures of fp32 launches and one case per launch path, for test_gpu_f32_paths.py (which describes them) and
# test_command_paths.py.


def launches_of(launches, kind):
    from grl_image_restoration_b200 import modules

    return [ln for ln in launches if isinstance(ln, getattr(modules, kind))]


# ------------------------------------------------------------------------------------------------------- attention


def attn_path(ln):
    """(role, D, d < D, Nq % 128 != 0, Nq > 128, Nk % 32 != 0, Nk > 32, use_mask, non-zero roll)."""
    d = ln.d
    D = 16 if d <= 16 else 32 if d <= 32 else 64
    nq, nk = ln.gq.wh * ln.gq.ww, ln.gk.wh * ln.gk.ww
    roll = any((g.sh, g.sw) != (0, 0) for g in (ln.gq, ln.gk))
    return (ln.role, D, d < D, nq % 128 != 0, nq > 128, nk % 32 != 0, nk > 32, bool(ln.use_mask), roll)


class AttnCase(NamedTuple):
    src: str      # the first released config / block that launches this path (or why an extra case exists)
    role: str     # "window", "stripe1" (anchors attend to the stripe's tokens), "stripe2" (tokens attend to anchors)
    win: tuple    # the token window of the pass: the attention window or the (oriented) stripe
    df: int       # anchor down factor (1 for window attention)
    shifted: bool
    heads: int
    d: int
    shift: tuple = None  # the roll when shifted; None: half the window


# one case per released path, from its first launcher (stage 0: block 0 or 1 unshifted, block 2 shifted stripes)
ATTN_CASES = [
    AttnCase("tiny/sr", "window", (32, 32), 1, True, 2, 16),
    AttnCase("tiny/sr", "stripe1", (64, 64), 4, True, 2, 16),
    AttnCase("tiny/sr", "stripe2", (64, 64), 4, True, 2, 16),
    AttnCase("tiny/deblur", "window", (12, 12), 1, True, 2, 16),
    AttnCase("tiny/deblur", "stripe1", (48, 96), 4, True, 2, 16),
    AttnCase("tiny/jpeg", "stripe2", (72, 144), 4, True, 2, 16),
    AttnCase("tiny/dm", "window", (8, 8), 1, True, 2, 16),
    AttnCase("tiny/dm", "stripe1", (32, 32), 4, True, 2, 16),
    AttnCase("tiny/sr", "window", (32, 32), 1, False, 2, 16),
    AttnCase("tiny/sr", "stripe1", (64, 64), 4, False, 2, 16),
    AttnCase("tiny/sr", "stripe2", (64, 64), 4, False, 2, 16),
    AttnCase("tiny/deblur", "window", (12, 12), 1, False, 2, 16),
    AttnCase("tiny/deblur", "stripe1", (48, 96), 4, False, 2, 16),
    AttnCase("tiny/jpeg", "stripe2", (72, 144), 4, False, 2, 16),
    AttnCase("tiny/dm", "window", (8, 8), 1, False, 2, 16),
    AttnCase("tiny/dm", "stripe1", (32, 32), 4, False, 2, 16),
    AttnCase("small/sr", "window", (32, 32), 1, True, 2, 32),
    AttnCase("small/sr", "stripe1", (64, 64), 4, True, 2, 32),
    AttnCase("small/sr", "stripe2", (64, 64), 4, True, 2, 32),
    AttnCase("small/deblur", "window", (12, 12), 1, True, 2, 32),
    AttnCase("small/deblur", "stripe1", (48, 96), 4, True, 2, 32),
    AttnCase("small/jpeg", "stripe2", (72, 144), 4, True, 2, 32),
    AttnCase("small/dm", "window", (8, 8), 1, True, 2, 32),
    AttnCase("small/dm", "stripe1", (32, 32), 4, True, 2, 32),
    AttnCase("small/sr", "window", (32, 32), 1, False, 2, 32),
    AttnCase("small/sr", "stripe1", (64, 64), 4, False, 2, 32),
    AttnCase("small/sr", "stripe2", (64, 64), 4, False, 2, 32),
    AttnCase("small/deblur", "window", (12, 12), 1, False, 2, 32),
    AttnCase("small/deblur", "stripe1", (48, 96), 4, False, 2, 32),
    AttnCase("small/jpeg", "stripe2", (72, 144), 4, False, 2, 32),
    AttnCase("small/dm", "window", (8, 8), 1, False, 2, 32),
    AttnCase("small/dm", "stripe1", (32, 32), 4, False, 2, 32),
    AttnCase("base/sr", "window", (32, 32), 1, True, 3, 30),
    AttnCase("base/sr", "stripe1", (64, 64), 2, True, 3, 30),
    AttnCase("base/sr", "stripe2", (64, 64), 2, True, 3, 30),
    AttnCase("base/deblur", "window", (12, 12), 1, True, 3, 30),
    AttnCase("base/deblur", "stripe1", (48, 96), 4, True, 3, 30),
    AttnCase("base/jpeg", "stripe2", (72, 144), 4, True, 3, 30),
    AttnCase("base/dm", "window", (8, 8), 1, True, 3, 30),
    AttnCase("base/dm", "stripe1", (32, 32), 4, True, 3, 30),
    AttnCase("base/sr", "window", (32, 32), 1, False, 3, 30),
    AttnCase("base/sr", "stripe1", (64, 64), 2, False, 3, 30),
    AttnCase("base/sr", "stripe2", (64, 64), 2, False, 3, 30),
    AttnCase("base/deblur", "window", (12, 12), 1, False, 3, 30),
    AttnCase("base/deblur", "stripe1", (48, 96), 4, False, 3, 30),
    AttnCase("base/jpeg", "stripe2", (72, 144), 4, False, 3, 30),
    AttnCase("base/dm", "window", (8, 8), 1, False, 3, 30),
    AttnCase("base/dm", "stripe1", (32, 32), 4, False, 3, 30),
]
ATTN_EXTRAS = [  # limits no released config uses, and the earlier operator tests' geometries
    AttnCase("extra: head_dim 64 (D = 64)", "window", (16, 16), 1, True, 2, 64),
    AttnCase("extra: head_dim 64 (D = 64)", "stripe2", (32, 32), 4, True, 2, 64),
    AttnCase("extra: 8 heads, the kernel's limit", "window", (8, 8), 1, True, 8, 8),
    AttnCase("extra: 8 heads, the kernel's limit", "stripe2", (16, 32), 2, False, 8, 12),
    AttnCase("extra: released jpeg window, 1296 keys", "window", (36, 36), 1, True, 2, 16),
    AttnCase("extra: 8x8 window, head_dim 9", "window", (8, 8), 1, True, 2, 9),
    AttnCase("extra: 8x8 window, head_dim 9", "window", (8, 8), 1, False, 2, 9),
    AttnCase("extra: 4x4 window, 16 keys", "window", (4, 4), 1, False, 3, 10),
    AttnCase("extra: 6x6 window, head_dim 40", "window", (6, 6), 1, True, 2, 40),
    AttnCase("extra: 8x16 stripes, head_dim 9", "stripe2", (8, 16), 2, True, 2, 9),
    AttnCase("extra: 16x8 stripes, head_dim 9", "stripe2", (16, 8), 2, False, 2, 9),
    AttnCase("extra: stripe groups, 4x16 stripes", "stripe2", (4, 16), 2, True, 2, 8),
    AttnCase("extra: stripe groups, 4x8 stripes", "stripe2", (4, 8), 2, False, 2, 8),
    AttnCase("extra: stripe groups, 32x8 stripes shifted by (0, 4)", "stripe2", (32, 8), 2, True, 2, 8, (0, 4)),
    AttnCase("extra: df 3, 1 head", "stripe2", (6, 12), 3, True, 1, 32),
]
# released paths outside the VARIANTS x TASKS grid of archs: GRL-Base blind SR's stripe pass 1 (head_dim 30 on 8 x 16
# anchors, 2048 keys).  They come after the extras because a case's seed is its index in the case list.
ATTN_ZOO_CASES = [
    AttnCase("base/bsr", "stripe1", (32, 64), 4, False, 3, 30),
    AttnCase("base/bsr", "stripe1", (32, 64), 4, True, 3, 30),
]


def attn_case_launch(case):
    """(x_size, launch descriptor) of a case: an image of 2 x 2 windows of the pass's grid."""
    from grl_image_restoration_b200 import geometry as G, modules

    wh, ww = case.win
    x_size = (2 * wh, 2 * ww)
    sh = (case.shift or (wh // 2, ww // 2)) if case.shifted else (0, 0)
    tok = G.token_grid(x_size, case.win, sh)
    gq = gk = tok
    if case.role != "window":
        anc = G.anchor_grid(x_size, case.win, sh, case.df)
        gq, gk = (anc, tok) if case.role == "stripe1" else (tok, anc)
    return x_size, modules.AttnF32(case.src, case.role, gq, gk, case.heads, case.d, case.shifted)


# ------------------------------------------------------------------------------------------------------------ GEMM


def gemm_path(g):
    """(conv, K % 16 != 0, k tiles, N % 64 != 0, N > 64, act, bias, residual)."""
    return (g.conv, g.K % 16 != 0, -(-g.K // 16), g.N % 64 != 0, g.N > 64, g.act, g.bias, g.res)


class GemmCase(NamedTuple):
    src: str
    conv: bool
    K: int
    N: int
    act: int = ACT_NONE
    res: bool = False
    slope: float = 0.01  # LeakyReLU only

    def call(self):
        from grl_image_restoration_b200 import modules

        return modules.GemmF32(self.src, self.conv, self.K, self.N, self.act,
                               self.slope if self.act == ACT_LEAKY else 0.0, True, self.res)


GEMM_CASES = [  # one case per released path, from its first launcher
    GemmCase("tiny/srx2 conv_first", True, 27, 64),
    GemmCase("tiny/srx2 qkv", False, 64, 192),
    GemmCase("tiny/srx2 anchor", False, 64, 32),
    GemmCase("tiny/srx2 proj", False, 64, 64),
    GemmCase("tiny/srx2 fc1", False, 64, 128, ACT_GELU),
    GemmCase("tiny/srx2 fc2", False, 128, 64),
    GemmCase("tiny/srx2 stage0.conv", True, 576, 64, res=True),
    GemmCase("tiny/srx2 upsample.up.0", True, 576, 12),
    GemmCase("tiny/dnx1 conv_last", True, 576, 3, res=True),
    GemmCase("small/srx2 conv_first", True, 27, 128),
    GemmCase("small/srx2 qkv", False, 128, 384),
    GemmCase("small/srx2 fc1", False, 128, 256, ACT_GELU),
    GemmCase("small/srx2 fc2", False, 256, 128),
    GemmCase("small/srx2 stage0.conv", True, 1152, 128, res=True),
    GemmCase("small/srx2 conv_before_upsample", True, 1152, 64, ACT_LEAKY),
    GemmCase("small/srx2 upsample.up.0", True, 576, 256),
    GemmCase("small/dnx1 conv_last", True, 1152, 3, res=True),
    GemmCase("base/srx2 conv_first", True, 27, 180),
    GemmCase("base/srx2 qkv", False, 180, 540),
    GemmCase("base/srx2 cab1", True, 1620, 45, ACT_GELU),
    GemmCase("base/srx2 cab2", True, 405, 180),
    GemmCase("base/srx2 fc1", False, 180, 360, ACT_GELU),
    GemmCase("base/srx2 fc2", False, 360, 180),
    GemmCase("base/srx2 stage0.conv", True, 1620, 180, res=True),
    GemmCase("base/srx2 conv_before_upsample", True, 1620, 64, ACT_LEAKY),
    GemmCase("base/dnx1 conv_last", True, 1620, 3, res=True),
]
GEMM_EXTRAS = [  # the earlier operator tests' shapes whose paths no released forward takes (all with a residual)
    GemmCase("extra: linear K 180 N 90 + residual", False, 180, 90, res=True),
    GemmCase("extra: linear K 180 N 360 GELU + residual", False, 180, 360, ACT_GELU, True),
    GemmCase("extra: linear K 360 N 180 + residual", False, 360, 180, res=True),
    GemmCase("extra: linear K 5 N 3 LeakyReLU 0.2 + residual", False, 5, 3, ACT_LEAKY, True, 0.2),
    GemmCase("extra: linear K 64 N 64 + residual", False, 64, 64, res=True),
    GemmCase("extra: conv Cin 36 N 9 GELU + residual", True, 324, 9, ACT_GELU, True),
    GemmCase("extra: conv Cin 3 N 64 + residual", True, 27, 64, res=True),
    GemmCase("extra: conv Cin 45 N 180 + residual", True, 405, 180, res=True),
    GemmCase("extra: conv Cin 64 N 12 LeakyReLU + residual", True, 576, 12, ACT_LEAKY, True),
    GemmCase("extra: conv Cin 180 N 45 GELU + residual", True, 1620, 45, ACT_GELU, True),
]
# released paths outside the grid of archs, after the extras for the same reason: 1- and 6-channel heads, the 3-channel
# tail without the input residual, the nearest+conv head's convs
GEMM_ZOO_CASES = [
    GemmCase("tiny/dnx1 c1 conv_first", True, 9, 64),
    GemmCase("small/dnx1 c1 conv_first", True, 9, 128),
    GemmCase("base/dnx1 c1 conv_first", True, 9, 180),
    GemmCase("base/bsrx4 conv_up1", True, 576, 64, ACT_LEAKY, slope=0.2),
    GemmCase("base/defocus_dual conv_first", True, 54, 180),
    GemmCase("base/defocus_dual conv_last", True, 1620, 3),
]
