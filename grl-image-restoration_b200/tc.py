"""bf16 tensor-core execution of a GRL block / stage / network (the throughput path).

Host-side orchestration only: one-time weight packing (pad head_dim to 32-wide slots, pad channel pitches to
multiples of 64, permute the QKV rows into [window q|k|v][stripe q|k|v] x head order, im2col-order the 3x3 kernels)
and the launch sequence of the wgmma kernels behind the C ABI (grl_tc_gemm / grl_tc_attn, include/grl_b200.h).  That
sequence is written once (forward / stage_forward / BlockPlan.run) and issued through a launcher: Device runs it,
Listing records its GEMMs without a device (gemm_launches).  The fp32 forward (modules.py) uses the same launchers.
Numerics contract (DESIGN.md): bf16 only for MMA operands; residual stream, LayerNorm, L2-normalisation, softmax
statistics and every accumulator are fp32.
Reference semantics: mixed_attn_block_efficient.py:351-381,:539-556; mixed_attn_block.py:948-983; grl.py:164-170,:506-551.
"""
import ctypes
import inspect
from typing import NamedTuple

import torch
from torch import nn

from . import capi
from . import functional as K
from . import geometry as G
from .streams import Produced

LOG2E = 1.4426950408889634
EPI_BIAS_ACT, EPI_QKV, EPI_LN = 0, 1, 2
SLOT = 32
FMT = {"fp16": 0, "bf16": 1}
DTYPE = {0: torch.float16, 1: torch.bfloat16}


def fmt_of(t):
    return 1 if t.dtype == torch.bfloat16 else 0


def round_up(a, b):
    return (a + b - 1) // b * b


LN_MAX_C = 188  # the widest LayerNorm row plan_gemm_tc takes (gemm_tc.cu)


def supported(C, heads_w, heads_s):
    """Architectures the tensor-core path covers: head_dim <= 32 (one 32-wide slot per head), <= 8 heads per
    attention, C % 4 == 0 and C <= LN_MAX_C (plan_gemm_tc's LayerNorm-epilogue limit).  Anything else runs on the
    fp32 kernels ("auto") or is rejected up front (explicit "fp16" / "bf16")."""
    c = C // 2
    return (C % 4 == 0 and C <= LN_MAX_C and c % heads_w == 0 and c % heads_s == 0 and c // heads_w <= SLOT
            and c // heads_s <= SLOT and heads_w <= 8 and heads_s <= 8)


def _h16(*shape, device, fmt, zero=False):
    return (torch.zeros if zero else torch.empty)(*shape, device=device, dtype=DTYPE[fmt])


def _mean4(mean, cin=3):
    """The host mean array grl_tc_head_pack reads: max(4, cin) floats, a single mean broadcast to all of them."""
    n = max(4, cin)
    m = [float(v) for v in (mean if isinstance(mean, (list, tuple)) else mean.flatten().tolist())]
    m = (m * n)[:n] if len(m) == 1 else (m + [0.0] * n)[:n]
    return (ctypes.c_float * n)(*m)


def head_pack(x, hp, wp, mean, img_range, cpad=64, fmt=0, want_f32=False, out=None):
    """Network input (B, Cin, H, W) fp32 -> 16-bit channels-last (B, hp, wp, cpad) [+ fp32 (B, hp, wp, Cin)]: reflect pad,
    (x - mean) * img_range, layout change and operand pack in one kernel (grl_tc_head_pack).  out: that pair, preallocated."""
    B, Cin, H, W = x.shape
    y16, y32 = out or (_h16(B, hp, wp, cpad, device=x.device, fmt=fmt),
                       torch.empty(B, hp, wp, Cin, device=x.device, dtype=torch.float32) if want_f32 else None)
    capi.check(capi.lib().grl_tc_head_pack(capi.ptr(x), B, Cin, H, W, hp, wp, _mean4(mean, Cin), float(img_range), capi.ptr(y16),
                                           cpad, capi.ptr(y32), fmt, capi.stream()))
    return y16, y32


def head_pack_rggb(cfa4, hp, wp, mean, img_range, cpad=64, fmt=0, want_f32=False, out=None):
    """head_pack of K.demosaic(cfa4) in one kernel (grl_tc_head_pack_rggb): packed RGGB planes (B, 4, h, w) fp32 ->
    (B, hp, wp, cpad) [+ fp32 (B, hp, wp, 3)] for the (2h, 2w) image, without writing the RGB image."""
    B, _, h, w = cfa4.shape
    y16, y32 = out or (_h16(B, hp, wp, cpad, device=cfa4.device, fmt=fmt),
                       torch.empty(B, hp, wp, 3, device=cfa4.device, dtype=torch.float32) if want_f32 else None)
    capi.check(capi.lib().grl_tc_head_pack_rggb(capi.ptr(cfa4), B, h, w, hp, wp, _mean4(mean), float(img_range),
                                                capi.ptr(y16), cpad, capi.ptr(y32), fmt, capi.stream()))
    return y16, y32


def pack_rows(x, cpad, fmt=0, out=None):
    """fp32 (..., C) contiguous -> 16-bit (..., cpad), zero padded."""
    C = x.shape[-1]
    M = x.numel() // C
    y = _h16(*x.shape[:-1], cpad, device=x.device, fmt=fmt) if out is None else out
    capi.check(capi.lib().grl_tc_pack16(capi.ptr(x), C, capi.ptr(y), M, C, cpad, fmt, capi.stream()))
    return y


def unpack_rows(x16, C, off=0):
    """16-bit (..., ld) -> fp32 (..., C) taking columns [off, off + C)."""
    ld = x16.shape[-1]
    M = x16.numel() // ld
    y = torch.empty(*x16.shape[:-1], C, device=x16.device, dtype=torch.float32)
    capi.check(capi.lib().grl_tc_unpack16(capi.ptr(x16), ld, off, capi.ptr(y), C, M, C, fmt_of(x16), capi.stream()))
    return y


def _slot_rows(first, n, d, device):
    """Rows (first + i) * SLOT + e of slots first .. first + n - 1, e < d, slot-major: an index map built on the device
    (a host list would be a blocking host-to-device copy)."""
    return ((first + torch.arange(n, device=device))[:, None] * SLOT + torch.arange(d, device=device)).reshape(-1)


def _pad_matrix(w, npad, kpad, row_map=None, col_map=None, fmt=0):
    """Scatter fp32 (N, K) into 16-bit (npad, kpad): dest row row_map[i] <- src row i, dest col col_map[j] <- src col j
    (maps: index tensors on w's device)."""
    N, Kd = w.shape
    out = torch.zeros(npad, kpad, device=w.device, dtype=torch.float32)
    r = torch.arange(N, device=w.device) if row_map is None else row_map
    c = torch.arange(Kd, device=w.device) if col_map is None else col_map
    out[r[:, None], c[None, :]] = w.detach().float()
    return out.to(DTYPE[fmt]).contiguous()


def _pad_vector(b, npad, row_map=None, device=None):
    """fp32 (N) -> (npad) with dest row_map[i] <- b[i]; b None (no bias): zeros on `device`."""
    out = torch.zeros(npad, device=b.device if b is not None else device, dtype=torch.float32)
    if b is not None:
        out[torch.arange(b.numel(), device=b.device) if row_map is None else row_map] = b.detach().float()
    return out


def pack_conv(conv, cin_pad, npad, fmt=0, ps_r=0):
    """nn.Conv2d(3x3) weight (Cout, Cin, 3, 3) -> 16-bit (npad, 9*cin_pad), k = (ky*3+kx)*cin_pad + c; bias fp32 (npad).
    ps_r > 0: the conv feeds nn.PixelShuffle(ps_r): output channel c*r^2 + q (torch order) is stored at row q*(Cout/r^2) + c,
    so the channels of one shuffled pixel are consecutive output columns (grl_tc_gemm's ps_r store)."""
    w = conv.weight.detach().float()
    co, ci = w.shape[:2]
    rows = torch.arange(co, device=w.device)
    if ps_r > 0:
        cq = co // (ps_r * ps_r)
        rows = (rows % (ps_r * ps_r)) * cq + rows // (ps_r * ps_r)
    out = torch.zeros(npad, 9, cin_pad, device=w.device, dtype=torch.float32)
    out[rows, :, :ci] = w.permute(0, 2, 3, 1).reshape(co, 9, ci)
    bias = torch.zeros(npad, device=w.device, dtype=torch.float32)
    if conv.bias is not None:
        bias[rows] = conv.bias.detach().float()
    return out.reshape(npad, 9 * cin_pad).to(DTYPE[fmt]).contiguous(), bias


class Spec(NamedTuple):
    """Shape and dtype of a tensor argument in a launch descriptor (GemmLaunch).  data_ptr() is a non-null stand-in:
    grl_tc_gemm_path only tests pointers for NULL."""
    shape: tuple
    dtype: torch.dtype

    def data_ptr(self):
        return 256


def _pitch(t):
    """Elements from one row of t's last dimension to the next: a view of a wider buffer keeps the buffer's pitch."""
    if isinstance(t, Spec) or t.dim() < 2:
        return t.shape[-1]
    if t.stride(-1) != 1 or any(t.shape[i] > 1 and t.stride(i) != t.stride(i + 1) * t.shape[i + 1] for i in range(t.dim() - 2)):
        raise RuntimeError("grl_b200: gemm outputs / residuals need unit-stride rows at one pitch")
    return t.stride(-2)


def gemm_problem(x16, w16, bias, *, M=0, image=None, kpad, npad, taps=1, epi=EPI_BIAS_ACT, n_store=0, n_real=0,
                 out_bf16=None, out_f32=None, res_f32=None, act=K.ACT_NONE, slope=0.0, slot_scale=None, C=0, gamma=None,
                 beta=None, eps=1e-5, res_scale=1.0, cab_y=None, cab_gate=None, L=1, ps_r=0, out_nchw=None, nchw_r=1,
                 post_scale=1.0, post_shift=None):
    """The GrlTcGemm of one launch (arguments: gemm)."""
    p = capi.GrlTcGemm()
    if x16.dtype != w16.dtype:
        raise RuntimeError("grl_b200: activation / weight operand formats differ")
    p.fmt = fmt_of(x16)
    p.x, p.w, p.bias = x16.data_ptr(), w16.data_ptr(), bias.data_ptr()
    p.M = M
    if image is not None:
        p.B, p.H, p.W = image
    p.kpad, p.npad, p.taps, p.epi = kpad, npad, taps, epi
    p.n_store, p.n_real = n_store, n_real
    if out_bf16 is not None:
        p.out_bf16, p.ldo_bf16 = out_bf16.data_ptr(), _pitch(out_bf16)
    if out_f32 is not None:
        p.out_f32, p.ldo_f32 = out_f32.data_ptr(), _pitch(out_f32)
    if res_f32 is not None:
        p.res_f32, p.ldr = res_f32.data_ptr(), _pitch(res_f32)
    p.act, p.slope = act, slope
    if slot_scale is not None:
        p.slot_scale = slot_scale.data_ptr()
    p.C = C
    if gamma is not None:
        p.gamma, p.beta = gamma.data_ptr(), beta.data_ptr()
    p.eps, p.res_scale = eps, res_scale
    if cab_y is not None:
        p.cab_y, p.ld_caby, p.cab_gate = cab_y.data_ptr(), _pitch(cab_y), cab_gate.data_ptr()
    p.L = L
    p.ps_r = ps_r
    if out_nchw is not None:  # (B, C_out, Hc, Wc) fp32 planes: denormalise + crop + bhwc -> bchw folded into the store
        p.out_nchw, p.nchw_r, p.Hc, p.Wc = out_nchw.data_ptr(), nchw_r, out_nchw.shape[2], out_nchw.shape[3]
        p.post_scale = post_scale
        for i in range(4):
            p.post_shift[i] = float(post_shift[i]) if post_shift is not None and i < len(post_shift) else 0.0
    return p


def gemm(x16, w16, bias, **kw):
    """One grl_tc_gemm launch (keyword arguments: gemm_problem)."""
    p = gemm_problem(x16, w16, bias, **kw)
    capi.check(capi.lib().grl_tc_gemm(ctypes.byref(p), capi.stream()))


class GemmLaunch(NamedTuple):
    """One tc.gemm call of a forward: `name` (e.g. "stage0.block1.fc1", "conv_last") and gemm_problem's arguments with
    their defaults applied and a Spec in place of every tensor."""
    name: str
    args: dict


def _spec(v):
    return Spec(tuple(v.shape), v.dtype) if isinstance(v, (torch.Tensor, Spec)) else v


def gemm_launch(name, x16, w16, bias, **kw):
    """The descriptor of gemm(x16, w16, bias, **kw)."""
    b = inspect.signature(gemm_problem).bind(x16, w16, bias, **kw)
    b.apply_defaults()
    return GemmLaunch(name, {k: _spec(v) for k, v in b.arguments.items()})


def gemm_path(launch):
    """grl_tc_gemm_path of a descriptor: the tile width, epilogue mode, tiling and grid the library picks for it."""
    out = capi.GrlTcGemmPath()
    p = gemm_problem(**launch.args)
    capi.check(capi.lib().grl_tc_gemm_path(ctypes.byref(p), ctypes.byref(out)))
    return out


class Device:
    """Launcher of a forward on the GPU: every kernel runs.  The forward hands it each launch a listing records
    (`listed`: its name, wrapper and arguments; the GEMMs, and the fp32 attention) and every other kernel (`run`, a
    wrapper and its arguments).  Outputs are allocated by the caller."""
    caches = True  # attention constants computed through it are real, so BlockPlan may keep them

    def listed(self, name, fn, *args, **kw):
        fn(*args, **kw)

    def run(self, fn, *args, **kw):
        fn(*args, **kw)


class Listing:
    """Launcher of a listing run: activations are meta tensors, every `listed` launch is recorded as (name, wrapper,
    args, kwargs) and nothing is launched."""
    caches = False

    def __init__(self):
        self.launches = []

    def listed(self, name, fn, *args, **kw):
        self.launches.append((name, fn, args, kw))

    def run(self, fn, *args, **kw):
        pass


DEVICE = Device()


def attention(gq, gk, q, q_off, k, k_off, v, v_off, out, o_off, B, heads, bias, use_mask, v_dense=False,
              o_dense=False, tag="attn", ones_col=False):
    p = capi.GrlTcAttn()
    p.fmt = fmt_of(q)
    p.gq, p.gk = gq, gk
    p.q, p.ldq, p.q_off = q.data_ptr(), q.shape[-1], q_off
    p.k, p.ldk, p.k_off = k.data_ptr(), k.shape[-1], k_off
    p.v, p.ldv, p.v_off, p.v_dense = v.data_ptr(), v.shape[-1], v_off, int(v_dense)
    p.out, p.ldo, p.o_off, p.o_dense = out.data_ptr(), out.shape[-1], o_off, int(o_dense)
    if bias.dim() != 3 or bias.shape[1] != 4:
        raise RuntimeError("grl_b200: attention bias must be the (heads, 4, rows_pad) table of bias_table_log2 / shifted_copies")
    p.B, p.heads, p.bias, p.use_mask = B, heads, bias.data_ptr(), int(use_mask)
    p.rows, p.rows_pad = (gq.wh + gk.wh - 1) * (gq.ww + gk.ww - 1), bias.shape[2]
    p.ones_col = int(ones_col)
    K._timed(tag, lambda: capi.check(capi.lib().grl_tc_attn(ctypes.byref(p), capi.stream())))


class AttnLaunch(NamedTuple):
    """One grl_tc_attn launch of a block.  q / k / v / out name an operand buffer and its first column: "qkv" (B*L,
    nslots*32) and "anchor" (B*La, hs*32) from the projections, "x1" the dense (B*nW*hs*Na, 32) stripe intermediate,
    "merged" (B*L, k_proj) the input of the output projection."""
    role: str  # "window", "stripe1" (anchors attend to the stripe's tokens), "stripe2" (tokens attend to the anchors)
    gq: object
    gk: object
    heads: int
    q: tuple
    k: tuple
    v: tuple
    out: tuple
    ones_col: bool
    use_mask: bool
    v_dense: bool
    o_dense: bool


def attention_launch(role, gq, gk, hw, hs, c, use_mask):
    """Descriptor of one of the three attention launches of a block with hw window heads, hs stripe heads and c = C / 2
    channels per half.  Host only: the QKV slot order is [window q|k|v][stripe q|k|v] x head (BlockPlan)."""
    if role == "window":
        return AttnLaunch(role, gq, gk, hw, ("qkv", 0), ("qkv", hw * SLOT), ("qkv", 2 * hw * SLOT), ("merged", 0),
                          c // hw < SLOT, use_mask, False, False)
    ones = c // hs < SLOT
    if role == "stripe1":  # writes X1 dense; with the ones column, X1[:, 31] == 1 is pass 2's denominator column
        return AttnLaunch(role, gq, gk, hs, ("anchor", 0), ("qkv", (3 * hw + hs) * SLOT), ("qkv", (3 * hw + 2 * hs) * SLOT),
                          ("x1", 0), ones, use_mask, False, True)
    if role == "stripe2":
        return AttnLaunch(role, gq, gk, hs, ("qkv", 3 * hw * SLOT), ("anchor", 0), ("x1", 0), ("merged", hw * SLOT), ones,
                          use_mask, True, False)
    raise ValueError(role)


def attention_launches(blk, x_size):
    """The three attention launches BlockPlan.run issues for block `blk` at resolution x_size: window attention, then
    stripe pass 1 and pass 2 through X1."""
    wa, sa = blk.attn.window_attn, blk.attn.stripe_attn
    hw, hs, c = wa.num_heads, sa.num_heads, blk.dim // 2
    s = wa.shift_size
    gw = G.token_grid(x_size, wa.window_size, (s, s))
    tok, anc = sa.grids(x_size)
    # the shift masks exist exactly for the shifted blocks (EfficientMixAttnTransformerBlock._get_table_index_mask)
    return (attention_launch("window", gw, gw, hw, hs, c, bool(blk.window_shift)),
            attention_launch("stripe1", anc, tok, hw, hs, c, bool(blk.stripe_shift)),
            attention_launch("stripe2", tok, anc, hw, hs, c, bool(blk.stripe_shift)))


def bias_rows_pad(rows):
    return round_up(rows + 16, 4)  # slack for the aligned over-reads of the shifted copies (16: staged rows, variant 4)


def shifted_copies(table_hr):
    """(heads, rows) fp32 -> (heads, 4, rows_pad): copy c shifted right by c entries (layout grl_tc_attn reads)."""
    heads, rows = table_hr.shape
    out = torch.zeros(heads, 4, bias_rows_pad(rows), device=table_hr.device, dtype=torch.float32)
    for c in range(4):
        out[:, c, c:c + rows] = table_hr
    return out


def bias_table_log2(transform, table, out):
    """16*sigmoid(cpb_mlp(table))*log2(e) as the 4-copy table of the attention kernel, written into `out`: zero-filled
    (heads, 4, bias_rows_pad(rows)) fp32."""
    t = table.reshape(-1, 2)
    w1, b1, w2 = transform.cpb_mlp[0].weight, transform.cpb_mlp[0].bias, transform.cpb_mlp[2].weight
    heads, hidden = w2.shape
    capi.check(capi.lib().grl_tc_bias_table4(capi.ptr(t), t.shape[0], capi.ptr(w1), capi.ptr(b1), capi.ptr(w2), hidden,
                                             heads, LOG2E, out.shape[2], capi.ptr(out), capi.stream()))


def slot_scale(ls_w, ls_s1, ls_s2, hw, hs, out):
    """The QKV epilogue's per-slot scales (nslots,) fp32 into `out` from the logit scales of window attention and of
    stripe passes 1 / 2, in slot order [window q|k|v][stripe q|k|v] x head (grl_tc_slot_scale)."""
    capi.check(capi.lib().grl_tc_slot_scale(capi.ptr(ls_w), capi.ptr(ls_s1), capi.ptr(ls_s2), hw, hs, capi.ptr(out),
                                            capi.stream()))


def avgpool16(x16, out, df):
    """Anchor pooling: the df x df mean of 16-bit (B, H, W, cpad) into 16-bit (B, H / df, W / df, cpad) `out`."""
    B, H, W, cpad = x16.shape
    capi.check(capi.lib().grl_tc_avgpool16(capi.ptr(x16), capi.ptr(out), B, H, W, cpad, df, fmt_of(x16), capi.stream()))


def maxpool16(x16, out, df):
    """Anchor pooling: the df x df max of 16-bit (B, H, W, cpad) into 16-bit (B, H / df, W / df, cpad) `out`."""
    B, H, W, cpad = x16.shape
    capi.check(capi.lib().grl_tc_maxpool16(capi.ptr(x16), capi.ptr(out), B, H, W, cpad, df, fmt_of(x16), capi.stream()))


def channel_gate(y16, ld, B, L, C, ca, gate):
    """CAB gate (B, C) fp32 into `gate` from the 16-bit features y16 (B*L, ld); ca: the packed ChannelAttention weights."""
    lib = capi.lib()
    nbytes = lib.grl_tc_channel_gate_workspace(B, L, C)
    ws = torch.empty(max(nbytes, 4) // 4, device=y16.device, dtype=torch.float32)
    w1, b1, w2, b2 = ca
    capi.check(lib.grl_tc_channel_gate(capi.ptr(y16), ld, fmt_of(y16), B, L, C, capi.ptr(w1), capi.ptr(b1), capi.ptr(w2),
                                       capi.ptr(b2), w1.shape[0], capi.ptr(gate), capi.ptr(ws), nbytes, capi.stream()))


def conv3x3(x16, wpack, bias, cin_pad, npad, *, n_store, launch=DEVICE, name="", **kw):
    """x16 16-bit (B, H, W, cin_pad) channels-last; kw: gemm's outputs, residual, activation and head-tail fusion."""
    B, H, W, _ = x16.shape
    launch.listed(name, gemm, x16, wpack, bias, image=(B, H, W), kpad=cin_pad, npad=npad, taps=9, epi=EPI_BIAS_ACT,
                  n_store=n_store, **kw)


def _version_key(module):
    return tuple((p.data_ptr(), p._version) for p in module.parameters())


class BlockPlan:
    """Packed weights + launch sequence of one EfficientMixAttnTransformerBlock.  `ready` orders the packed weights
    for the streams that read them, `_consts` the attention constants (streams.Produced)."""

    def __init__(self, blk, fmt):
        self.key = (_version_key(blk), fmt)
        self.fmt = fmt
        self._const_key, self._consts = None, None
        at = blk.attn
        C = blk.dim
        c = C // 2
        hw, hs = at.window_attn.num_heads, at.stripe_attn.num_heads
        dw, ds = c // hw, c // hs
        self.C, self.cpad, self.hw, self.hs = C, round_up(C, 64), hw, hs
        self.nslots = 3 * hw + 3 * hs
        dev = at.qkv.body.weight.device
        # --- QKV: dest row = slot*32 + e, slots [window q|k|v][stripe q|k|v] x head; source rows are already ordered
        # (half, t, head, e) in the reference layout (efficient.py:150,:251,:362)
        rmap = torch.cat([_slot_rows(0, 3 * hw, dw, dev), _slot_rows(3 * hw, 3 * hs, ds, dev)])
        self.n_qkv = self.nslots * SLOT
        self.w_qkv = _pad_matrix(at.qkv.body.weight, self.n_qkv, self.cpad, row_map=rmap, fmt=fmt)
        self.b_qkv = _pad_vector(at.qkv.body.bias if at.qkv.body.bias is not None else torch.zeros(3 * C, device=dev), self.n_qkv, rmap)
        # ones-column (attn_tc.cu): with head_dim < 32 the last slot column of every VALUE slot is 1 (set through the
        # bias; its weight row is zero), so the P V MMA also produces the softmax denominator.  The stripe pass-1 output
        # X1 inherits it (O[:, 31] / O[:, 31] == 1) and is the value operand of pass 2.
        self.ones_w, self.ones_s = dw < SLOT, ds < SLOT
        for half, (hh, on) in enumerate(((hw, self.ones_w), (hs, self.ones_s))):
            if on:
                base = (0 if half == 0 else 3 * hw) + 2 * hh
                self.b_qkv.view(-1, SLOT)[base:base + hh, SLOT - 1].fill_(1.0)  # fill_: a scalar store would sync
        # --- anchor projection: its stages (AnchorProjection.body), each a pooling or a patch gather (K.anchor_gather:
        # K = taps * C padded to 64) in front of one GEMM.  The last writes the anchors at row head*32 + e (EPI_QKV);
        # the others write their C/2 channels at a 64-padded pitch (bias epilogue, PatchMerging's bias is zero).
        amap = _slot_rows(0, hs, ds, dev)
        self.n_anc = hs * SLOT
        self.anc_scale = torch.ones(hs, device=dev, dtype=torch.float32)
        self.anc_stages = []
        cin = C
        body = list(at.anchor.body)
        for i, m in enumerate(body):
            last = i == len(body) - 1
            if hasattr(m, "pooling_mode"):  # AnchorLinear: kind "avgpool" / "maxpool", geo = the pooling window df
                kind, w, b, geo, kpad = m.pooling_mode, m.reduction.weight, m.reduction.bias, m.down_factor, self.cpad
            else:  # AnchorConv2d / PatchMerging: kind "gather", geo = its modules.AnchorGather
                kind, (w, b), geo = "gather", m.packed(), m.gather
                kpad = round_up(geo.ksize ** 2 * cin, 64)
            npad = round_up(self.n_anc, 32) if last else round_up(C // 2, 64)
            rmap = amap if last else None
            self.anc_stages.append((kind, geo, _pad_matrix(w, npad, kpad, row_map=rmap, fmt=fmt), _pad_vector(b, npad, rmap, dev),
                                    cin, kpad, npad))
            cin = C // 2
        self.w_anc, self.b_anc = self.anc_stages[-1][2:4]  # the projection that writes the anchors
        # --- output projection: K index = slot*32 + e over [window heads | stripe heads]
        cmap = torch.cat([_slot_rows(0, hw, dw, dev), _slot_rows(hw, hs, ds, dev)])
        self.k_proj = round_up((hw + hs) * SLOT, 64)
        self.n_ln = 64 if C <= 64 else 128 if C <= 128 else 192 if C <= 192 else 256
        self.w_proj = _pad_matrix(at.proj.weight, self.n_ln, self.k_proj, col_map=cmap, fmt=fmt)
        self.b_proj = _pad_vector(at.proj.bias, self.n_ln)
        # --- MLP
        hid = blk.mlp.fc1.weight.shape[0]
        self.hid, self.hpad = hid, round_up(hid, 64)
        self.w_fc1 = _pad_matrix(blk.mlp.fc1.weight, self.hpad, self.cpad, fmt=fmt)
        self.b_fc1 = _pad_vector(blk.mlp.fc1.bias, self.hpad)
        self.w_fc2 = _pad_matrix(blk.mlp.fc2.weight, self.n_ln, self.hpad, fmt=fmt)
        self.b_fc2 = _pad_vector(blk.mlp.fc2.bias, self.n_ln)
        # --- CAB
        self.cab = bool(blk.args.local_connection)
        if self.cab:
            c0, c2 = blk.conv.cab[0], blk.conv.cab[2]
            self.cmid = c0.weight.shape[0]
            self.cmid_pad = round_up(self.cmid, 64)
            self.w_cab1, self.b_cab1 = pack_conv(c0, self.cpad, self.cmid_pad, fmt)
            self.w_cab2, self.b_cab2 = pack_conv(c2, self.cmid_pad, self.cpad, fmt)
            a1, a3 = blk.conv.cab[3].attention[1], blk.conv.cab[3].attention[3]
            self.ca = (a1.weight.detach().reshape(a1.weight.shape[0], -1).contiguous(), a1.bias.detach(),
                       a3.weight.detach().reshape(a3.weight.shape[0], -1).contiguous(), a3.bias.detach())
        self.ready = Produced([v for k, v in vars(self).items() if k != "_consts"])

    @torch.no_grad()
    def run(self, blk, x32, x16, x_size, all_table_index_mask, launch=DEVICE, name=""):
        """x32 fp32 (B, L, C), x16 16-bit (B, L, cpad) or None -> (x32', x16').  Launches through `launch`; GEMMs are
        named "{name}.qkv" etc."""
        t = blk._get_table_index_mask(all_table_index_mask)
        x32 = x32 if x32.is_contiguous() else x32.contiguous()
        B, L, C = x32.shape
        H, W = x_size
        dev = x32.device
        at = blk.attn
        hw, hs, cpad = self.hw, self.hs, self.cpad
        fmt = self.fmt
        if x16 is None or x16.dtype != DTYPE[fmt]:
            x16 = _h16(B, L, cpad, device=dev, fmt=fmt)
            launch.run(pack_rows, x32, cpad, fmt, out=x16)
        wa, sa = at.window_attn, at.stripe_attn
        # attention constants of this block (slot scales + activated bias tables): functions of the parameters and
        # the coordinate tables only, so they are cached until a parameter or the resolution changes
        ckey = (self.key, t["table_w"].data_ptr(), t["table_s"].data_ptr(), t["table_s"].shape)
        if self._const_key == ckey:
            scales, bias_w, bias_1, bias_2 = self._consts.use()
        else:
            scales = torch.empty(self.nslots, device=dev, dtype=torch.float32)
            launch.run(slot_scale, wa.attn_transform.logit_scale, sa.attn_transform1.logit_scale,
                       sa.attn_transform2.logit_scale, hw, hs, scales)
            tables = ((wa.attn_transform, t["table_w"]), (sa.attn_transform1, t["table_s"]),
                      (sa.attn_transform2, t["table_s"]))
            bias_w, bias_1, bias_2 = [torch.zeros(tr.cpb_mlp[2].weight.shape[0], 4, bias_rows_pad(tb.numel() // 2),
                                                  device=dev, dtype=torch.float32) for tr, tb in tables]
            for (tr, tb), out in zip(tables, (bias_w, bias_1, bias_2)):
                launch.run(bias_table_log2, tr, tb, out)
            if launch.caches:  # never keep a listing run's meta constants: a later forward would launch with them
                self._const_key, self._consts = ckey, Produced((scales, bias_w, bias_1, bias_2))
        # projections
        qkv = _h16(B * L, self.n_qkv, device=dev, fmt=fmt)
        launch.listed(f"{name}.qkv", gemm, x16, self.w_qkv, self.b_qkv, M=B * L, kpad=cpad, npad=self.n_qkv,
                      epi=EPI_QKV, n_store=self.n_qkv, out_bf16=qkv, slot_scale=scales)
        a16, (h, w) = x16.view(B, H, W, cpad), (H, W)
        for i, (kind, geo, w_a, b_a, cin, kpad, npad) in enumerate(self.anc_stages):
            last = i == len(self.anc_stages) - 1
            if kind != "gather":
                h, w = h // geo, w // geo
                rows = _h16(B, h, w, cpad, device=dev, fmt=fmt)
                launch.run(avgpool16 if kind == "avgpool" else maxpool16, a16, rows, geo)
            else:
                h, w = K.gather_size(h, w, geo.ksize, geo.stride, geo.pad)
                rows = _h16(B * h * w, kpad, device=dev, fmt=fmt)
                launch.run(K.anchor_gather, a16, cin, *geo, kpad, out=rows)
            out = _h16(B * h * w, npad, device=dev, fmt=fmt)
            if last:
                launch.listed(f"{name}.anchor", gemm, rows, w_a, b_a, M=B * h * w, kpad=kpad, npad=npad, epi=EPI_QKV,
                              n_store=npad, out_bf16=out, slot_scale=self.anc_scale)
            else:
                launch.listed(f"{name}.anchor.{i}", gemm, rows, w_a, b_a, M=B * h * w, kpad=kpad, npad=npad,
                              epi=EPI_BIAS_ACT, n_store=npad, out_bf16=out)
            a16 = out.view(B, h, w, npad)
        anchor = out
        # attention
        merged = _h16(B * L, self.k_proj, device=dev, fmt=fmt, zero=self.k_proj != (hw + hs) * SLOT)
        launches = attention_launches(blk, x_size)
        anc = launches[1].gq
        nW = (anc.H // anc.wh) * (anc.W // anc.ww)
        x1 = _h16(B * nW * hs * anc.wh * anc.ww, SLOT, device=dev, fmt=fmt)
        buf = {"qkv": qkv, "anchor": anchor, "x1": x1, "merged": merged}
        bias = {"window": bias_w, "stripe1": bias_1, "stripe2": bias_2}
        for ln in launches:
            launch.run(attention, ln.gq, ln.gk, buf[ln.q[0]], ln.q[1], buf[ln.k[0]], ln.k[1], buf[ln.v[0]], ln.v[1],
                       buf[ln.out[0]], ln.out[1], B, ln.heads, bias[ln.role], ln.use_mask, v_dense=ln.v_dense,
                       o_dense=ln.o_dense, tag="window_attn" if ln.role == "window" else "stripe_attn", ones_col=ln.ones_col)
        # CAB
        cab_y = gate = None
        if self.cab:
            t1 = _h16(B, H, W, self.cmid_pad, device=dev, fmt=fmt)
            conv3x3(x16.view(B, H, W, cpad), self.w_cab1, self.b_cab1, cpad, self.cmid_pad, n_store=self.cmid_pad,
                    act=K.ACT_GELU, out_bf16=t1, launch=launch, name=f"{name}.cab1")
            cab_y = _h16(B * L, cpad, device=dev, fmt=fmt)
            conv3x3(t1, self.w_cab2, self.b_cab2, self.cmid_pad, cpad, n_store=cpad, out_bf16=cab_y, launch=launch,
                    name=f"{name}.cab2")
            gate = torch.empty(B, C, device=dev, dtype=torch.float32)
            launch.run(channel_gate, cab_y, cpad, B, L, C, self.ca, gate)
        # proj + LN1 + residual (+ CAB)
        y32 = torch.empty(B, L, C, device=dev, dtype=torch.float32)
        y16 = _h16(B, L, cpad, device=dev, fmt=fmt)
        launch.listed(f"{name}.proj", gemm, merged, self.w_proj, self.b_proj, M=B * L, kpad=self.k_proj,
                      npad=self.n_ln, epi=EPI_LN, n_store=self.n_ln, n_real=C, out_bf16=y16, out_f32=y32, res_f32=x32,
                      C=C, gamma=blk.norm1.weight, beta=blk.norm1.bias, eps=blk.norm1.eps, res_scale=blk.res_scale,
                      cab_y=cab_y, cab_gate=gate, L=L)
        # MLP + LN2 + residual
        hid = _h16(B * L, self.hpad, device=dev, fmt=fmt)
        launch.listed(f"{name}.fc1", gemm, y16, self.w_fc1, self.b_fc1, M=B * L, kpad=cpad, npad=self.hpad,
                      epi=EPI_BIAS_ACT, n_store=self.hpad, act=K.ACT_GELU, out_bf16=hid)
        z32 = torch.empty(B, L, C, device=dev, dtype=torch.float32)
        z16 = _h16(B, L, cpad, device=dev, fmt=fmt)
        launch.listed(f"{name}.fc2", gemm, hid, self.w_fc2, self.b_fc2, M=B * L, kpad=self.hpad, npad=self.n_ln,
                      epi=EPI_LN, n_store=self.n_ln, n_real=C, out_bf16=z16, out_f32=z32, res_f32=y32, C=C,
                      gamma=blk.norm2.weight, beta=blk.norm2.bias, eps=blk.norm2.eps, res_scale=blk.res_scale, L=L)
        return z32, z16


def block_plan(blk, fmt):
    plan = getattr(blk, "_tc_plan", None)
    if plan is None or plan.key != (_version_key(blk), fmt):
        plan = BlockPlan(blk, fmt)
        blk._tc_plan = plan
    plan.ready.use()
    return plan


class ConvPlan:
    """One packed 3x3 conv (stage conv / head convs), or a 1x1 conv / per-pixel nn.Linear (stage conv types "1conv1x1",
    "linear" and the middle conv of "3conv": one GEMM over the pixels)."""

    def __init__(self, conv, cin_pad, fmt, ps_r=0):
        self.key = (_version_key(conv), fmt, ps_r)
        self.cout = conv.weight.shape[0]
        self.cin_pad, self.ps_r = cin_pad, ps_r
        self.npad = round_up(self.cout, 64)
        self.taps = 9 if conv.weight.dim() == 4 and conv.weight.shape[2] == 3 else 1
        if self.taps == 9:
            self.w, self.b = pack_conv(conv, cin_pad, self.npad, fmt, ps_r)
        else:
            self.w = _pad_matrix(conv.weight.reshape(self.cout, -1), self.npad, cin_pad, fmt=fmt)
            self.b = _pad_vector(conv.bias, self.npad)
        self.ready = Produced((self.w, self.b))

    def run(self, launch, name, x16, *, want16=True, want_f32=False, rows=False, **kw):
        """One launch on x16 (B, H, W, cin_pad) channels-last -> (16-bit out, fp32 out), each None unless asked for:
        (B, H, W, npad) and (B, H, W, cout), or (B, H*W, .) with rows; with ps_r the 16-bit output is the shuffled
        (B, H r, W r, cout / r^2).  kw: residual, activation and the NCHW tail (conv3x3)."""
        B, H, W, _ = x16.shape
        r, dev = self.ps_r, x16.device
        px = (B, H * W) if rows else (B, H, W)
        o16 = o32 = None
        if r:
            o16 = torch.empty(B, H * r, W * r, self.cout // (r * r), device=dev, dtype=self.w.dtype)
        elif want16:
            o16 = torch.empty(*px, self.npad, device=dev, dtype=self.w.dtype)
        if want_f32:
            o32 = torch.empty(*px, self.cout, device=dev, dtype=torch.float32)
        if self.taps == 1:
            launch.listed(name, gemm, x16, self.w, self.b, M=B * H * W, kpad=self.cin_pad, npad=self.npad,
                          epi=EPI_BIAS_ACT, n_store=self.npad, n_real=self.cout, out_bf16=o16, out_f32=o32, **kw)
        else:
            conv3x3(x16, self.w, self.b, self.cin_pad, self.npad, n_store=self.cout if r else self.npad,
                    n_real=self.cout, out_bf16=o16, out_f32=o32, ps_r=r, launch=launch, name=name, **kw)
        return o16, o32


def conv_plan(owner, name, conv, cin_pad, fmt, ps_r=0):
    cache = owner.__dict__.setdefault("_tc_convs", {})
    plan = cache.get(name)
    if plan is None or plan.key != (_version_key(conv), fmt, ps_r) or plan.cin_pad != cin_pad:
        plan = ConvPlan(conv, cin_pad, fmt, ps_r)
        cache[name] = plan
    plan.ready.use()
    return plan


def last_conv(owner, key, x16, fmt, launch, name, **kw):
    """build_last_conv's block `owner.<key>` on x16 (B, H, W, cin_pad), as ConvPlan.run (kw: its outputs and the
    residual).  "3conv" runs conv3x3 + LeakyReLU, conv1x1 + LeakyReLU (launched as "{name}.0", ".2") at the 64-padded
    C/4 width, then the last conv with kw as "{name}.4"."""
    m = owner.get_submodule(key)
    if isinstance(m, nn.Sequential):
        t, _ = conv_plan(owner, f"{key}.0", m[0], x16.shape[-1], fmt).run(launch, f"{name}.0", x16, act=K.ACT_LEAKY,
                                                                          slope=m[1].negative_slope)
        t, _ = conv_plan(owner, f"{key}.2", m[2], t.shape[-1], fmt).run(launch, f"{name}.2", t, act=K.ACT_LEAKY,
                                                                        slope=m[3].negative_slope)
        return conv_plan(owner, f"{key}.4", m[4], t.shape[-1], fmt).run(launch, f"{name}.4", t, **kw)
    return conv_plan(owner, key, m, x16.shape[-1], fmt).run(launch, name, x16, **kw)


@torch.no_grad()
def stage_forward(stage, x32, x16, x_size, table_index_mask, launch=DEVICE, name=""):
    """TransformerStage on the explicit (fp32 stream (B, L, C), 16-bit operand copy or None) pair: its blocks, then
    conv3x3 + residual; returns the pair.  GEMMs are named "{name}.block{i}.qkv", ..., "{name}.conv"."""
    B, L, C = x32.shape
    H, W = x_size
    fmt = FMT[stage.blocks[0].precision]
    cpad = round_up(C, 64)
    r32, r16 = x32, x16
    for bi, blk in enumerate(stage.blocks):
        r32, r16 = block_plan(blk, FMT[blk.precision]).run(blk, r32, r16, x_size, table_index_mask, launch,
                                                           f"{name}.block{bi}")
    if r16 is None or r16.dtype != DTYPE[fmt]:
        r16 = _h16(B, L, cpad, device=x32.device, fmt=fmt)
        launch.run(pack_rows, r32.contiguous(), cpad, fmt, out=r16)
    o16, o32 = last_conv(stage, "conv", r16.view(B, H, W, cpad), fmt, launch, f"{name}.conv", want_f32=True, rows=True,
                         res_f32=x32.contiguous())
    return o32, o16


@torch.no_grad()
def forward(model, x, rggb=False, launch=DEVICE):
    """GRL `model` on the tensor-core kernels (grl.py:506-551); x is the RAW (B, Cin, H, W) fp32 input, or with rggb its
    packed (B, 4, H/2, W/2) Bayer planes.  Head: one kernel does [dm_matlab +] check_image_size + (x - mean) * img_range +
    bchw -> bhwc + operand pack; tail: the last conv's epilogue writes x / img_range + mean, cropped, as bchw planes;
    PixelShuffle is a store-address pattern of the conv before it.  Buffers are allocated on x's device."""
    dev = x.device
    fmt = FMT[model.precision]
    B, Cin, H, W = x.shape
    if rggb:
        Cin, H, W = 3, 2 * H, 2 * W
    Hp, Wp = round_up(H, model.pad_size), round_up(W, model.pad_size)
    C = model.embed_dim
    cpad = round_up(C, 64)
    s = model.upscale
    need_res = model.upsampler not in ("pixelshuffle", "pixelshuffledirect", "nearest+conv") and model.in_channels == model.out_channels
    mean = model._mean_list
    x16 = _h16(B, Hp, Wp, 64, device=dev, fmt=fmt)
    xc32 = torch.empty(B, Hp, Wp, Cin, device=dev, dtype=torch.float32) if need_res else None
    launch.run(head_pack_rggb if rggb else head_pack, x, Hp, Wp, mean, model.img_range, 64, fmt, out=(x16, xc32))
    shift = mean if len(mean) > 1 else mean * 4

    def conv(name, module, inp16, ps_r=0, **kw):
        return conv_plan(model, name, module, inp16.shape[-1], fmt, ps_r).run(launch, name, inp16, **kw)

    def last(name, module, inp16, r=1, res=None):  # network output: (B, C_out, H s, W s) planes straight from the epilogue
        y = torch.empty(B, model.out_channels, H * s, W * s, device=dev, dtype=torch.float32)
        conv(name, module, inp16, want16=False, res_f32=res, out_nchw=y, nchw_r=r, post_scale=1.0 / model.img_range,
             post_shift=shift)
        return y

    def ln(norm, u):
        out = torch.empty(u.shape, device=dev, dtype=torch.float32)  # not empty_like: on meta, its first call imports sympy
        launch.run(K.ln_residual, None, u, norm.weight, norm.bias, norm.eps, out=out)
        return out

    _, f32 = conv("conv_first", model.conv_first, x16, want_f32=True)
    t = ln(model.norm_start, f32.view(B, Hp * Wp, C))
    tim = model.get_table_index_mask(dev, (Hp, Wp))
    t16 = None  # 16-bit operand copy of the residual stream, carried explicitly from block to block
    for si, layer in enumerate(model.layers):
        t, t16 = stage_forward(layer, t, t16, (Hp, Wp), tim, launch, f"stage{si}")
    t = ln(model.norm_end, t)
    t16 = _h16(B, Hp, Wp, cpad, device=dev, fmt=fmt)
    launch.run(pack_rows, t, cpad, fmt, out=t16)
    body16, _ = last_conv(model, "conv_after_body", t16, fmt, launch, "conv_after_body", res_f32=f32)
    if model.upsampler == "pixelshuffle":
        u16, _ = conv("conv_before_upsample", model.conv_before_upsample[0], body16, act=K.ACT_LEAKY, slope=0.01)
        mods = list(model.upsample.up)
        for i, m in enumerate(mods):
            if isinstance(m, nn.Conv2d):  # always followed by its PixelShuffle (upsample.py:6-30)
                u16, _ = conv(f"upsample.up.{i}", m, u16, ps_r=mods[i + 1].upscale_factor)
        return last("conv_last", model.conv_last, u16)
    if model.upsampler == "pixelshuffledirect":
        return last("upsample.up.0", model.upsample.up[0], body16, model.upsample.up[1].upscale_factor)
    if model.upsampler == "nearest+conv":
        u16, _ = conv("conv_before_upsample", model.conv_before_upsample[0], body16, act=K.ACT_LEAKY, slope=0.01)
        up = lambda v: v.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).contiguous()
        u16, _ = conv("conv_up1", model.conv_up1, up(u16), act=K.ACT_LEAKY, slope=0.2)
        u16, _ = conv("conv_up2", model.conv_up2, up(u16), act=K.ACT_LEAKY, slope=0.2)
        u16, _ = conv("conv_hr", model.conv_hr, u16, act=K.ACT_LEAKY, slope=0.2)
        return last("conv_last", model.conv_last, u16)
    return last("conv_last", model.conv_last, body16, res=xc32)


def gemm_launches(model, x_shape):
    """Descriptors of every GEMM launch of one tensor-core forward of GRL `model` on a (B, Cin, H, W) input, in launch
    order (operand format: model.precision): `forward` run with the Listing launcher on a meta input.  With
    model.input_format == "rggb", x_shape is the packed (B, 4, h, w) Bayer input and the network runs on the (2h, 2w)
    image.  Needs no device: weights are packed on the model's device and nothing is launched."""
    listing = Listing()
    forward(model, torch.empty(x_shape, device="meta"), model.input_format == "rggb", listing)
    return [gemm_launch(name, *args, **kw) for name, _, args, kw in listing.launches]
