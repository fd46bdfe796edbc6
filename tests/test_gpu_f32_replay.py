"""Real fp32 forwards checked launch by launch against float64, and the caches that outlive a forward.

`Replay32` is a tc.Device launcher for GRL._forward_f32: before each launch it fills the launch's outputs with NaN, then
runs it, synchronises and checks it on the operands the forward really handed it before the next one runs.  So every
kernel of csrc/ops_f32.cu is gated on what the previous kernels wrote (trained-like bias tables, real residual streams,
correlated q / k), with the bounds and gates of test_gpu_f32_paths.py (tests/f32_cases.py):
  K.linear / K.conv3x3: grl_oracle.gemm_launch_reference of the input the launch received, within gemm_bound per
    element; a conv's reference weight is its module's current `weight`, and the packed weight it received must equal
    K.pack_conv_weight(weight) bit for bit (a stale `_f32_convs` entry fails);
  K.window_attention: attn_ref of the launch's own qkv view, grid, logit scales, table and mask flag (GATE_ATTN);
  K.stripe_attention: issued again with a workspace the checker owns (its output must equal the launch's bit for bit),
    then pass 1's X1 and pass 2 on the kernel's own X1 against attn_ref (GATE_ATTN), and pass 2 against the float64
    chain (GATE_CHAIN).  Each attention gate also allows the sequential sums' error over the launch's key count
    (f32_cases.attn_ratio): a GRL-Base stripe pass 1 over 9216 keys whose v share one sign exceeds the ulp gate alone
    (2255 / 1695 ulp) while within 0.3 of that term.  At most 16 windows per attention launch (the first, the last (masked and rolled) and 14 seeded
    others); every window in the first and last block of each stage;
  K.bias_table within bias_table_bound on the coordinates it received; those coordinates equal grl_oracle.coords_table
    of the consuming attention's own geometry (window, oriented stripe, df), and the table an attention launch receives
    was written by its own block's AffineTransform for that pass;
  K.ln_residual within grl_oracle.ln_bound, K.channel_gate within gate_bound, K.avgpool bit for bit, K.demosaic bit for
    bit against the library's host demosaic;
  consumers: the input of each block's QKV linear, anchor avgpool, CAB conv and fc1, and of each stage conv and
    conv_after_body, is bit for bit the latest fp32 residual-stream output; the stage conv's residual is the stage's
    input; each ln_residual gets its block's proj / fc2 output, CAB features and gate; conv_first's input is
    (check_image_size(x) - mean) img_range recomputed here; every tail conv's input is the torch-op glue (pixel shuffle,
    nearest x2) of the conv before it, and the output is the last conv's, cropped, / img_range + mean;
  integrity: every output element is written; every written buffer is check-summed right after its launch and must
    have the same sum when a later launch reads it; a wrapper without a checker fails.
Mutation controls, computed on the reference side (never an edited kernel), at the first and last block of each stage
that has a previous block: the QKV linear fed the previous block's input, ln_residual given the previous block's
residual, window attention with the previous block's table and logit scales, the CAB gate of the previous block; and at
the sizes the test commands run (`command:` cases, tests/command_cases.py) the output cropped at the padded pitch (where
Wc < Wp) and shifted window attention with the shift mask of the transposed window grid (non-square grids).  A
mutation applies where it moves the float64 result by more than twice the gate, and must fail its gate wherever it
applies; the other blocks are counted apart.  A `command:` case's output is also compared end to end with
oracle.grl_forward on the device (command_cases.end_to_end).
"""
import copy
import time
import weakref

import pytest
import torch
import torch.nn.functional as F

import archs
import command_cases as CC
import f32_cases as C
import grl_oracle as O
from _pkgload import load_package
from f32_cases import GATE_ATTN, GATE_CHAIN
from replay_base import Recorder, ReplayBase, replay_case
from support import bound_ratio, grid_t

load_package()
from grl_image_restoration_b200 import capi, functional as KF, tc as TC  # noqa: E402

MUTATIONS = ("qkv fed the previous block's input", "ln_residual given the previous block's residual",
             "window attention with the previous block's table and logit scales", "CAB gate of the previous block",
             "output cropped at the padded pitch", "window attention on the transposed window grid's geometry")
STREAM_READERS = (".qkv", ".cab1", ".fc1", ".conv", "conv_after_body")  # launches whose input is the residual stream
TAIL = ("conv_first", "conv_after_body", "conv_before_upsample", "upsample.", "conv_up1", "conv_up2", "conv_hr",
        "conv_last")


def checkers(K):
    """Wrapper -> Replay32 method that checks it: every kernel GRL._forward_f32 launches must have one."""
    return {K.linear: "linear", K.conv3x3: "conv", K.window_attention: "window", K.stripe_attention: "stripe",
            K.bias_table: "bias_table", K.ln_residual: "ln_residual", K.channel_gate: "channel_gate",
            K.avgpool: "avgpool", K.demosaic: "demosaic"}


def same32(a, b):
    """Same shape and the same 32-bit patterns everywhere."""
    return a.numel() == b.numel() and bool(torch.equal(a.contiguous().view(torch.int32).reshape(-1),
                                                       b.contiguous().view(torch.int32).reshape(-1)))


def conv_module(model, name):
    """The nn.Conv2d a conv launch of the fp32 forward is named after."""
    parts = name.split(".")
    if parts[0].startswith("stage"):
        layer = model.layers[int(parts[0][5:])]
        if parts[1] == "conv":
            return layer.conv
        return layer.blocks[int(parts[1][5:])].conv.cab[{"cab1": 0, "cab2": 2}[parts[2]]]
    if name == "conv_before_upsample":
        return model.conv_before_upsample[0]
    return model.get_submodule(name)


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


class Replay32(ReplayBase, TC.Device):
    """tc.Device that checks every launch of GRL._forward_f32 (module docstring); x and rggb are the forward's input.
    Results as replay_base.ReplayBase."""
    poison = True

    def __init__(self, model, x, rggb=False, mutate=True, seed=0):
        super().__init__(model, MUTATIONS, mutate, seed)
        self.methods = checkers(KF)
        self.x, self.rggb = x, rggb
        self.tables = {}  # data_ptr of a bias_table output -> (weakref to it, the coordinates it got, block, role)
        self.transform = {}  # id(cpb_mlp[0].weight) -> (block, role)
        self.norm = {id(model.norm_start.weight): (None, "norm_start"), id(model.norm_end.weight): (None, "norm_end")}
        for name, (blk, _, _, _) in self.blocks.items():
            wa, sa = blk.attn.window_attn, blk.attn.stripe_attn
            for role, tr in (("window", wa.attn_transform), ("stripe1", sa.attn_transform1),
                             ("stripe2", sa.attn_transform2)):
                self.transform[id(tr.cpb_mlp[0].weight)] = (name, role)
            self.norm[id(blk.norm1.weight)] = (name, "norm1")
            self.norm[id(blk.norm2.weight)] = (name, "norm2")
        self.stream32 = None  # the latest fp32 residual-stream output
        self.stage_in = None  # the input of the current stage
        self.outs = {}  # launch name -> output, for the current block's GEMMs and the head and tail convs
        self.gate_out = None  # the current block's CAB gate

    def _block_changed(self):
        self.outs = {k: v for k, v in self.outs.items() if ".block" not in k}
        self.gate_out = None

    # ---- outputs of each wrapper ------------------------------------------------------------------
    def _outs_linear(self, *a, out=None, **kw):
        return [out]

    _outs_conv = _outs_linear
    _outs_bias_table = _outs_linear
    _outs_ln_residual = _outs_linear
    _outs_channel_gate = _outs_linear
    _outs_avgpool = _outs_linear
    _outs_demosaic = _outs_linear

    def _outs_window(self, *a):
        return [a[7]]

    def _outs_stripe(self, *a):
        return [a[11]]

    # ---- GEMM -------------------------------------------------------------------------------------
    def _gemm(self, name, conv, x, w64, bias, act, slope, res, out):
        """Gates `out` of act(x w^T + b) (+ res) against float64; returns (reference, bound, reference of another x)."""
        N = w64.shape[0]
        taps = 9 if conv else 1
        x64 = x.double() if conv else x.reshape(-1, x.shape[-1]).double()
        b64 = torch.zeros(N, dtype=torch.float64, device=x.device) if bias is None else bias.detach().double()
        r64 = None if res is None else res.reshape(-1, N).double()

        def ref(xx, **kw):
            return O.gemm_launch_reference(xx, w64, b64, taps=taps, **kw)["y"]

        v = ref(x64)
        absdot = O.gemm_launch_reference(x64.abs(), w64.abs(), torch.zeros_like(b64), taps=taps)["y"]
        bound, _ = C.gemm_bound_of(v, absdot, w64.shape[1], act, slope, r64)
        y = ref(x64, act=act, slope=slope, n_res=N, res=r64)
        r = bound_ratio(out.reshape(-1, N), y, bound)
        self._gate(f"{'conv' if conv else 'linear'} (error / bound)", r, 1.0, r <= 1.0, name)
        return y, bound, lambda xx: ref(xx.double(), act=act, slope=slope, n_res=N, res=r64)

    def _check_linear(self, x, weight, bias=None, act=0, slope=0.0, res=None, out=None, _name=None):
        if ".block" in _name:
            self._set_block(_name.rsplit(".", 1)[0])
        self._consumer(_name, x, res)
        y, bound, other = self._gemm(_name, False, x, weight.detach().double(), bias, act, slope, res, out)
        if _name.endswith(".qkv"):
            px = self.saved.get(self.prev, {}).get("x")
            if self._mutation_here() and px is not None and px.shape == x.shape:
                self._control(MUTATIONS[0], bound_ratio, out.reshape(y.shape), y, other(px.reshape(y.shape[0], -1)),
                              bound, 1.0)
            self.saved.setdefault(self.block, {})["x"] = x.clone()
        self.outs[_name] = out

    def _check_conv(self, x, wpacked, bias=None, act=0, slope=0.0, res=None, out=None, _name=None):
        weight = conv_module(self.model, _name).weight
        self._exact("packed conv weight == pack_conv_weight(module weight)",
                    same32(wpacked, KF.pack_conv_weight(weight)), _name)
        self._consumer(_name, x, res)
        N = weight.shape[0]
        self._gemm(_name, True, x, weight.detach().double().permute(0, 2, 3, 1).reshape(N, -1), bias, act, slope, res,
                   out)
        self.outs[_name] = out
        if _name.startswith("stage") and _name.endswith(".conv"):
            self.stream32 = out

    def _control(self, name, stat, got, ref, mut, bound, gate):
        """A mutation control: it applies where `mut` is more than twice the gate from `ref`, and then `got` must fail
        the gate against it."""
        if stat(mut, ref, bound) > 2 * gate:
            self._mut(name, stat(got, mut, bound) > gate)
        else:
            self._below(name)

    # ---- consumers --------------------------------------------------------------------------------
    def _head_ref(self):
        """conv_first's input: (check_image_size(x) - mean) img_range, channels last, recomputed with torch ops."""
        m = self.model
        x = KF.demosaic_host(self.x.cpu()).to(self.x.device) if self.rggb else self.x.float()
        H, W = x.shape[2:]
        ph, pw = (m.pad_size - H % m.pad_size) % m.pad_size, (m.pad_size - W % m.pad_size) % m.pad_size
        pad = (0, pw, 0, ph)
        x = F.pad(x, pad, "reflect") if (ph < H and pw < W) else F.pad(x, pad, "constant", 0.0)
        return nhwc((x - m.mean.to(x.device)) * m.img_range)

    def _tail_in(self, name):
        """The input the torch-op glue of the tail gives the conv `name`, from the outputs of the convs before it."""
        m, o = self.model, self.outs
        up = lambda t: nhwc(F.interpolate(nchw(t), scale_factor=2, mode="nearest"))  # noqa: E731
        if name == "conv_first":
            return self._head_ref()
        if name == "conv_before_upsample":
            return o["conv_after_body"]
        if name.startswith("upsample.up."):
            i = int(name.rsplit(".", 1)[1])
            if i == 0:
                return o["conv_before_upsample" if m.upsampler == "pixelshuffle" else "conv_after_body"]
            return nhwc(F.pixel_shuffle(nchw(o[f"upsample.up.{i - 2}"]), m.upsample.up[i - 1].upscale_factor))
        if name == "conv_up1":
            return up(o["conv_before_upsample"])
        if name == "conv_up2":
            return up(o["conv_up1"])
        if name == "conv_hr":
            return o["conv_up2"]
        if name == "conv_last":
            if m.upsampler == "pixelshuffle":
                n = len(m.upsample.up)
                return nhwc(F.pixel_shuffle(nchw(o[f"upsample.up.{n - 2}"]), m.upsample.up[n - 1].upscale_factor))
            return o["conv_hr"] if m.upsampler == "nearest+conv" else o["conv_after_body"]
        return None

    def _consumer(self, name, x, res):
        if name.endswith(STREAM_READERS):
            self._exact("input == latest residual stream", same32(x, self.stream32), name)
        if name.endswith(".block0.qkv"):
            self.stage_in = self.stream32
        if name.startswith("stage") and name.endswith(".conv"):
            self._exact("stage conv residual == stage input", same32(res, self.stage_in), name)
        elif name == "conv_after_body":
            self._exact("conv_after_body residual == conv_first output", same32(res, self.outs["conv_first"]), name)
        elif name == "conv_last" and res is not None:
            self._exact("conv_last residual == the normalised input", same32(res, self._head_ref()), name)
        if name != "conv_after_body" and name.startswith(TAIL):
            self._exact("head / tail glue (input of the conv)", same32(x, self._tail_in(name)), name)

    def check_output(self, y, H, W):
        """The forward's output: the last conv's output, through the tail glue, / img_range + mean, cropped."""
        m, o = self.model, self.outs
        if m.upsampler == "pixelshuffledirect":
            last = F.pixel_shuffle(nchw(o["upsample.up.0"]), m.upsample.up[1].upscale_factor)
        else:
            last = nchw(o["conv_last"])
        s = m.upscale
        full = last / m.img_range + m.mean.to(y.device)
        ref = full[:, :, :H * s, :W * s]
        self._exact("output == tail glue of the last conv", same32(y, ref), "tail")
        if self.mutate and W * s < full.shape[3]:  # the crop taken at the padded pitch
            self._mut(MUTATIONS[4], not same32(y, full.flatten(2)[..., :H * s * W * s].reshape(ref.shape)))

    # ---- glue -------------------------------------------------------------------------------------
    def _check_ln_residual(self, x, u, gamma, beta, eps=1e-5, res_scale=1.0, cab_y=None, cab_gate=None, out=None,
                           _name=None):
        blk_name, which = self.norm[id(gamma)]
        where = f"{blk_name}.{which}" if blk_name else which
        if blk_name:
            self._set_block(blk_name)
        Bn, L, Cn = u.shape
        o = self.outs
        want_u = {"norm1": o.get(f"{blk_name}.proj"), "norm2": o.get(f"{blk_name}.fc2"),
                  "norm_start": o.get("conv_first"), "norm_end": self.stream32}[which]
        ok = want_u is not None and same32(u, want_u)
        if x is not None:
            ok = ok and same32(x, self.stream32)
        if cab_y is not None:
            ok = ok and same32(cab_y, o[f"{blk_name}.cab2"]) and self.gate_out is not None and same32(cab_gate,
                                                                                                      self.gate_out)
        self._exact("ln_residual operands (its block's outputs and stream)", ok, where)
        f = torch.float64
        u64, g64, b64 = u.reshape(-1, Cn).double(), gamma.detach().double(), beta.detach().double()
        x64 = None if x is None else x.reshape(-1, Cn).double()
        rows = torch.arange(Bn * L, device=u.device) // L
        ones = torch.ones(Bn * L // O.L_LN + 1, Cn, dtype=f, device=u.device)  # ln_reference's gate rows: cy carries it

        def ref_bound(xx=x64, gate=cab_gate):
            cg = None if cab_y is None else cab_y.reshape(-1, Cn).double() * gate.double()[rows]
            one = None if cg is None else ones
            return (O.ln_reference(u64, g64, b64, eps, res_scale, xx, cg, one),
                    O.ln_bound(u64, g64, b64, eps, res_scale, xx, cg, one))

        ref, bound = ref_bound()
        got = out.reshape(-1, Cn)
        r = bound_ratio(got, ref, bound)
        self._gate("ln_residual (error / bound)", r, 1.0, r <= 1.0, where)
        if which == "norm1":
            pv = self.saved.get(self.prev, {})
            if self._mutation_here() and pv.get("res") is not None and pv["res"].shape == x.shape:
                self._control(MUTATIONS[1], bound_ratio, got, ref, ref_bound(xx=pv["res"].reshape(-1, Cn).double())[0],
                              bound, 1.0)
            if self._mutation_here() and cab_y is not None and pv.get("gate") is not None:
                self._control(MUTATIONS[3], bound_ratio, got, ref, ref_bound(gate=pv["gate"])[0], bound, 1.0)
            sv = self.saved.setdefault(self.block, {})
            sv["res"] = x.clone()
            sv["gate"] = None if cab_gate is None else cab_gate.clone()
        self.stream32 = out

    def _check_channel_gate(self, y, w1, b1, w2, b2, out=None, _name=None):
        att = self._blk().conv.cab[3].attention
        where = f"{self.block}:channel_gate"
        ok = all(a.data_ptr() == b.data_ptr() for a, b in ((w1, att[1].weight), (b1, att[1].bias), (w2, att[3].weight),
                                                           (b2, att[3].bias)))
        self._exact("channel gate: its block's CAB features and MLP", ok and same32(y, self.outs[f"{self.block}.cab2"]),
                    where)
        d64 = [y.double()] + [t.detach().double() for t in (w1, b1, w2, b2)]
        ref, bound = C.gate_reference(*d64), C.gate_bound(*d64)
        r = bound_ratio(out, ref, bound)
        i = int(((out.double() - ref).abs() / bound).argmax())
        self._gate("channel_gate (error / bound)", r, 1.0, r <= 1.0, where,
                   f"got {out.reshape(-1)[i].item():.6g} ref {ref.reshape(-1)[i].item():.6g}")
        self.gate_out = out

    def _check_avgpool(self, x, df, out=None, _name=None):
        where = f"{self.block}:avgpool"
        self._exact("input == latest residual stream", same32(x, self.stream32), where)
        Bn, H, W, Cn = x.shape
        v = x.cpu().view(Bn, H // df, df, W // df, df, Cn)
        s = torch.zeros(Bn, H // df, W // df, Cn)
        for dy in range(df):
            for dx in range(df):
                s = s + v[:, :, dy, :, dx]
        # on the CPU: torch divides a CUDA tensor by a Python number as a multiplication by its reciprocal, which is not
        # the kernel's IEEE division when df * df is not a power of two
        self._exact("avgpool", same32(out.cpu(), s / float(df * df)), where)

    def _check_demosaic(self, x, out=None, _name=None):
        self._exact("demosaic", same32(out, KF.demosaic_host(x.cpu()).to(x.device)), "head")

    # ---- attention --------------------------------------------------------------------------------
    def _check_bias_table(self, table, w1, b1, w2, out=None, _name=None):
        blk_name, role = self.transform[id(w1)]
        t = table.reshape(-1, 2).double()
        bound, ref = C.bias_table_bound(t, w1.detach().double(), b1.detach().double(), w2.detach().double())
        r = bound_ratio(out, ref, bound)
        self._gate("bias_table (error / bound)", r, 1.0, r <= 1.0, f"{blk_name}.{role}:bias_table")
        self.tables[out.data_ptr()] = (weakref.ref(out), table.clone(), blk_name, role)

    def _table(self, bias, role, gt, df, where):
        """The table an attention pass received: written by this block's transform for `role`, from the coordinates of
        the pass's own geometry (token window gt[2:4], anchor down factor df)."""
        e = self.tables.get(bias.data_ptr())
        ok = e is not None and e[0]() is bias and e[2:] == (self.block, role)
        self._exact("attention table from its own block's transform", ok, f"{where}.{role}")
        coords = O.coords_table([gt[2], gt[3]], df).reshape(-1, 2).to(bias.device)
        okc = e is not None and e[1].numel() == coords.numel() and torch.equal(e[1].reshape(-1, 2), coords)
        self._exact("bias_table coordinates == coords_table of the consuming pass", okc, f"{where}.{role}")

    def _attn(self, family, got, p, heads, sel, gate, where, v=None):
        """Gates one attention output with f32_cases.attn_ratio (the ulp statistic alone is reported); returns (reference,
        reference on |v|)."""
        v = p.v if v is None else v
        geo = dict(zip(("index", "mask"), self._geometry(p.gq, p.gk, p.use_mask)))
        ref = C.attn_ref(p, heads, v=v, sel=sel, **geo)
        absref = C.attn_ref(p, heads, v=v.abs(), sel=sel, **geo)
        nk = p.gk[2] * p.gk[3]  # keys per window
        r = C.attn_ratio(got, ref, absref, nk, gate)
        self._gate(f"{family} (error / bound)", r, 1.0, r <= 1.0, where)
        u = C.ulp_stats(got, ref)
        self._gate(f"{family} (ulp, reported)", u, gate, True, where)
        return ref, absref, nk

    def _check_window(self, qkv, B, grid, heads, logit_scale, bias, use_mask, out, _name=None):
        self._set_block(_name.rsplit(".", 1)[0])
        tr = self._blk().attn.window_attn.attn_transform
        where = self.block
        g = grid_t(grid)
        self._table(bias, "window", g, 1, where)
        self._exact("logit scales are the pass's own", logit_scale is tr.logit_scale, f"{where}.window")
        c = qkv.shape[2] // 3
        tok = qkv.double().reshape(B, g[0], g[1], 3 * c)
        p = C.Pass(g, g, tok[..., :c], tok[..., c:2 * c], tok[..., 2 * c:], False, False, logit_scale.detach(), bias,
                   use_mask)
        sel = self._windows(B * (g[0] // g[2]) * (g[1] // g[3])).to(qkv.device)
        got = C.windows(out.reshape(B, g[0], g[1], c), g, heads)[sel]
        ref, absref, nk = self._attn("window attention", got, p, heads, sel, GATE_ATTN, f"{where}.window")
        pv = self.saved.get(self.prev, {}).get("window")
        if self._mutation_here() and pv is not None and pv[0].shape == bias.shape:
            mut = C.attn_ref(p._replace(table=pv[0], scale=pv[1]), heads, sel=sel,
                             **dict(zip(("index", "mask"), self._geometry(g, g, use_mask))))
            self._control(MUTATIONS[2], lambda a, b, _: C.attn_ratio(a, b, absref, nk, GATE_ATTN), got, ref, mut, None,
                          1.0)
        if self.mutate and self._full_windows() and use_mask and g[0] // g[2] != g[1] // g[3]:
            gt = (g[1], g[0], g[3], g[2], g[5], g[4])  # the transposed window grid (square windows)
            index = self._geometry(g, g, use_mask)[0]
            mut = C.attn_ref(p, heads, index=index, mask=self._geometry(gt, gt, True)[1], sel=sel)
            self._control(MUTATIONS[5], lambda a, b, _: C.attn_ratio(a, b, absref, nk, GATE_ATTN), got, ref, mut, None,
                          1.0)
        self.saved.setdefault(self.block, {})["window"] = (bias.clone(), logit_scale.detach().clone())

    def _check_stripe(self, qkv, anchor, B, tok_grid, anc_grid, heads, scale1, bias1, scale2, bias2, use_mask, out,
                      _name=None):
        self._set_block(_name.rsplit(".", 1)[0])
        sa = self._blk().attn.stripe_attn
        where = self.block
        tg, ag = grid_t(tok_grid), grid_t(anc_grid)
        df = tg[2] // ag[2]
        self._table(bias1, "stripe1", tg, df, where)
        self._table(bias2, "stripe2", tg, df, where)
        self._exact("logit scales are the pass's own",
                    scale1 is sa.attn_transform1.logit_scale and scale2 is sa.attn_transform2.logit_scale,
                    f"{where}.stripe")
        # X1 lives in the wrapper's own workspace: issue the same call again with one this checker owns
        c = qkv.shape[2] // 3
        d = c // heads
        lib = capi.lib()
        nbytes = lib.grl_stripe_attn_workspace(B, tok_grid, anc_grid, heads, d)
        ws = torch.full((nbytes // 4,), float("nan"), device=qkv.device)
        out2 = torch.full((B, qkv.shape[1], c), float("nan"), device=qkv.device)
        capi.check(lib.grl_stripe_attn_f32(capi.ptr(qkv), qkv.stride(1), capi.ptr(anchor), c, capi.ptr(out2), c, B,
                                           tok_grid, anc_grid, heads, d, capi.ptr(scale1), capi.ptr(bias1),
                                           capi.ptr(scale2), capi.ptr(bias2), int(use_mask), capi.ptr(ws), nbytes,
                                           capi.stream()))
        torch.cuda.synchronize()
        self._exact("stripe output == a second call's", same32(out, out2), f"{where}.stripe")
        self._exact("every output element written", bool(ws.isfinite().all()), f"{where}.stripe X1")
        Na = ag[2] * ag[3]
        x1 = ws.view(-1, heads, Na, d)
        tok = qkv.double().reshape(B, tg[0], tg[1], 3 * c)
        anc = anchor.double()
        p1 = C.Pass(ag, tg, anc, tok[..., c:2 * c], tok[..., 2 * c:], False, True, scale1.detach(), bias1, use_mask)
        p2 = C.Pass(tg, ag, tok[..., :c], anc, x1.double(), True, False, scale2.detach(), bias2, use_mask)
        sel = self._windows(x1.shape[0]).to(qkv.device)
        r1, _, _ = self._attn("stripe pass 1", x1[sel], p1, heads, sel, GATE_ATTN, f"{where}.stripe1")
        got = C.windows(out.reshape(B, tg[0], tg[1], c), tg, heads)[sel]
        self._attn("stripe pass 2 on its own X1", got, p2, heads, sel, GATE_ATTN, f"{where}.stripe2")
        chain = x1.double().clone()
        chain[sel] = r1
        self._attn("stripe chain", got, p2, heads, sel, GATE_CHAIN, f"{where}.stripe2", v=chain)

def replay(model, x, rggb=False, mutate=True, seed=0, label=""):
    """One checked fp32 forward; returns (output, Replay32)."""
    rp = Replay32(model, x, rggb, mutate, seed)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    y = model._forward_f32(x.float().contiguous(), rggb, rp)
    torch.cuda.synchronize()
    H, W = x.shape[2:]
    rp.check_output(y, 2 * H if rggb else H, 2 * W if rggb else W)
    rp.report(label, time.perf_counter() - t0, torch.cuda.max_memory_allocated())
    return y, rp


def _assert_clean(rp):
    assert not rp.failures, f"{len(rp.failures)} failed checks, first: {rp.failures[:5]}"


# ---------------------------------------------------------------------------------------------------------- CPU


def test_every_f32_wrapper_has_a_replay_checker(pkg):
    """GRL._forward_f32 of every architecture of archs.architectures (and once from packed Bayer planes), on a meta
    input: every wrapper it launches through must have a checker in Replay32."""
    from grl_image_restoration_b200 import functional as K

    known = checkers(K)
    seen = {}
    for name, model, shape in archs.architectures(pkg, "fp32"):
        rec = Recorder()
        model._forward_f32(torch.empty(shape, device="meta"), False, rec)
        if model.in_channels == 3 and K.demosaic not in seen:
            model._forward_f32(torch.empty(shape[0], 4, shape[2] // 2, shape[3] // 2, device="meta"), True, rec)
        for fn, first in rec.fns.items():
            seen.setdefault(fn, f"{name}: {first}")
    missing = {getattr(fn, "__qualname__", repr(fn)): w for fn, w in seen.items() if fn not in known}
    print(f"{len(seen)} wrappers launched: " + ", ".join(sorted(getattr(f, "__qualname__", repr(f)) for f in seen)))
    assert not missing, f"wrappers without a Replay32 checker: {missing}"
    assert set(seen) == set(known), f"checkers no forward uses: {set(known) - set(seen)}"


# ---------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def lib(pkg, device):
    if capi.lib().grl_device_ok() != 1:
        pytest.skip("the library is built for sm_90a")
    return capi.lib()


MICRO = ["micro_cab_x2", "micro_pad_dn", "micro_groups", "micro_odd_d", "micro_gray"]
CASES = (["native:cfg2-fp32", "native:cfg3-fp32", "native:cfg4-fp32", "native:cfg5-fp32", "zoo:bsr_b2_40x56-fp32",
          "zoo:defocus_dual_b2_48x80-fp32", "zoo:dn_small_c1_b2_100x72-fp32", "dm:b2_40x56-fp32"] +
         [f"micro:{n}-fp32" for n in MICRO] + ["micro:micro_groups@24x32-fp32"] + CC.f32_names())


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_replay_f32(pkg, oracle, cases, golden_loader, lib, device, name):
    model, x, rggb = replay_case(pkg, oracle, cases, golden_loader, device, name)
    y, rp = replay(model, x, rggb, label=name)
    assert torch.equal(y, model(x)), "the replayed forward differs from model(x)"
    _assert_clean(rp)
    if sum(len(layer.blocks) for layer in model.layers) > 1:
        applied = {m: rp.mutations[m][1] for m in MUTATIONS[:2]}
        assert all(applied.values()), applied
    if name.startswith("command:"):
        case = CC.BY_NAME[name.rsplit("-", 1)[0]]
        for m, applies in zip(MUTATIONS[4:], CC.expected_mutations(model, case, rggb)):
            assert (rp.mutations[m][1] > 0) == applies, (m, applies, rp.mutations[m])
        del rp
        torch.cuda.empty_cache()
        ok, msg = CC.end_to_end(pkg, oracle, case, device, "fp32", y, x, rggb)
        print(f"  end to end: {msg}")
        assert ok, msg


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["micro_groups", "small"])
def test_cache_coherence_replayed_f32(pkg, oracle, cases, lib, device, which):
    """Forward at A, at B (another stripe geometry), at A again, then at A after in-place edits of one logit_scale,
    one cpb_mlp weight and one conv weight: every forward passes the replay checks against the parameters as they are
    then (a stale packed conv weight fails), and equals bit for bit the forward of a fresh deep copy of the model."""
    if which == "small":
        cfg = pkg.configs.grl_config("small", "sr", 2, 64)
        sizes = {"A": (64, 64), "B": (64, 128)}
    else:
        cfg = cases[which]["cfg"]
        sizes = {"A": (16, 16), "B": (24, 32)}
    model = pkg.GRL(**cfg)
    model.load_state_dict(oracle.synth_state_dict(cfg, seed=0, style="routed"), strict=False)
    model = model.to(device).eval()
    assert model.set_precision("fp32") == "fp32"
    xs = {k: oracle.synth_input((1, cfg["in_channels"], *hw), seed=7 + i).to(device) for i, (k, hw) in enumerate(sizes.items())}
    blk = model.layers[0].blocks[-1]

    def edit():
        with torch.no_grad():
            blk.attn.window_attn.attn_transform.logit_scale.add_(0.25)
            blk.attn.stripe_attn.attn_transform1.cpb_mlp[0].weight.mul_(1.1)
            model.layers[0].conv.weight.mul_(0.9)

    for step, (res, action) in enumerate([("A", None), ("B", None), ("A", None), ("A", edit)]):
        if action:
            action()
        y, rp = replay(model, xs[res], mutate=False, seed=step, label=f"{which} step {step} at {sizes[res]}")
        _assert_clean(rp)
        fresh = copy.deepcopy(model)
        assert torch.equal(y, fresh(xs[res])), f"step {step}: differs from a fresh copy"
