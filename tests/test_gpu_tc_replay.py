"""Real tensor-core forwards checked launch by launch against float64, and the caches that outlive a forward.

`Replay` is a tc.Device launcher: it runs each launch of tc.forward, synchronises and checks that launch on the operands
the forward really handed it before the next one runs.  So every kernel is gated on what the previous kernels wrote
(correlated q / k, trained-like bias tables, real residual streams), not only on the seeded operands of the launch-path
tests, with the gates of those tests:
  GEMM (every `listed` launch): grl_oracle.gemm_launch_reference through gemm_cases.evaluate (fp32, 16-bit,
    PixelShuffle and NCHW-tail outputs and the 16-bit == RNE(own fp32) identity; no high-mean row split);
  attention: grl_oracle.attn_launch_reference of the launch's own q / k / v and copy 0 of its bias table, through
    attn_cases.compare and GATE_ULP, stripe pass 2 also against the chained emulation (GATE_CHAIN).  At most 16
    windows per launch (the first, the last (masked and rolled) and 14 seeded others); every window in the first and
    last block of each stage;
  glue: pack_rows, head_pack / head_pack_rggb and avgpool16 bit for bit; slot scales exactly as
    test_slot_scale_layout, from the block's parameters as they are then; bias_table_log2 within test_bias_table4's
    bound of float64 16 sigmoid(MLP(coords)) log2 e, copies 1-3 exact shifts, the pad zero; channel_gate within
    test_tc_channel_gate's bound; K.ln_residual within grl_oracle.ln_bound;
  consumers: the slot scales a QKV GEMM receives and the table an attention launch receives are checked whether they
    were computed in this forward or come from the block's constant cache; the 16-bit operand a GEMM reads as the
    residual stream's copy (qkv, cab1, fc1, stage conv, conv_after_body) is bit for bit RNE16 of the latest fp32 stream;
  integrity: every buffer a launch writes is check-summed right after it; a later launch that reads it must see the
    same sum (a stray write into a live neighbouring allocation), and a wrapper without a checker fails.
Mutation controls, computed on the reference side (never an edited kernel), at the first block of every stage after the
first block of the network and at the last block of every stage: the QKV GEMM fed the previous block's 16-bit input, the
proj LayerNorm epilogue with the previous block's residual, window attention with the previous block's bias table and
slot scales.  Two more show only at the sizes the test commands run (`command:` cases, tests/command_cases.py): the
NCHW tail's crop taken at the padded pitch (where Wc < Wp) and, at the first and last block of each stage, shifted
window attention with the shift mask of the transposed window grid (non-square grids).  Each must fail its gate wherever
it applies.  A `command:` case's output is also compared end to end with oracle.grl_forward on the device
(command_cases.end_to_end).
"""
import copy
import inspect
import math
import time
import types
import weakref

import pytest
import torch

import archs
import attn_cases as A
import command_cases as CC
import gemm_cases as G
import grl_oracle as O
from _pkgload import load_package
from replay_base import Recorder, ReplayBase, _base, replay_case
from support import bound_ratio, grid_t, ulp

load_package()
from grl_image_restoration_b200 import functional as KF, tc as TC  # noqa: E402

U = 2.0 ** -24
STREAM_READERS = (".qkv", ".cab1", ".fc1", ".conv", "conv_after_body")  # GEMMs whose x16 is the residual stream's copy
MUTATIONS = ("qkv fed the previous block's input", "proj residual of the previous block",
             "window attention with the previous block's constants", "NCHW tail cropped at the padded pitch",
             "window attention on the transposed window grid's geometry")


def checkers(tc, K):
    """Wrapper -> Replay method that checks it: every kernel tc.forward launches must have one."""
    return {tc.gemm: "gemm", tc.pack_rows: "pack_rows", tc.head_pack: "head_pack", tc.head_pack_rggb: "head_pack_rggb",
            tc.slot_scale: "slot_scale", tc.bias_table_log2: "bias_table", tc.avgpool16: "avgpool16",
            tc.attention: "attention", tc.channel_gate: "channel_gate", K.ln_residual: "ln_residual"}


def same16(a, b):
    return bool((a.contiguous().view(torch.int16) == b.contiguous().view(torch.int16)).all())


def slot_scale_ref(blk):
    """test_slot_scale_layout's reference from the block's current logit scales."""
    wa, sa = blk.attn.window_attn, blk.attn.stripe_attn
    sc = lambda ls: torch.exp(ls.detach().double().reshape(-1).clamp(max=O.LN100_F32)) / math.log(2.0)  # noqa: E731
    hw, hs = wa.num_heads, sa.num_heads
    d = wa.attn_transform.logit_scale.device
    z = lambda n, v: torch.full((n,), v, dtype=torch.float64, device=d)  # noqa: E731
    return torch.cat([sc(wa.attn_transform.logit_scale), z(hw, 1.0), z(hw, 0.0), sc(sa.attn_transform2.logit_scale),
                      sc(sa.attn_transform1.logit_scale), z(hs, 0.0)])


def slot_scale_ok(got, ref):
    got = got.double()
    exact = ref.eq(0) | ref.eq(1)
    rel = ((got - ref).abs() / ref)[~exact]
    return bool(torch.equal(got[exact], ref[exact])) and (rel.numel() == 0 or float(rel.max()) <= 6 * U)


def bias_ratio(transform, coords, out):
    """test_bias_table4's check of a (heads, 4, rows_pad) table against `transform`'s cpb_mlp on coords (rows, 2):
    copy 0's worst error / bound, or inf when copies 1-3 are not exact shifts or the pad is not zero."""
    from grl_image_restoration_b200 import tc

    t = coords.reshape(-1, 2).double().to(out.device)
    rows = t.shape[0]
    w1, b1 = transform.cpb_mlp[0].weight.detach().double(), transform.cpb_mlp[0].bias.detach().double()
    w2 = transform.cpb_mlp[2].weight.detach().double()
    h = torch.relu(t @ w1.T + b1)
    sg = torch.sigmoid(h @ w2.T)
    ref = (16 * sg * tc.LOG2E).T
    dh = 2 * U * (t.abs() @ w1.abs().T + b1.abs())
    da = w1.shape[0] * U * (h @ w2.abs().T) + dh @ w2.abs().T
    bound = 2 * (16 * tc.LOG2E * sg * (1 - sg) * da + 6 * U * 16 * tc.LOG2E * sg).T
    if out.shape[2] != tc.bias_rows_pad(rows):
        return float("inf")
    mask = torch.zeros_like(out, dtype=torch.bool)
    for c in range(4):
        mask[:, c, c:c + rows] = True
        if c and not torch.equal(out[:, c, c:c + rows], out[:, 0, :rows]):
            return float("inf")
    if bool(out[~mask].any()):
        return float("inf")
    return float(((out[:, 0, :rows].double() - ref).abs() / bound).max())


class Replay(ReplayBase, TC.Device):
    """tc.Device that checks every launch (module docstring).  Results as replay_base.ReplayBase, plus `rescales` and
    `sat16`."""

    def __init__(self, model, mutate=True, seed=0):
        super().__init__(model, MUTATIONS, mutate, seed)
        self.tc, self.K = TC, KF
        self.fmt = TC.FMT[model.precision]
        self.dtype = TC.DTYPE[self.fmt]
        self.methods = checkers(TC, KF)
        self.pass1 = {}  # block name -> (window indices, emulated X1 of those windows)
        self.stream32 = None
        self.rescales, self.sat16 = 0, 0
        self.derived16 = []  # launches whose 16-bit-only output needed the accumulation term

    def _record_writes(self, tensors, where):
        super()._record_writes(tensors, where)
        for t in tensors:
            if _base(t).dtype == torch.float16:
                self.sat16 += int((t.float().abs() == 65504.0).sum())

    def _block_changed(self):
        self.pass1 = {}

    # ---- outputs of each wrapper ------------------------------------------------------------------
    def _outs_gemm(self, *a, **kw):
        return [kw[k] for k in ("out_bf16", "out_f32", "out_nchw") if kw.get(k) is not None]

    def _outs_pack_rows(self, x, cpad, fmt=0, out=None):
        return [out]

    def _outs_head_pack(self, x, hp, wp, mean, rng, cpad, fmt, out):
        return [t for t in out if t is not None]

    _outs_head_pack_rggb = _outs_head_pack

    def _outs_slot_scale(self, *a):
        return [a[-1]]

    def _outs_bias_table(self, tr, table, out):
        return [out]

    def _outs_avgpool16(self, x16, out, df):
        return [out]

    def _outs_attention(self, gq, gk, q, q_off, k, k_off, v, v_off, out, *a, **kw):
        return [out]

    def _outs_channel_gate(self, *a):
        return [a[-1]]

    def _outs_ln_residual(self, *a, out, **kw):
        return [out]

    # ---- GEMM -------------------------------------------------------------------------------------
    def _check_gemm(self, x16, w16, bias, _name, **kw):
        tc = self.tc
        a = inspect.signature(tc.gemm_problem).bind(x16, w16, bias, **kw)
        a.apply_defaults()
        a = a.arguments
        if ".block" in _name:
            self._set_block(_name.rsplit(".", 1)[0])
        conv = a["taps"] == 9
        x = x16 if conv else x16.reshape(-1, x16.shape[-1])[:a["M"]]
        ops = dict(taps=a["taps"], epi=a["epi"], act=a["act"], slope=a["slope"])
        if a["epi"] == tc.EPI_QKV:
            ops["slot_scale"] = a["slot_scale"]
            if _name.endswith(".qkv"):  # the constants this launch receives, cached or not
                ok = slot_scale_ok(a["slot_scale"], slot_scale_ref(self._blk()))
                self._gate("slot scales (QKV consumer)", 0.0 if ok else 1.0, "exact", ok, _name)
        if a["epi"] == tc.EPI_LN:
            ops.update(gamma=a["gamma"], beta=a["beta"], eps=a["eps"], res_scale=a["res_scale"], L=a["L"])
            if a["cab_y"] is not None:
                ops.update(cab_y=a["cab_y"], cab_gate=a["cab_gate"])
        if a["res_f32"] is not None:
            ops["res"], ops["n_res"] = a["res_f32"], a["res_f32"].shape[-1]
        if a["out_f32"] is not None:
            ops["n_res"] = a["n_real"]
        if a["out_nchw"] is not None:
            o = a["out_nchw"]
            ops.update(nchw_r=a["nchw_r"], crop=tuple(o.shape[2:]), post_scale=a["post_scale"],
                       post_shift=a["post_shift"], n_res=a["n_real"])
        if a["ps_r"]:
            ops["ps_r"] = a["ps_r"]
        got = {k: a[k] for k in ("out_bf16", "out_f32", "out_nchw") if a[k] is not None}
        run = types.SimpleNamespace(kw=a)

        def verdict(xx=x, extra=None, acc_err=None):
            o = dict(ops, **(extra or {}))
            ref = O.gemm_launch_reference(xx, w16, bias, **o)
            return G.evaluate(tc, run, got, ref, self.fmt, high_mean_rows=(), acc_err=acc_err)

        res = verdict()
        if a["epi"] == tc.EPI_BIAS_ACT and "16-bit" in res and not res["16-bit"][1]:
            # the seeded gate does not grow with sum |x| |w|: where a real operand cancels, add gamma_K of that sum
            absdot = O.gemm_launch_reference(x.abs(), w16.abs(), torch.zeros_like(bias), taps=a["taps"])["y"]
            acc = O.gamma(w16.shape[1]) * absdot
            res["16-bit"] = verdict(acc_err=acc)["16-bit"]
            self.derived16.append(_name)
            self._report16(_name, O.gemm_launch_reference(x, w16, bias, **ops)["y"], a, absdot, acc, res["16-bit"][1])
        for what, (s, ok) in res.items():
            stat = s[1] if isinstance(s, tuple) else s
            self._gate(f"gemm {what}", stat, "evaluate", ok, _name, str(s))
        # the residual stream's operand copy
        if _name.endswith(STREAM_READERS) and self.stream32 is not None:
            s32 = self.stream32.reshape(-1, self.stream32.shape[-1])
            ok = same16(x16.reshape(s32.shape[0], -1)[:, :s32.shape[1]], self._to16(s32))
            self._gate("x16 == RNE16(stream)", 0.0 if ok else 1.0, "bitwise", ok, _name)
        # mutation controls
        if self._mutation_here() and _name.endswith(".qkv") and self.prev in self.saved:
            px = self.saved[self.prev].get("x16")
            if px is not None and px.shape == x.shape:
                self._mut(MUTATIONS[0], not all(ok for _, ok in verdict(xx=px).values()))
        if self._mutation_here() and _name.endswith(".proj") and self.prev in self.saved:
            pr = self.saved[self.prev].get("res")
            if pr is not None and pr.shape == a["res_f32"].shape:
                self._mut(MUTATIONS[1], not all(ok for _, ok in verdict(extra={"res": pr}).values()))
        if ".block" in _name:
            sv = self.saved.setdefault(self.block, {})
            if _name.endswith(".qkv"):
                sv["x16"], sv["scales"] = x.clone(), a["slot_scale"].clone()
            elif _name.endswith(".proj"):
                sv["res"] = a["res_f32"].clone()
        if a["out_nchw"] is not None and self.mutate:
            o, r = a["out_nchw"], a["nchw_r"]
            full = (x.shape[1] * r, x.shape[2] * r)
            if o.shape[3] < full[1]:  # a tail that crops Hc x Wc out of the padded image at its pitch Wp
                ref = O.gemm_launch_reference(x, w16, bias, **dict(ops, crop=full))["nchw"]
                mut = ref.flatten(2)[..., :o.shape[2] * o.shape[3]].reshape(o.shape)
                self._mut(MUTATIONS[3], G.stats32(o, mut) > G.GATE32)
        if a["out_f32"] is not None and (a["epi"] == tc.EPI_LN or _name.endswith(".conv")):
            self.stream32 = a["out_f32"]

    def _report16(self, name, y, a, absdot, acc, ok):
        """Prints the 16-bit-only output's elements outside the seeded gate: the worst, with its float64 value, sum |x||w|
        and gamma_K of that sum."""
        n = a["n_real"] or a["n_store"]
        yr, g = y[:, :n], a["out_bf16"].reshape(y.shape[0], -1)[:, :n].double()
        delta = G.GATE32 * ulp(G.row_scale(yr), torch.float32) + (O.GELU_AS_ABS_ERR if a["act"] == 1 else 0.0)
        lo, hi = (yr - delta).to(self.dtype).double(), (yr + delta).to(self.dtype).double()
        out = torch.maximum(lo - g, g - hi).clamp_min(0.0)
        r, c = divmod(int(out.argmax()), n)
        print(f"  {name}: {int((out > 0).sum())} 16-bit elements outside the seeded gate; the worst (row {r}, column "
              f"{c}): got {float(g[r, c]):.6g}, allowed [{float(lo[r, c]):.6g}, {float(hi[r, c]):.6g}], float64 "
              f"{float(yr[r, c]):.6g}, sum |x||w| {float(absdot[r, c]):.6g}, gamma_K of it {float(acc[r, c]):.3g}; "
              f"within the derived gate: {ok}")

    # ---- glue -------------------------------------------------------------------------------------
    def _to16(self, x):
        return O.to16(x, self.fmt)

    def _check_pack_rows(self, x, cpad, fmt=0, out=None, _name=None):
        C = x.shape[-1]
        o = out.reshape(-1, cpad)
        ok = same16(o[:, :C], self._to16(x.reshape(-1, C))) and not bool(o[:, C:].float().any())
        self._gate("pack_rows", 0.0 if ok else 1.0, "bitwise", ok, f"{self.block}:pack_rows")

    def _check_head_pack_rggb(self, cfa4, hp, wp, mean, rng, cpad, fmt, out, _name=None):
        # the library's host demosaic (bit-exact against the kernel: test_gpu_demosaic.py), then head_pack's reference
        self._check_head_pack(self.K.demosaic_host(cfa4.cpu()).to(cfa4.device), hp, wp, mean, rng, cpad, fmt, out)

    def _check_head_pack(self, raw, hp, wp, mean, rng, cpad, fmt, out, _name=None):
        import torch.nn.functional as F

        y16, y32 = out
        B, Cin, H, W = raw.shape
        pad = (0, wp - W, 0, hp - H)
        xp = F.pad(raw, pad, "reflect") if (hp - H < H and wp - W < W) else F.pad(raw, pad, "constant", 0.0)
        m = list(mean)
        m = m * Cin if len(m) == 1 else (m + [0.0] * Cin)[:Cin]
        ref32 = ((xp - torch.tensor(m, device=raw.device).view(1, Cin, 1, 1)) * rng).permute(0, 2, 3, 1).contiguous()
        ok = same16(y16[..., :Cin], self._to16(ref32)) and not bool(y16[..., Cin:].float().any())
        if y32 is not None:
            ok = ok and torch.equal(y32, ref32)
        self._gate("head_pack", 0.0 if ok else 1.0, "bitwise", ok, "head")

    def _check_slot_scale(self, ls_w, ls_s1, ls_s2, hw, hs, out, _name=None):
        self._set_block(self.owner[id(ls_w)])
        ok = slot_scale_ok(out, slot_scale_ref(self._blk()))
        self._gate("slot_scale", 0.0 if ok else 1.0, "exact", ok, f"{self.block}:slot_scale")

    def _check_bias_table(self, tr, table, out, _name=None):
        self._set_block(self.owner[id(tr)])
        r = bias_ratio(tr, table, out)
        self._gate("bias_table_log2 (error / bound)", r, 1.0, r <= 1.0, f"{self.block}:bias_table")

    def _check_avgpool16(self, x16, out, df, _name=None):
        B, H, W, Cp = x16.shape
        v = x16.float().view(B, H // df, df, W // df, df, Cp)
        s = torch.zeros(B, H // df, W // df, Cp, device=x16.device)
        for dy in range(df):
            for dx in range(df):
                s = s + v[:, :, dy, :, dx]
        ref = self._to16(s * torch.tensor(1.0 / (df * df), dtype=torch.float32))
        ok = same16(out, ref)
        self._gate("avgpool16", 0.0 if ok else 1.0, "bitwise", ok, f"{self.block}:avgpool16")

    def _check_channel_gate(self, y16, ld, B, L, C, ca, gate, _name=None):
        att = self._blk().conv.cab[3].attention
        w1, b1 = att[1].weight.detach().reshape(att[1].weight.shape[0], -1), att[1].bias.detach()
        w2, b2 = att[3].weight.detach().reshape(att[3].weight.shape[0], -1), att[3].bias.detach()
        R = w1.shape[0]
        y = y16.reshape(B, L, ld)[..., :C].float()
        ref, m, h = O.channel_gate_reference(y, w1, b1, w2, b2)
        chunks = (L + 511) // 512
        dm = (512 + chunks) * U * y.double().abs().mean(1)
        dh = dm @ w1.double().abs().T + (C + 1) * U * (m.abs() @ w1.double().abs().T + b1.double().abs())
        ds = dh @ w2.double().abs().T + (R + 1) * U * (h.abs() @ w2.double().abs().T + b2.double().abs())
        bound = 2 * (ds / 4 + 4 * U * ref)
        r = float(((gate.double() - ref).abs() / bound).max())
        self._gate("channel_gate (error / bound)", r, 1.0, r <= 1.0, f"{self.block}:channel_gate")

    def _check_ln_residual(self, x, u, gamma, beta, eps=1e-5, res_scale=1.0, cab_y=None, cab_gate=None, out=None,
                           _name=None):
        C = u.shape[-1]
        u64 = u.reshape(-1, C).double()
        g64, b64 = gamma.detach().double(), beta.detach().double()
        x64 = None if x is None else x.reshape(-1, C).double()
        ref = O.ln_reference(u64, g64, b64, eps, res_scale, x64, None, None)
        bound = O.ln_bound(u64, g64, b64, eps, res_scale, x64, None, None)
        r = bound_ratio(out.reshape(-1, C), ref, bound)
        self._gate("ln_residual (error / bound)", r, 1.0, r <= 1.0, "norm_start" if self.block is None else "norm_end")
        self.stream32 = out

    # ---- attention --------------------------------------------------------------------------------
    def _check_attention(self, gq, gk, q, q_off, k, k_off, v, v_off, out, o_off, B, heads, bias, use_mask,
                         v_dense=False, o_dense=False, tag="attn", ones_col=False, _name=None):
        blk = self._blk()
        wa, sa = blk.attn.window_attn, blk.attn.stripe_attn
        role = "window" if tag == "window_attn" else "stripe2" if v_dense else "stripe1"
        tr = {"window": wa.attn_transform, "stripe1": sa.attn_transform1, "stripe2": sa.attn_transform2}[role]
        d = blk.dim // 2 // heads
        where = f"{self.block}.{role}"
        # the table it received (computed now or cached): against this block's cpb_mlp at this resolution
        tg = gq if gq.wh >= gk.wh else gk
        df = tg.wh // min(gq.wh, gk.wh)
        coords = O.coords_table([tg.wh, tg.ww], df)
        r = bias_ratio(tr, torch.as_tensor(coords), bias)
        self._gate("attention table (error / bound)", r, 1.0, r <= 1.0, where)
        buf = {"q": q, "k": k, "v": v, "o": out, "x1": v if v_dense else out}
        spec = lambda name, off, dense: ("x1", 0) if dense else (name, off)  # noqa: E731
        qq = A.operand(buf, ("q", q_off), gq, heads, B)
        kk = A.operand(buf, ("k", k_off), gk, heads, B)
        vv = A.operand(buf, spec("v", v_off, v_dense), gk, heads, B)
        got = A.operand(buf, spec("o", o_off, o_dense), gq, heads, B)
        idx = self._windows(qq.shape[0]).to(q.device)
        index, mask = self._geometry(grid_t(gq), grid_t(gk), use_mask)
        index = index.to(q.device)
        msel = None if mask is None else mask.to(q.device)[idx % mask.shape[0]]
        table = bias[:, 0, :(gq.wh + gk.wh - 1) * (gq.ww + gk.ww - 1)]

        def emulate(qs, vs=None, tab=table):
            return O.attn_launch_reference(qs, kk[idx], vv[idx] if vs is None else vs, tab, index, msel, self.dtype)

        exact, emul, info = emulate(qq[idx])
        self.rescales += info["rescales"]
        s = A.compare(got[idx], emul, d, self.dtype)
        self._gate(f"attention {role} (ulp)", s[0], A.GATE_ULP, s[0] <= A.GATE_ULP, where, f"mismatch {s[1]:.4f}")
        if role == "stripe1":
            self.pass1[self.block] = (idx, emul.to(self.dtype))
        if role == "stripe2" and self.pass1.get(self.block) is not None and torch.equal(self.pass1[self.block][0], idx):
            _, em_c, _ = emulate(qq[idx], vs=self.pass1[self.block][1])
            sc = A.compare(got[idx], em_c, d, self.dtype)
            self._gate("attention stripe2 chain (ulp)", sc[0], A.GATE_CHAIN, sc[0] <= A.GATE_CHAIN, where)
        if role == "window" and self._mutation_here() and self.prev in self.saved:
            pv = self.saved[self.prev]
            pt, pscale = pv.get("table_w"), pv.get("scales")
            cur = self.saved[self.block]["scales"]
            if pt is not None and pt.shape == table.shape and not (torch.equal(pt, table) and torch.equal(pscale, cur)):
                hw = heads
                f = (pscale[:hw].double() / cur[:hw].double()).view(1, hw, 1, 1)
                qm = (qq[idx].double() * f).to(self.dtype)
                _, em_m, _ = emulate(qm, tab=pt)
                # it applies where it moves the emulated output by more than twice the gate: under "init" weights the
                # blocks' constants can be that close (bf16, dual-pixel defocus model)
                if A.compare(em_m, emul, d, self.dtype)[0] > 2 * A.GATE_ULP:
                    self._mut(MUTATIONS[2], A.compare(got[idx], em_m, d, self.dtype)[0] > A.GATE_ULP)
                else:
                    self._below(MUTATIONS[2])
        if role == "window" and self.mutate and self._full_windows() and use_mask and \
                gq.H // gq.wh != gq.W // gq.ww:
            gt = (gq.W, gq.H, gq.ww, gq.wh, gq.sw, gq.sh)  # the transposed window grid (square windows)
            mt = self._geometry(gt, gt, True)[1].to(q.device)
            _, em_t, _ = O.attn_launch_reference(qq[idx], kk[idx], vv[idx], table, index, mt[idx % mt.shape[0]],
                                                 self.dtype)
            if A.compare(em_t, emul, d, self.dtype)[0] > 2 * A.GATE_ULP:
                self._mut(MUTATIONS[4], A.compare(got[idx], em_t, d, self.dtype)[0] > A.GATE_ULP)
            else:
                self._below(MUTATIONS[4])
        if role == "window":
            self.saved.setdefault(self.block, {})["table_w"] = table.clone()

    def report(self, label, seconds, peak):
        super().report(label, seconds, peak, f", warp rescales {self.rescales}, fp16 operands at +-65504: {self.sat16}"
                       f", 16-bit outputs gated with the accumulation term: {self.derived16}")


def replay(tc, model, x, rggb=False, mutate=True, seed=0, label=""):
    """One checked forward; returns (output, Replay)."""
    rp = Replay(model, mutate, seed)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    y = tc.forward(model, x.float().contiguous(), rggb, rp)
    torch.cuda.synchronize()
    rp.report(label, time.perf_counter() - t0, torch.cuda.max_memory_allocated())
    return y, rp


# ---------------------------------------------------------------------------------------------------------- CPU


def test_every_forward_wrapper_has_a_replay_checker(pkg):
    """tc.forward of every architecture of archs.architectures (and once with the packed-Bayer head), on a meta
    input: every wrapper it launches through must have a checker in Replay."""
    from grl_image_restoration_b200 import functional as K, tc

    known = checkers(tc, K)
    seen = {}
    for name, model, shape in archs.architectures(pkg, "fp16"):
        rec = Recorder()
        tc.forward(model, torch.empty(shape, device="meta"), False, rec)
        if model.in_channels == 3 and tc.head_pack_rggb not in seen:  # the head of input_format "rggb"
            tc.forward(model, torch.empty(shape[0], 4, shape[2] // 2, shape[3] // 2, device="meta"), True, rec)
        for fn, first in rec.fns.items():
            seen.setdefault(fn, f"{name}: {first}")
    missing = {getattr(fn, "__qualname__", repr(fn)): w for fn, w in seen.items() if fn not in known}
    print(f"{len(seen)} wrappers launched: " + ", ".join(sorted(getattr(f, "__qualname__", repr(f)) for f in seen)))
    assert not missing, f"wrappers without a Replay checker: {missing}"
    assert tc.head_pack_rggb in seen and tc.channel_gate in seen and tc.avgpool16 in seen


# ---------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def tc(pkg, device):
    from grl_image_restoration_b200 import capi, tc as T

    if capi.lib().grl_device_ok() != 1:
        pytest.skip("wgmma path needs sm_90")
    return T


MICRO = ["micro_cab_x2", "micro_pad_dn", "micro_groups", "micro_odd_d", "micro_gray"]
CASES = (["native:cfg2-fp16", "native:cfg3-fp16", "native:cfg4-fp16", "native:cfg4-bf16", "native:cfg5-fp16",
          "zoo:bsr_b2_40x56-fp16", "zoo:defocus_dual_b2_48x80-fp16", "zoo:defocus_dual_b2_48x80-bf16",
          "zoo:dn_small_c1_b2_100x72-fp16", "dm:b2_40x56-fp16"] +
         [f"micro:{n}-{p}" for n in MICRO for p in ("fp16", "bf16")] + CC.tc_names())


def _assert_clean(rp):
    assert not rp.failures, f"{len(rp.failures)} failed checks, first: {rp.failures[:5]}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_replay(pkg, oracle, cases, golden_loader, tc, device, name):
    model, x, rggb = replay_case(pkg, oracle, cases, golden_loader, device, name)
    model.use_cuda_graph = False
    y, rp = replay(tc, model, x, rggb, label=name)  # first: the attention constants are computed under the replay
    assert torch.equal(y, model(x).float()), "the replayed forward differs from model(x)"
    _assert_clean(rp)
    nblocks = sum(len(layer.blocks) for layer in model.layers)
    if nblocks > 1:
        assert all(n > 0 for n, m in ((rp.mutations[m][1], m) for m in MUTATIONS[:2])), rp.mutations
    if name.startswith("command:"):
        case = CC.BY_NAME[name.rsplit("-", 1)[0]]
        for m, applies in zip(MUTATIONS[3:], CC.expected_mutations(model, case, rggb)):
            assert (rp.mutations[m][1] > 0) == applies, (m, applies, rp.mutations[m])
        del rp
        torch.cuda.empty_cache()
        ok, msg = CC.end_to_end(pkg, oracle, case, device, model.precision, y, x, rggb)
        print(f"  end to end: {msg}")
        assert ok, msg


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["micro_groups", "small"])
def test_cache_coherence_replayed(pkg, oracle, cases, tc, device, which):
    """Forward at A, at B (another stripe geometry), at A again, then at A after in-place edits of one logit_scale,
    one cpb_mlp weight and one conv weight: every forward passes the replay checks against the parameters as they are
    then, and equals bit for bit the forward of a fresh deep copy of the model."""
    if which == "small":
        cfg = pkg.configs.grl_config("small", "sr", 2, 64)
        sizes = {"A": (64, 64), "B": (64, 128)}
    else:
        cfg = cases[which]["cfg"]
        sizes = {"A": (16, 16), "B": (24, 32)}
    model = pkg.GRL(**cfg)
    model.load_state_dict(oracle.synth_state_dict(cfg, seed=0, style="routed"), strict=False)
    model = model.to(device).eval()
    model.use_cuda_graph = False
    model.set_precision("fp16")
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
        y, rp = replay(tc, model, xs[res], mutate=False, seed=step, label=f"{which} step {step} at {sizes[res]}")
        _assert_clean(rp)
        fresh = copy.deepcopy(model)
        assert torch.equal(y, fresh(xs[res])), f"step {step}: differs from a fresh copy"


@pytest.mark.gpu
def test_cuda_graph_follows_precision_and_weights(pkg, oracle, cases, tc, device):
    """use_cuda_graph: capture fp16, switch to bf16 and forward; before anything can replay the fp16 graph, its entry is
    either gone or still holds every plan it reads.  Then graphed forwards equal eager ones bit for bit in fp16, in bf16
    and after an in-place edit."""
    cfg = cases["micro_cab_x2"]["cfg"]
    model = pkg.GRL(**cfg)
    model.load_state_dict(oracle.synth_state_dict(cfg, seed=0, style="routed"), strict=False)
    model = model.to(device).eval()
    x = oracle.synth_input((2, 3, 32, 32), seed=1234).to(device)

    def graphed():
        model.use_cuda_graph = True
        return model(x)

    def eager():
        model.use_cuda_graph = False
        return model(x)

    model.set_precision("fp16")
    graphed()
    key16 = next(k for k in model._graphs if k[2] == "fp16")
    refs = [weakref.ref(p) for p in model._graph_plans()]
    model.set_precision("bf16")
    graphed()
    ent = model._graphs.get(key16)
    alive = sum(r() is not None for r in refs)
    print(f"\nafter the bf16 forward: fp16 entry {'kept' if ent is not None else 'dropped'}, {alive} / {len(refs)} of "
          f"its plans alive")
    assert ent is None or alive == len(refs), "a kept fp16 graph reads freed plans"
    for precision in ("fp16", "bf16", "fp16"):
        model.set_precision(precision)
        assert torch.equal(graphed(), eager()), precision
    with torch.no_grad():
        model.layers[0].blocks[1].attn.proj.weight.mul_(1.05)
        model.conv_first.bias.add_(0.01)
    g = graphed()
    assert torch.equal(g, eager()), "graph replayed the weights from before the edit"
    model.reset_cuda_graphs()  # a captured graph cannot be deep-copied
    fresh = copy.deepcopy(model)
    fresh.use_cuda_graph = False
    assert torch.equal(g, fresh(x))
