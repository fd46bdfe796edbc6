"""The launch-path cases of the tensor-core GEMM / implicit-GEMM conv kernel (csrc/gemm_tc.cu) and the machinery that
instantiates, gates and checks them, shared by test_gpu_tc_gemm.py (one small instance per path), test_gpu_tc_scale.py
(the benchmark's sizes) and test_gpu_tc_replay.py (real forwards).  A case's seed is its index in ALL_CASES.  The gates
are described in test_gpu_tc_gemm.py."""
import math
from typing import NamedTuple

import torch

import archs
import grl_oracle as O
from support import ulp

GATE32 = 255.0         # 2 x the worst case, 127.4 ulp (fp16 operands, base stage conv: K = 9 x 192)
GATE_LN_SHIFT = 214.0  # 2 x the worst high-mean row, 107.0 ulp (bf16 operands, GRL-Tiny proj); naive moments: >= 819
B, L_CASE, HT, WT = 2, 100, 13, 21
HIGH_MEAN_ROWS = (5, 133)
ZERO_QKV_ROW = 3
GUARD = 3  # guard rows before and after every output buffer
ROW_CHUNK = 1 << 16  # operands with more rows are drawn in chunks of this many rows


def path(launch):
    """Launch-path signature: (BN, epi, conv, epi_mode, n_tiles > 1, partial last N tile, min(k chunks, 5), act,
    residual, 16-bit out, fp32 out, ps_r, nchw_r (0 = no NCHW tail), residual on the NCHW tail, CAB, 16-bit pitch >
    n_store)."""
    from grl_image_restoration_b200 import tc

    a, q = launch.args, tc.gemm_path(launch)
    nchw, o16 = a["out_nchw"] is not None, a["out_bf16"]
    return (q.bn, a["epi"], bool(q.conv), q.epi_mode, q.n_tiles > 1, q.n_tiles * q.bn > a["npad"], min(q.nk_total, 5),
            a["act"], a["res_f32"] is not None, o16 is not None, a["out_f32"] is not None, a["ps_r"],
            a["nchw_r"] if nchw else 0, nchw and a["res_f32"] is not None, a["cab_y"] is not None,
            o16 is not None and o16.shape[-1] > a["n_store"])


# one case per released path: (variant, task, scale, launch) of its first launcher
CASES = [
    ("tiny", "sr", 2, "conv_first"), ("tiny", "sr", 2, "stage0.block0.qkv"), ("tiny", "sr", 2, "stage0.block0.anchor"),
    ("tiny", "sr", 2, "stage0.block0.proj"), ("tiny", "sr", 2, "stage0.block0.fc1"), ("tiny", "sr", 2, "stage0.conv"),
    ("tiny", "sr", 2, "conv_after_body"), ("tiny", "sr", 2, "upsample.up.0"), ("tiny", "sr", 3, "upsample.up.0"),
    ("tiny", "sr", 4, "upsample.up.0"), ("tiny", "dn", 1, "conv_last"),
    ("small", "sr", 2, "conv_first"), ("small", "sr", 2, "stage0.block0.qkv"), ("small", "sr", 2, "stage0.block0.anchor"),
    ("small", "sr", 2, "stage0.block0.proj"), ("small", "sr", 2, "stage0.block0.fc1"),
    ("small", "sr", 2, "stage0.block0.fc2"), ("small", "sr", 2, "stage0.conv"), ("small", "sr", 2, "conv_after_body"),
    ("small", "sr", 2, "conv_before_upsample"), ("small", "sr", 2, "upsample.up.0"), ("small", "sr", 2, "conv_last"),
    ("small", "sr", 3, "upsample.up.0"),
    ("base", "sr", 2, "conv_first"), ("base", "sr", 2, "stage0.block0.qkv"), ("base", "sr", 2, "stage0.block0.anchor"),
    ("base", "sr", 2, "stage0.block0.cab1"), ("base", "sr", 2, "stage0.block0.cab2"), ("base", "sr", 2, "stage0.block0.proj"),
    ("base", "sr", 2, "stage0.block0.fc1"), ("base", "sr", 2, "stage0.block0.fc2"), ("base", "sr", 2, "stage0.conv"),
    ("base", "sr", 2, "conv_after_body"),
]


def _extras():
    """Paths no released config takes, kept from the earlier operator tests: direct stores on a linear, odd fp32
    widths, a single-tile QKV and LayerNorm widths / k depths of other architectures."""
    from grl_image_restoration_b200 import tc

    h, f = tc.Spec, torch.float32
    x16 = lambda *s: h(s, torch.float16)

    def lin(name, kpad, npad, n, act=0, slope=0.0):
        return tc.gemm_launch(name, x16(64, kpad), x16(npad, kpad), h((npad,), f), M=64, kpad=kpad, npad=npad, n_store=npad,
                              n_real=n, out_bf16=x16(64, npad), out_f32=h((64, n), f), act=act, slope=slope)

    def conv(name, kpad, npad, n, act=0, slope=0.0):
        return tc.gemm_launch(name, x16(1, 8, 16, kpad), x16(npad, 9 * kpad), h((npad,), f), image=(1, 8, 16), kpad=kpad,
                              npad=npad, taps=9, n_store=npad, n_real=n, out_bf16=x16(1, 8, 16, npad),
                              out_f32=h((1, 8, 16, n), f), res_f32=h((1, 8, 16, n), f), act=act, slope=slope)

    def ln(name, kpad, C, cab):
        n_ln, cpad = 64 if C <= 64 else 128 if C <= 128 else 192, tc.round_up(C, 64)
        kw = dict(cab_y=x16(64, cpad), cab_gate=h((1, C), f)) if cab else {}
        return tc.gemm_launch(name, x16(64, kpad), x16(n_ln, kpad), h((n_ln,), f), M=64, kpad=kpad, npad=n_ln, epi=tc.EPI_LN,
                              n_store=n_ln, n_real=C, out_bf16=x16(64, cpad), out_f32=h((64, C), f), res_f32=h((64, C), f),
                              C=C, gamma=h((C,), f), beta=h((C,), f), eps=1e-5, res_scale=0.5, L=64, **kw)

    return [
        lin("extra: linear, direct stores, 2 N tiles, GELU", 192, 384, 360, act=1),
        lin("extra: linear, direct stores, fp32 width 30, LeakyReLU", 64, 64, 30, act=2, slope=0.2),
        lin("extra: linear, direct stores, 3 N tiles", 192, 576, 540),
        lin("extra: linear, fp32 staging, BN 192", 384, 192, 180),
        lin("extra: linear, fp32 staging, BN 64", 64, 64, 64),
        conv("extra: conv, direct stores, GELU + residual", 192, 64, 45, act=1),
        conv("extra: conv, fp32 staging, LeakyReLU + residual", 64, 64, 36, act=2, slope=0.01),
        tc.gemm_launch("extra: QKV in one N tile", x16(64, 192), x16(192, 192), h((192,), f), M=64, kpad=192, npad=192,
                       epi=tc.EPI_QKV, n_store=192, out_bf16=x16(64, 192), slot_scale=h((6,), f)),
        ln("extra: LayerNorm C 64, 3 k chunks", 192, 64, False),
        ln("extra: LayerNorm C 128, 3 k chunks", 192, 128, False),
        ln("extra: LayerNorm C 36 + CAB", 192, 36, True),
    ]


EXTRA_NAMES = ["extra: linear, direct stores, 2 N tiles, GELU", "extra: linear, direct stores, fp32 width 30, LeakyReLU",
               "extra: linear, direct stores, 3 N tiles", "extra: linear, fp32 staging, BN 192",
               "extra: linear, fp32 staging, BN 64", "extra: conv, direct stores, GELU + residual",
               "extra: conv, fp32 staging, LeakyReLU + residual", "extra: QKV in one N tile",
               "extra: LayerNorm C 64, 3 k chunks", "extra: LayerNorm C 128, 3 k chunks", "extra: LayerNorm C 36 + CAB"]


def case_launch(pkg, case):
    from grl_image_restoration_b200 import tc

    if isinstance(case, str):
        return next(e for e in _extras() if e.name == case)
    v, t, s, name = case
    return next(ln for ln in tc.gemm_launches(*archs.model(pkg, v, t, s, 3, "fp16")) if ln.name == name)


ALL_CASES = CASES + EXTRA_NAMES




def row_scale(x):
    """max(|x|, rms of the row) over the last dimension."""
    return torch.maximum(x.abs(), x.pow(2).mean(-1, keepdim=True).sqrt())


def stats32(got, ref, extra=0.0):
    """max |got - ref| in fp32 ulps at max(|ref|, row rms), after subtracting `extra` (absolute) from the error."""
    err = ((got.double() - ref).abs() - extra).clamp_min(0.0)
    return float((err / ulp(row_scale(ref), torch.float32)).max())


def check16_only(got, ref, dtype, gelu, acc_err=None):
    """16-bit-only output: RNE16(ref) unless ref lies within delta of a rounding boundary.  Returns (ok, fraction of
    elements allowed either neighbour, fraction that differ from RNE16(ref)).  acc_err: an absolute bound on the fp32
    accumulation's error per element, added to delta (through GELU: times max |GELU'| = 1.13)."""
    delta = GATE32 * ulp(row_scale(ref), torch.float32) + (O.GELU_AS_ABS_ERR if gelu else 0.0)
    if acc_err is not None:
        delta = delta + (1.13 if gelu else 1.0) * acc_err
    lo, hi, mid = (ref - delta).to(dtype).double(), (ref + delta).to(dtype).double(), ref.to(dtype)
    g = got.double()
    ok = bool(((g >= lo) & (g <= hi)).all())
    return ok, float((lo != hi).double().mean()), float((got != mid).double().mean())


def nan_buffer(shape, dtype, device, guard_cols=0):
    """A NaN-filled buffer with GUARD rows before and after and `guard_cols` extra columns: (view, whole buffer)."""
    rows, cols = math.prod(shape[:-1]), shape[-1]
    buf = torch.full((rows + 2 * GUARD, cols + guard_cols), float("nan"), device=device, dtype=dtype)
    return buf[GUARD:GUARD + rows].view(*shape[:-1], cols + guard_cols)[..., :cols], buf


class Run(NamedTuple):
    launch: object  # the descriptor
    kw: dict        # gemm arguments of the case
    ops: dict       # float64 operands for the reference
    bufs: dict      # output name -> (view, whole buffer)
    sig: tuple


def instantiate(tc, launch, fmt, device, seed, batch=B, size=(HT, WT), L=L_CASE):
    """The case of a descriptor: its launch on `batch` images (conv: of `size` pixels; linear: of L rows), with seeded
    operands and NaN output buffers.  The defaults are the test size."""
    a = dict(launch.args)
    dt = tc.DTYPE[fmt]
    conv = a["taps"] == 9
    kpad, npad, epi = a["kpad"], a["npad"], a["epi"]
    g = torch.Generator(device=device).manual_seed(seed)

    def randn(*s):
        return torch.randn(*s, generator=g, device=device, dtype=torch.float64)

    def spread(n, lo, hi):
        return torch.exp2(lo + (hi - lo) * torch.rand(n, generator=g, device=device, dtype=torch.float64))

    def scaled(rows, cols, lo, hi, dtype):
        """randn(rows, cols) * spread(rows, lo, hi)[:, None], rounded to dtype."""
        if rows <= ROW_CHUNK:
            return (randn(rows, cols) * spread(rows, lo, hi)[:, None]).to(dtype)
        # production sizes: the row scales first, then the rows chunk by chunk, so that no float64 copy of the whole
        # operand exists
        s, out = spread(rows, lo, hi), torch.empty(rows, cols, device=device, dtype=dtype)
        for r0 in range(0, rows, ROW_CHUNK):
            r1 = min(rows, r0 + ROW_CHUNK)
            out[r0:r1] = (randn(r1 - r0, cols) * s[r0:r1, None]).to(dtype)
        return out

    tok = (batch, *size) if conv else (batch * L,)
    rows = math.prod(tok)
    real = a["C"] if epi == tc.EPI_LN else (a["n_real"] or a["n_store"]) if epi == tc.EPI_BIAS_ACT else npad
    x16 = scaled(rows, kpad, -2, 1, dt)  # zero rows and rows of 100 below are exact in both formats
    w = randn(npad, a["taps"] * kpad) * (a["taps"] * kpad) ** -0.5 * spread(npad, -1, 1)[:, None]
    bias = randn(npad) * (2.0 if a["act"] == 1 else 0.1 if epi == tc.EPI_LN else 0.5)
    w[real:], bias[real:] = 0, 0
    kw = {"M": batch * L if not conv else 0, "image": tok if conv else None}
    ops = {}
    if epi == tc.EPI_QKV:
        x16[ZERO_QKV_ROW] = 0
        bias[:32] = 0
        ns = a["slot_scale"].shape[0]
        sc = torch.exp(math.log(100.0) * torch.rand(ns, generator=g, device=device, dtype=torch.float64)) * O.LOG2E
        if ns % 6 == 0:  # [window q|k|v][stripe q|k|v] x heads: value slots keep their scale 0
            h = ns // 6
            sc[(torch.arange(ns, device=device) // h) % 3 == 2] = 0
        kw["slot_scale"] = ops["slot_scale"] = sc.float()
    if epi == tc.EPI_LN:
        C = a["C"]
        # rows of mean 100 and std 1 from one exact product per column, 100 w[n, 0]: their accumulators are exact, so
        # what the gate sees is the epilogue (acc + b in fp32, then the moments)
        w[:C, 0] = 1.0 + 0.01 * randn(C)
        x16[list(HIGH_MEAN_ROWS)] = 0.0
        x16[list(HIGH_MEAN_ROWS), 0] = 100.0
        kw.update(C=C, gamma=(1 + 0.3 * randn(C)).float(), beta=(0.2 * randn(C)).float(), eps=a["eps"],
                  res_scale=a["res_scale"], L=L)
        ops.update(gamma=kw["gamma"], beta=kw["beta"], eps=a["eps"], res_scale=a["res_scale"], L=L)
        if a["cab_y"] is not None:
            ld = a["cab_y"].shape[-1]
            kw["cab_y"] = scaled(rows, ld, -1, 1, dt)
            kw["cab_gate"] = torch.sigmoid(randn(batch, C)).float()
            ops.update(cab_y=kw["cab_y"], cab_gate=kw["cab_gate"])
    x16 = x16.view(*tok, kpad)
    w16, b32 = w.to(dt), bias.float()
    ops.update(x=x16, w=w16, bias=b32, taps=a["taps"], epi=epi, act=a["act"], slope=a["slope"])
    if a["res_f32"] is not None:
        n = a["res_f32"].shape[-1]
        kw["res_f32"] = ops["res"] = scaled(rows, n, -1, 1, torch.float32).view(*tok, n)
        ops["n_res"] = n
    bufs = {}
    if a["out_bf16"] is not None:
        ld = a["out_bf16"].shape[-1]
        shape = (batch, size[0] * a["ps_r"], size[1] * a["ps_r"], ld) if a["ps_r"] else (*tok, ld)
        bufs["out_bf16"] = nan_buffer(shape, dt, device)
    if a["out_f32"] is not None:
        bufs["out_f32"] = nan_buffer((*tok, a["out_f32"].shape[-1]), torch.float32, device, guard_cols=4)
        ops["n_res"] = a["n_real"]
    if a["out_nchw"] is not None:
        r = a["nchw_r"]
        crop = (size[0] * r - 1, size[1] * r - 3)
        bufs["out_nchw"] = nan_buffer((batch, a["out_nchw"].shape[1], *crop), torch.float32, device)
        kw.update(nchw_r=r, post_scale=a["post_scale"], post_shift=a["post_shift"])
        ops.update(nchw_r=r, crop=crop, post_scale=a["post_scale"], post_shift=a["post_shift"], n_res=a["n_real"])
    for k, (view, _) in bufs.items():
        kw[k] = view
    if a["ps_r"]:
        kw["ps_r"] = ops["ps_r"] = a["ps_r"]
    kw.update(kpad=kpad, npad=npad, taps=a["taps"], epi=epi, n_store=a["n_store"], n_real=a["n_real"], act=a["act"],
              slope=a["slope"])
    run_launch = tc.gemm_launch(launch.name, x16, w16, b32, **kw)
    return Run(launch, dict(x16=x16, w16=w16, bias=b32, **kw), ops, bufs, path(run_launch))


def evaluate(tc, run, got, ref, fmt, row0=0, high_mean_rows=HIGH_MEAN_ROWS, acc_err=None):
    """Gate results {what: (statistic, passes)} of the kernel outputs `got` against reference `ref`, whose rows are
    the problem's rows from row0 on.  LayerNorm rows listed in high_mean_rows are gated by GATE_LN_SHIFT.  acc_err: see
    check16_only (16-bit-only outputs of a bias / activation epilogue)."""
    a, dt = run.kw, tc.DTYPE[fmt]
    epi = a["epi"]
    gelu = a["act"] == 1
    out = {}
    y = ref["y"]
    real = y.shape[1] if epi != tc.EPI_BIAS_ACT else (a["n_real"] or a["n_store"])
    has32 = "out_f32" in got
    if has32:
        g32 = got["out_f32"].reshape(y.shape[0], -1)
        n = g32.shape[1]
        extra = O.GELU_AS_ABS_ERR if gelu else 0.0
        if epi == tc.EPI_LN:
            hm = torch.isin(torch.arange(row0, row0 + y.shape[0], device=y.device),
                            torch.tensor(high_mean_rows, dtype=torch.long, device=y.device))
            s = stats32(g32[~hm], y[~hm, :n])
            out["fp32"] = (s, s <= GATE32)
            if bool(hm.any()):
                s = stats32(g32[hm], y[hm, :n])
                out["fp32 high-mean rows"] = (s, s <= GATE_LN_SHIFT)
        else:
            s = stats32(g32, y[:, :n], extra)
            out["fp32"] = (s, s <= GATE32)
    if "out_bf16" in got and not a.get("ps_r"):
        g16 = got["out_bf16"].reshape(y.shape[0], -1)[:, :real]
        if has32:
            r16 = got["out_f32"].reshape(y.shape[0], -1)[:, :real].to(dt)
            same = bool((g16.view(torch.int16) == r16.view(torch.int16)).all())
            out["16-bit == RNE(own fp32)"] = (float((g16 != r16).double().mean()), same)
        else:
            yr = y[:, :real]
            if epi == tc.EPI_QKV:  # the row of a normalised output is its 32-wide slot
                g16, yr = g16.reshape(-1, 32), yr.reshape(-1, 32)
            ok, allowed, differ = check16_only(g16, yr, dt, gelu, None if acc_err is None else acc_err[:, :real])
            out["16-bit"] = ((allowed, differ), ok)
    if a.get("ps_r"):
        ok, allowed, differ = check16_only(got["out_bf16"], ref["ps"], dt, gelu)
        out["16-bit PixelShuffle"] = ((allowed, differ), ok)
    if "out_nchw" in got:
        s = stats32(got["out_nchw"], ref["nchw"])
        out["NCHW tail"] = (s, s <= GATE32)
    return out


def check_buffers(tc, run, fmt, mode):
    """Every element the kernel owns is written (finite; 16-bit pad columns exactly 0), nothing else is."""
    a = run.kw
    for name, (view, buf) in run.bufs.items():
        full = buf.float()
        assert bool(full[:GUARD].isnan().all() and full[-GUARD:].isnan().all()), f"{name}: wrote into a guard row"
        inner = full[GUARD:-GUARD]
        if name == "out_f32":
            n = view.shape[-1]
            assert bool(inner[:, :n].isfinite().all()), "out_f32: an element was not written (or is not finite)"
            assert bool(inner[:, n:].isnan().all()), "out_f32: wrote into the guard columns"
        elif name == "out_nchw" or a.get("ps_r"):
            assert bool(inner.isfinite().all()), f"{name}: an element was not written"
        else:
            ld = inner.shape[1]
            real = a["C"] if a["epi"] == tc.EPI_LN else (a["n_real"] or a["n_store"]) if a["epi"] == tc.EPI_BIAS_ACT else a["npad"]
            written = ld if mode == 1 else min(ld, a["n_store"])
            assert bool(inner[:, :written].isfinite().all()), "out_bf16: an element was not written"
            assert bool((inner[:, real:written] == 0).all()), "out_bf16: pad columns are not exactly 0"
            assert bool(inner[:, written:].isnan().all()), "out_bf16: wrote beyond the stored columns"
    if a["epi"] == tc.EPI_QKV:
        z = run.bufs["out_bf16"][0].float()[ZERO_QKV_ROW, :32]
        assert bool((z == 0).all()), "all-zero QKV row: not exactly 0"
