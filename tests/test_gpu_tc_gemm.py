"""The tensor-core GEMM / implicit-GEMM conv kernel (csrc/gemm_tc.cu) on every launch path the released configs take,
against a float64 reference of the same launch (grl_oracle.gemm_launch_reference).

A launch's path is its signature (`path`).  The library's answer for it (grl_tc_gemm_path, the host-side selection the
launch itself runs): the N tile width BN, the epilogue, conv or linear, the store mode epi_mode, more than one N tile, a
partial last N tile and min(k chunks, 5) (5 and more wrap the 4-stage operand ring).  Flags of the problem: the
activation, a residual, 16-bit / fp32 / PixelShuffle / NCHW-tail outputs, the residual on the NCHW tail, the CAB add and
a 16-bit pitch wider than the stored columns.  The image size does not enter it.  tc.gemm_launches lists the launches of
one forward (checked one for one against the launches of real forwards by test_recorded_launches_match_descriptors);
test_released_gemm_paths_have_cases (CPU) walks every architecture of archs.architectures through it and fails on a
signature without a case.

Every case is the released launch (or an extra) at a small size with its edges built in: B = 2, a partial last row tile
(linear: M = 200 rows, 2 images of L = 100, so the image boundary lies inside a row tile), conv images of 13 x 21 pixels
(H % 8 != 0, W % 16 != 0).  Inputs have a spread of row and column scales; GELU inputs reach below -8; one QKV row is
all zero; LayerNorm rows 5 and 133 have a mean about 100 times their std.  Outputs are views into NaN-filled buffers
with guard rows (fp32: also guard columns): every element the kernel owns must be written and nothing else.

Gates (measured on an H100 80GB HBM3 at a 400 W power limit, set to 2 x the worst unmutated case):
  fp32 outputs: |got - ref| in fp32 ulps at max(|ref|, the row's rms) <= GATE32 (the high-mean LayerNorm rows:
    GATE_LN_SHIFT, since the fp32 sum acc + b alone costs about ulp(mean) / std there).  The worst case grows with K:
    the wgmma accumulation is not an IEEE fp32 sum;
  16-bit outputs of a launch that also writes fp32: bit-exact round-to-nearest-even of the kernel's own fp32 value;
  16-bit-only outputs: RNE16(ref) unless ref lies within delta = GATE32 fp32 ulps (+ GELU_AS_ABS_ERR after GELU) of a
    rounding boundary, in which case either neighbour passes (QKV: the rms is the 32-wide slot's).  The fraction of
    elements allowed either neighbour and the fraction that differ from RNE16(ref) are printed.
Mutation controls are derived from the reference (a kernel bug's effect, never an edited kernel) and must fail the
gate on every case where they apply.
"""
import copy
import math
from typing import NamedTuple

import numpy as np
import pytest
import torch

import archs
import grl_oracle as O

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


def test_released_gemm_paths_have_cases(pkg):
    """Every launch path of every architecture of archs.architectures has a case, and every case of CASES is a
    launched path."""
    from grl_image_restoration_b200 import tc

    cases = [(path(case_launch(pkg, c)), c) for c in CASES + EXTRA_NAMES]
    assert len(dict(cases)) == len(cases), "two cases share a path"
    launched = [(path(ln), f"{name} {ln.name}") for name, model, shape in archs.architectures(pkg, "fp16")
                for ln in tc.gemm_launches(model, shape)]
    archs.check_walk("tensor-core gemm", launched, cases[:len(CASES)], cases[len(CASES):])


def test_gelu_as_bound():
    """gelu_as (gemm_tc.cu) against float64 erf-GELU on a dense fp32 grid: |err| <= GELU_AS_ABS_ERR (measured 3.8e-7).
    Relative to fp16 that is up to 1.2 ulp on [-4, -1] and 2 subnormal ulp below -4, which the 16-bit gate allows for."""
    from scipy.special import erf

    x = np.concatenate([np.linspace(-12, 12, (1 << 22) + 1, dtype=np.float32),
                        np.linspace(-4, -1, 1 << 20, dtype=np.float32)])
    got = O.gelu_as_emulate(x).astype(np.float64)
    xd = x.astype(np.float64)
    ref = 0.5 * xd * (1 + erf(xd / math.sqrt(2)))
    err = np.abs(got - ref)
    band = (x >= -4) & (x <= -1)
    ulp16 = np.spacing(np.abs(ref[band]).astype(np.float16)).astype(np.float64)
    print(f"gelu_as: max |err| {err.max():.3e}; on [-4, -1] max {float((err[band] / ulp16).max()):.2f} fp16 ulp")
    assert err.max() <= O.GELU_AS_ABS_ERR


# ----------------------------------------------------------------------------------------------------------------- GPU


def ulp32(x):
    return torch.clamp(torch.finfo(torch.float32).eps * torch.exp2((torch.frexp(x.abs())[1] - 1).double()),
                       min=2.0 ** -149)


def row_scale(x):
    """max(|x|, rms of the row) over the last dimension."""
    return torch.maximum(x.abs(), x.pow(2).mean(-1, keepdim=True).sqrt())


def stats32(got, ref, extra=0.0):
    """max |got - ref| in fp32 ulps at max(|ref|, row rms), after subtracting `extra` (absolute) from the error."""
    err = ((got.double() - ref).abs() - extra).clamp_min(0.0)
    return float((err / ulp32(row_scale(ref))).max())


def rtz16(v, dtype):
    """float64 -> dtype rounded toward zero (the truncating-store mutation)."""
    r = v.to(dtype)
    bits = r.view(torch.int16)
    return torch.where(r.double().abs() > v.abs(), bits - 1, bits).view(dtype)


def check16_only(got, ref, dtype, gelu):
    """16-bit-only output: RNE16(ref) unless ref lies within delta of a rounding boundary.  Returns (ok, fraction of
    elements allowed either neighbour, fraction that differ from RNE16(ref))."""
    delta = GATE32 * ulp32(row_scale(ref)) + (O.GELU_AS_ABS_ERR if gelu else 0.0)
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


def reference(run, bn, mutation=None):
    o = dict(run.ops)
    return O.gemm_launch_reference(o.pop("x"), o.pop("w"), o.pop("bias"), bn=bn, mutation=mutation, **o)


def evaluate(tc, run, got, ref, fmt, row0=0, high_mean_rows=HIGH_MEAN_ROWS):
    """Gate results {what: (statistic, passes)} of the kernel outputs `got` against reference `ref`, whose rows are
    the problem's rows from row0 on.  LayerNorm rows listed in high_mean_rows are gated by GATE_LN_SHIFT."""
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
            ok, allowed, differ = check16_only(g16, yr, dt, gelu)
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


def mutations(tc, run, q):
    """Mutation name -> None (applies to the reference) or "store" (the 16-bit store), for the ones this case has."""
    a = run.kw
    out = {}
    if "out_bf16" in run.bufs:
        out["16-bit stores truncate"] = "store"
    if q.n_tiles > 1:
        out["bias_tile_local"] = None
        if a["epi"] == tc.EPI_QKV:
            out["slot_scale_per_tile"] = None
    if q.nk_total >= 5:
        out["drop_kchunk"] = None
    if a["taps"] == 9:
        out["taps_transposed"] = None
    if a["epi"] == tc.EPI_LN:
        out.update(ln_unbiased=None, ln_no_eps=None, ln_naive_fp32=None)
        if a.get("cab_y") is not None:
            out["cab_gate_per_tile"] = None
    if a.get("res_f32") is not None:
        out["no_residual_last_tile"] = None
    if a["act"] == 1:
        out["gelu_tanh"] = None
    if a.get("ps_r"):
        out["ps_swapped"] = None
    return out


ALL_CASES = CASES + EXTRA_NAMES


def case_id(c):
    return c.split(":")[1].strip().replace(" ", "_") if isinstance(c, str) else f"{c[0]}-{c[1]}x{c[2]}-{c[3]}"


@pytest.fixture(scope="module")
def tc(pkg, device):
    from grl_image_restoration_b200 import capi, tc as T

    if capi.lib().grl_device_ok() != 1:
        pytest.skip("wgmma path needs sm_90")
    return T


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", ALL_CASES, ids=case_id)
def test_gemm_path(pkg, tc, device, case, fmt):
    launch = case_launch(pkg, case)
    sig = path(launch)
    run = instantiate(tc, launch, fmt, device, seed=ALL_CASES.index(case) * 2 + fmt)
    assert run.sig == sig, f"the case runs path {run.sig}, not its launch's {sig}"
    q = tc.gemm_path(launch)
    tc.gemm(**run.kw)
    torch.cuda.synchronize()
    check_buffers(tc, run, fmt, q.epi_mode)
    got = {k: v for k, (v, _) in run.bufs.items()}
    ref = reference(run, q.bn)
    res = evaluate(tc, run, got, ref, fmt)
    print(f"\n[{tc.DTYPE[fmt]}] {case} path={sig}")
    for what, (s, ok) in res.items():
        print(f"  {what}: {s} {'ok' if ok else 'FAILS'}")
    assert all(ok for _, ok in res.values()), res

    missed = []
    for name, kind in mutations(tc, run, q).items():
        if kind == "store":
            mgot = dict(got)
            src = got["out_f32"].reshape(-1, got["out_f32"].shape[-1]).double() if "out_f32" in got else None
            if src is not None and not run.kw.get("ps_r"):
                g16 = got["out_bf16"].reshape(src.shape[0], -1).clone()
                n = min(src.shape[1], g16.shape[1])
                g16[:, :n] = rtz16(src[:, :n], tc.DTYPE[fmt])
                mgot["out_bf16"] = g16
            else:
                key = "ps" if run.kw.get("ps_r") else "y"
                t = rtz16(ref[key], tc.DTYPE[fmt])
                mgot["out_bf16"] = t
            mres = evaluate(tc, run, mgot, ref, fmt)
        else:
            mres = evaluate(tc, run, got, reference(run, q.bn, name), fmt)
        caught = not all(ok for _, ok in mres.values())
        print(f"  mutation '{name}': {'FAILS the gate' if caught else 'passes the gate'} "
              f"{ {k: v[0] for k, v in mres.items()} }")
        if not caught:
            missed.append(name)
    assert not missed, f"mutations the gate does not catch: {missed}"


@pytest.mark.gpu
@pytest.mark.parametrize("variant,task,scale", [("tiny", "sr", 2), ("small", "sr", 3), ("base", "sr", 4), ("base", "dn", 1)])
def test_recorded_launches_match_descriptors(pkg, tc, device, monkeypatch, variant, task, scale):
    """tc.gemm_launches lists, one for one and in order, the tc.gemm calls of a real forward (smallest padded size, an
    input that needs padding)."""
    cfg = pkg.configs.grl_config(variant, task, scale)
    model = pkg.GRL(**dict(cfg, img_size=archs.smallest_size(cfg)))
    model.use_cuda_graph = False
    model = model.to(device).eval()
    model.set_precision("fp16")
    S = model.pad_size
    x = torch.rand(1, 3, S - 5, S - 3, generator=torch.Generator().manual_seed(0)).to(device)
    recorded, gemm = [], tc.gemm

    def spy(x16, w16, bias, **kw):
        recorded.append(tc.gemm_launch("", x16, w16, bias, **kw).args)
        gemm(x16, w16, bias, **kw)

    monkeypatch.setattr(tc, "gemm", spy)
    y = model(x)
    torch.cuda.synchronize()
    assert y.shape == (1, 3, (S - 5) * cfg["upscale"], (S - 3) * cfg["upscale"])
    want = tc.gemm_launches(model, tuple(x.shape))
    assert len(recorded) == len(want), (len(recorded), len(want))
    for got, ln in zip(recorded, want):
        diff = {k: (got[k], v) for k, v in ln.args.items() if got[k] != v}
        assert not diff, f"{ln.name}: {diff}"


@pytest.mark.gpu
def test_listing_first_leaves_the_forward_unchanged(pkg, tc, device):
    """gemm_launches on a fresh model, then its forward at the model's own resolution (where both read the registered
    coordinate tables): bitwise the forward of an identical model that was never listed.  A listing run packs weights
    on the device, but its attention constants are meta tensors and must not be kept for the forward."""
    cfg = pkg.configs.grl_config("tiny", "sr", 2)
    cfg = dict(cfg, img_size=archs.smallest_size(cfg))
    torch.manual_seed(0)
    listed = pkg.GRL(**cfg)
    fresh = copy.deepcopy(listed)
    S = listed.pad_size
    x = torch.rand(1, 3, S, S, generator=torch.Generator().manual_seed(0)).to(device)
    ys = []
    for model, list_first in ((fresh, False), (listed, True)):
        model.use_cuda_graph = False
        model = model.to(device).eval()
        model.set_precision("fp16")
        if list_first:
            assert len(tc.gemm_launches(model, tuple(x.shape))) > 0
        ys.append(model(x))
    torch.cuda.synchronize()
    assert torch.equal(ys[0], ys[1])
