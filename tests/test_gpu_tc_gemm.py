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

import numpy as np
import pytest
import torch

import archs
import grl_oracle as O
from gemm_cases import ALL_CASES, CASES, EXTRA_NAMES, case_launch, check_buffers, evaluate, instantiate, path


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


def rtz16(v, dtype):
    """float64 -> dtype rounded toward zero (the truncating-store mutation)."""
    r = v.to(dtype)
    bits = r.view(torch.int16)
    return torch.where(r.double().abs() > v.abs(), bits - 1, bits).view(dtype)


def reference(run, bn, mutation=None):
    o = dict(run.ops)
    return O.gemm_launch_reference(o.pop("x"), o.pop("w"), o.pop("bias"), bn=bn, mutation=mutation, **o)


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
