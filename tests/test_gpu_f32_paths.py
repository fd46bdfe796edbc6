"""The fp32 parity path's kernels (csrc/ops_f32.cu) on every launch path the released configs take, against float64.

Launch paths.  An attention launch's signature (`attn_path`) is the kernel specialisation plus its tile edges: the role
(window, stripe pass 1, stripe pass 2: this fixes dense V and dense output), the head_dim template D, d < D, a partial
and a second 128-query tile, a partial and a second 32-key tile, the shift mask and a non-zero roll.  A GEMM's
(`gemm_path`) is conv or linear, a partial last 16-wide k tile, the number of k tiles, a partial and a second 64-wide N
tile, the activation, bias and residual.  The CPU tests walk every architecture of archs.architectures through
f32_launches, the fp32 forward run in listing mode: its K.linear / K.conv3x3 calls and the passes of its
K.window_attention / K.stripe_attention calls, and fail naming any path without a case.
test_recorded_launches_match_lists checks that list one for one against the C-ABI calls of real fp32 forwards.

Cases call the C ABI directly and write into NaN-filled buffers with guard rows (and guard columns where a pitch
allows): every owned element must be written and nothing else.  Attention: 2 x 2 windows of the pass's grid, B = 2, the
config's heads and head_dim, the production 6c-wide qkv pitch; q and k un-normalised with one all-zero token, per-head
logit scales across the ln 100 clamp, a CPB-like bias table.  Stripe pass 2 is checked on the kernel's own X1, and the
whole chain against the float64 chain.  GEMM: B = 2, M = 200 linear rows (an image boundary inside a 64-row tile), conv
images of 13 x 21, spread row and column scales, GELU inputs below -8, and rows (linear) or pixels (conv, every tap)
of zero input, whose accumulators are exact, so the gate there sees the epilogue alone.

Gates: |got - ref64| <= bound per element, with bounds derived from the kernels' fixed summation orders (u = 2^-24,
gamma_n = n u / (1 - n u), erff / expf errors from the CUDA Programming Guide):
  GEMM / conv: gamma_K sum |a_k w_k| for the FMA chain, one rounding each for bias, activation and residual; the erf
    term of GELU counts as absolute, 0.5 |x| (erff error + 3 u), since 1 + erf cancels below about -3;
  ln_residual: two-pass moments over C with the warp's lane-strided order (ceil(C / 32) + 5 additions per sum);
  channel gate: 256-row chunk sums, a sequential sum over the chunks, the MLP (lane-strided + warp tree, then a
    sequential chain), expf;
  bias table: the 2-FMA hidden unit, ReLU, a 512-long FMA chain, expf;
  avgpool: bit-exact (a sequential fp32 sum in (dy, dx) order times an exact power-of-two division).
Attention is gated as measured: |got - ref64| in fp32 ulps at max(|ref|, the row's rms) <= GATE_ATTN (pass 2 on the
whole chain: GATE_CHAIN), 2 x the worst case of one run on an H100 80GB HBM3 at a 400 W power limit.  Every case
prints its worst error / bound ratio.  Mutation controls are derived from the float64 reference (a kernel bug's
effect, never an edited kernel); each must fail its gate on every case where it applies, and each case prints which
of them the old operator tests' 2e-4 max-abs bound would have missed.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

import archs
import grl_oracle as O
from f32_cases import (ACT_GELU, ACT_LEAKY, ACT_NONE, ATTN_CASES, ATTN_EXTRAS, ATTN_ZOO_CASES, B, GATE_ATTN, GATE_CHAIN,
                       GEMM_CASES, GEMM_EXTRAS, GEMM_ZOO_CASES, POOL_ROWS, Pass, attn_case_launch, attn_path,
                       attn_ref, bias_table_bound, gate_bound, gate_reference, gemm_bound, gemm_path, im2col, launches_of,
                       ulp_stats, windows)
from grl_oracle import L_LN, ln_bound, ln_reference
from support import bound_ratio, grid_t

GUARD = 3          # NaN guard rows before and after every output buffer
OLD_TOL = 2e-4     # the max-abs bound of the operator tests this file replaces


# ------------------------------------------------------------------------------------------------------- attention


def test_released_attention_paths_have_cases(pkg):
    """Every attention path of every block of every architecture of archs.architectures has a case, and every case of
    ATTN_CASES and ATTN_ZOO_CASES is a launched path."""
    from grl_image_restoration_b200 import modules

    cases = [(attn_path(attn_case_launch(c)[1]), c) for c in ATTN_CASES + ATTN_ZOO_CASES]
    assert len(dict(cases)) == len(cases), "two cases share a path"
    launched = [(attn_path(ln), f"{name} {ln.name} {ln.role}")
                for name, model, shape in archs.architectures(pkg, "fp32")
                for ln in launches_of(modules.f32_launches(model, shape), "AttnF32")]
    archs.check_walk("fp32 attention", launched, cases, [(attn_path(attn_case_launch(c)[1]), c) for c in ATTN_EXTRAS])


# ------------------------------------------------------------------------------------------------------------ GEMM


def test_released_gemm_paths_have_cases(pkg):
    """Every GEMM path of the fp32 forward of every architecture of archs.architectures has a case, and every case of
    GEMM_CASES and GEMM_ZOO_CASES is a launched path."""
    from grl_image_restoration_b200 import modules

    released = GEMM_CASES + GEMM_ZOO_CASES
    cases = [(gemm_path(c.call()), c) for c in released + GEMM_EXTRAS]
    assert len(dict(cases)) == len(cases), "two cases share a path"
    launched = [(gemm_path(g), f"{name} {g.name}") for name, model, shape in archs.architectures(pkg, "fp32")
                for g in launches_of(modules.f32_launches(model, shape), "GemmF32")]
    archs.check_walk("fp32 gemm", launched, cases[:len(released)], cases[len(released):])


# ----------------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def lib(pkg, device):
    from grl_image_restoration_b200 import capi

    if capi.lib().grl_device_ok() != 1:
        pytest.skip("the library is built for sm_90a")
    return capi.lib()


def ptr(t, offset=0):
    return ctypes.c_void_p(t.data_ptr() + 4 * offset)


def stream():
    from grl_image_restoration_b200 import capi

    return capi.stream()


def nan_rows(rows, cols, device, guard_cols=0):
    """A NaN-filled (rows, cols + guard_cols) fp32 buffer with GUARD rows before and after: (inner rows, whole)."""
    buf = torch.full((rows + 2 * GUARD, cols + guard_cols), float("nan"), device=device)
    return buf[GUARD:GUARD + rows], buf


def check_written(buf, cols, what, guard_cols=0):
    """The inner rows' first `cols` columns are all written (finite); guard rows and columns are untouched."""
    assert bool(buf[:GUARD].isnan().all() and buf[-GUARD:].isnan().all()), f"{what}: wrote into a guard row"
    inner = buf[GUARD:-GUARD]
    assert bool(inner[:, :cols].isfinite().all()), f"{what}: an owned element was not written"
    if guard_cols:
        assert bool(inner[:, cols:].isnan().all()), f"{what}: wrote into the guard columns"


def old_misses(mut, ref):
    """The old operator tests' bound would pass a kernel that computes `mut` instead of `ref`."""
    return float((mut - ref).abs().nan_to_num(float("inf")).max()) <= OLD_TOL


def report(name, ratio, gate, kind="bound"):
    caught = not ratio <= gate
    print(f"  mutation '{name}': {ratio:.3g} x {kind} -> {'FAILS the gate' if caught else 'passes the gate'}")
    return caught


# --------------------------------------------------------------------------------------------------- GPU: attention


def cpb_like(rows_hw, df, heads, seed, device):
    """(heads, rows) 16 sigmoid(MLP(coords)) of a random CPB-like MLP over a launch's relative coordinates."""
    coords = O.coords_table(list(rows_hw), df).reshape(-1, 2).double()
    g = torch.Generator().manual_seed(seed)
    w1, b1 = torch.randn(512, 2, generator=g).double() * 0.7, torch.randn(512, generator=g).double() * 0.1
    w2 = torch.randn(heads, 512, generator=g).double() * 0.15
    return (16 * torch.sigmoid(torch.relu(coords @ w1.T + b1) @ w2.T)).T.float().contiguous().to(device)


def logit_scales(heads, reverse, device):
    """Per-head logit scales (natural log) from ln 5 to ln 150: they cross the clamp at ln 100."""
    s = torch.linspace(math.log(5.0), math.log(150.0), heads) if heads > 1 else torch.tensor([math.log(150.0)])
    return (s.flip(0) if reverse else s).float().to(device)


def attn_mutations(p, heads, x1_kernel=None):
    """Mutation name -> the float64 reference of a kernel with that bug, for the mutations that apply to this pass."""
    out = {}
    index, mask = O.attn_pair_geometry(p.gq, p.gk, p.use_mask)
    nk = index.shape[1]
    # the relative position whose neighbour's entry moves the softmax most, on the last window: max p (1 - p) |e^delta - 1|
    q, k = windows(p.q, p.gq, heads)[-1:], windows(p.k, p.gk, heads)[-1:]
    tab = p.table.double()
    idx = index.to(tab.device)
    x = F.normalize(q, dim=-1) @ F.normalize(k, dim=-1).transpose(-1, -2)
    x = x * torch.exp(p.scale.double().clamp(max=math.log(100.0)))[:, None, None] + tab[:, idx]
    if mask is not None:
        x = x + mask[-1].to(x)
    pr = torch.softmax(x, -1)
    nb = (idx + 1).clamp(max=tab.shape[1] - 1)
    hit = (pr * (1 - pr) * (torch.exp(tab[:, nb] - tab[:, idx]) - 1).abs()).reshape(-1, idx.numel()).amax(0).argmax()
    r = int(idx.flatten()[hit])
    out["bias entry read from its neighbour"] = attn_ref(p, heads, index=torch.where(index == r, r + 1, index))
    if mask is not None and bool((mask[-1] != 0).any()):
        w = mask.shape[0] - 1  # the bottom-right window: masked and wrapped
        rq = O.region_ids(p.gq[:2], p.gq[2:4], p.gq[4:6])[w]
        rk = O.region_ids(p.gk[:2], p.gk[2:4], p.gk[4:6])[w]
        i, j = (mask[w] != 0).nonzero()[0].tolist()
        m2 = mask.clone()
        m2[w] = torch.where((rq[:, None] == rq[i]) & (rk[None, :] == rk[j]), 0.0, mask[w])
        out["shift-mask region pair unmasked"] = attn_ref(p, heads, mask=m2)
    if any(p.gq[4:6]) or any(p.gk[4:6]):
        out["roll missing"] = attn_ref(p, heads, roll=False)
    if nk % 32:
        out["last key of the partial key tile dropped"] = attn_ref(p, heads, drop_last_key=True)
    if bool((p.scale > math.log(100.0)).any()):
        out["logit scale not clamped at ln 100"] = attn_ref(p, heads, "scale_unclamped")
    out["k not normalised"] = attn_ref(p, heads, "k_unnormalised")
    if nk > 32:
        out["rescale missing from the denominator"] = attn_ref(p, heads, "rescale_missing_l")
    if x1_kernel is not None and heads > 1:
        out["pass 2 reads X1 of the neighbouring head"] = attn_ref(p, heads, v=x1_kernel.roll(-1, 1))
    return out


def attn_inputs(case, x_size, device, seed):
    """qkv (B L, 6c) with per-token-head scales 2^U(-2, 2) and one all-zero token; anchors (B, Ha, Wa, c) likewise."""
    h, d = case.heads, case.d
    c = h * d
    H, W = x_size
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B * H * W, 6 * h, d, generator=g) * torch.exp2(4 * torch.rand(B * H * W, 6 * h, 1, generator=g) - 2)
    qkv[H * W + 5] = 0.0  # batch 1: q = k = v = 0 takes the F.normalize eps path
    Ha, Wa = H // case.df, W // case.df
    anc = torch.randn(B * Ha * Wa, h, d, generator=g) * torch.exp2(4 * torch.rand(B * Ha * Wa, h, 1, generator=g) - 2)
    anc[Ha * Wa + 1] = 0.0
    return qkv.view(B * H * W, 6 * c).to(device), anc.view(B, Ha, Wa, c).to(device)


def attn_id(c):
    return (f"{c.src.split(':')[0].replace('/', '-')}-{c.role}-{c.win[0]}x{c.win[1]}-df{c.df}-"
            f"{'s' if c.shifted else 'u'}-h{c.heads}d{c.d}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ATTN_CASES + ATTN_EXTRAS + ATTN_ZOO_CASES, ids=attn_id)
def test_attention_path(lib, device, case):
    from grl_image_restoration_b200 import capi

    x_size, ln = attn_case_launch(case)
    sig = attn_path(ln)
    h, d = case.heads, case.d
    c = h * d
    H, W = x_size
    L = H * W
    seed = (ATTN_CASES + ATTN_EXTRAS + ATTN_ZOO_CASES).index(case)
    qkv, anc = attn_inputs(case, x_size, device, seed)
    merged, mbuf = nan_rows(B * L, 2 * c, device)
    if case.role == "window":
        gq = ln.gq
        scale = logit_scales(h, False, device)
        table = cpb_like(case.win, 1, h, seed + 100, device)
        capi.check(lib.grl_window_attn_f32(ptr(qkv), 6 * c, ptr(merged), 2 * c, B, gq, h, d, ptr(scale), ptr(table),
                                           int(ln.use_mask), stream()))
        torch.cuda.synchronize()
        check_written(mbuf[:, :c], c, "output")
        assert bool(mbuf[:, c:].isnan().all()), "wrote outside its half of the merged buffer"
        tok = qkv.double().view(B, H, W, 6 * c)
        p = Pass(grid_t(gq), grid_t(gq), tok[..., :c], tok[..., c:2 * c], tok[..., 2 * c:3 * c], False, False, scale,
                 table, ln.use_mask)
        got = windows(merged.view(B, H, W, 2 * c)[..., :c], p.gq, h)
        x1 = None
    else:
        tokg, ancg = (ln.gk, ln.gq) if case.role == "stripe1" else (ln.gq, ln.gk)
        s1, s2 = logit_scales(h, False, device), logit_scales(h, True, device)
        t1, t2 = cpb_like(case.win, case.df, h, seed + 100, device), cpb_like(case.win, case.df, h, seed + 200, device)
        nbytes = lib.grl_stripe_attn_workspace(B, tokg, ancg, h, d)
        ws, wbuf = nan_rows(nbytes // 4 // d, d, device)
        capi.check(lib.grl_stripe_attn_f32(ptr(qkv, 3 * c), 6 * c, ptr(anc), c, ptr(merged, c), 2 * c, B, tokg, ancg,
                                           h, d, ptr(s1), ptr(t1), ptr(s2), ptr(t2), int(ln.use_mask), ptr(ws),
                                           nbytes, stream()))
        torch.cuda.synchronize()
        check_written(wbuf, d, "X1")
        check_written(mbuf[:, c:], c, "output")
        assert bool(mbuf[:, :c].isnan().all()), "wrote outside its half of the merged buffer"
        tok = qkv.double().view(B, H, W, 6 * c)[..., 3 * c:]
        Na = ancg.wh * ancg.ww
        x1 = ws.view(-1, h, Na, d)
        p1 = Pass(grid_t(ancg), grid_t(tokg), anc.double(), tok[..., c:2 * c], tok[..., 2 * c:], False, True, s1, t1,
                  ln.use_mask)
        p2 = Pass(grid_t(tokg), grid_t(ancg), tok[..., :c], anc.double(), x1.double(), True, False, s2, t2,
                  ln.use_mask)
        p, got = (p1, x1) if case.role == "stripe1" else (p2, windows(merged.view(B, H, W, 2 * c)[..., c:], p2.gq, h))
    ref = attn_ref(p, h)
    stats = ulp_stats(got, ref)
    print(f"\n[fp32 attention] {case.src} {case.role} {case.win} df{case.df} shifted={case.shifted} h{h} d{d} path={sig}: "
          f"{stats:.1f} ulp ({stats / GATE_ATTN:.3f} x gate)")
    ok = stats <= GATE_ATTN
    if case.role == "stripe2":
        chain = attn_ref(p2, h, v=attn_ref(p1, h))
        sc = ulp_stats(got, chain)
        print(f"  chain vs float64 chain: {sc:.1f} ulp ({sc / GATE_CHAIN:.3f} x gate)")
        ok = ok and sc <= GATE_CHAIN
    missed, old = [], []
    for name, m in attn_mutations(p, h, x1.double() if case.role == "stripe2" else None).items():
        if not report(name, ulp_stats(got, m), GATE_ATTN, "ulp"):
            missed.append(name)
        if old_misses(m, ref):
            old.append(name)
    print(f"  the old {OLD_TOL} bound misses {len(old)}: {old}")
    assert ok, (case, stats)
    assert not missed, f"mutations the gate does not catch: {missed}"


# -------------------------------------------------------------------------------------------------------- GPU: GEMM


HT, WT, M_LIN = 13, 21, 200
ZERO_ROWS = (7, 150)  # linear rows of zero input: the accumulator is exactly 0


def gemm_operands(case, device, seed):
    g = torch.Generator().manual_seed(seed)
    K, N = case.K, case.N
    cin = K // 9 if case.conv else K
    rows = B * HT * WT if case.conv else M_LIN

    def spread(n, lo, hi):
        return torch.exp2(lo + (hi - lo) * torch.rand(n, generator=g))

    x = torch.randn(rows, cin, generator=g) * spread(rows, -2, 1)[:, None] * spread(cin, -1, 1)[None, :]
    w = torch.randn(N, K, generator=g) * K ** -0.5 * spread(N, -1, 1)[:, None]
    b = torch.randn(N, generator=g) * (3.0 if case.act == ACT_GELU else 0.5)
    if case.act == ACT_GELU:
        b[::5] = -12.0  # GELU inputs below -8, where 1 + erf cancels
    res = (torch.randn(rows, N, generator=g) * spread(rows, -1, 1)[:, None]) if case.res else None
    if case.conv:  # pixel (5, 9) of both images sees zeros on every tap
        x = x.view(B, HT, WT, cin)
        x[:, 4:7, 8:11] = 0.0
    else:
        x[list(ZERO_ROWS)] = 0.0
    return [t if t is None else t.float().to(device) for t in (x, w, b, res)]


def gemm_id(c):
    return c.src.replace("extra: ", "extra-").replace(" ", "_").replace(",", "").replace("/", "-")


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEMM_CASES + GEMM_EXTRAS + GEMM_ZOO_CASES, ids=gemm_id)
def test_gemm_path(lib, device, case):
    from grl_image_restoration_b200 import capi

    x, w, b, res = gemm_operands(case, device, (GEMM_CASES + GEMM_EXTRAS + GEMM_ZOO_CASES).index(case))
    slope = case.call().slope
    K, N = case.K, case.N
    if case.conv:
        M = B * HT * WT
        y, buf = nan_rows(M, N, device)
        capi.check(lib.grl_conv3x3_f32(ptr(x), ptr(w), ptr(b), ptr(res) if res is not None else None, ptr(y), B, HT,
                                       WT, K // 9, N, case.act, slope, stream()))
        guard_cols = 0
    else:
        M, guard_cols = M_LIN, 4
        y, buf = nan_rows(M, N, device, guard_cols)
        capi.check(lib.grl_linear_f32(ptr(x), K, ptr(w), ptr(b), ptr(res) if res is not None else None, N, ptr(y),
                                      N + guard_cols, M, N, K, case.act, slope, stream()))
    torch.cuda.synchronize()
    check_written(buf, N, "output", guard_cols)
    got = y[:, :N]
    x64, w64, b64 = x.double(), w.double(), b.double()
    r64 = None if res is None else res.double()
    A = im2col(x64) if case.conv else x64

    def ref(A=A, w=w64, b=b64, r=r64, mutation=None):
        return O.gemm_launch_reference(A, w, b, act=case.act, slope=slope, n_res=N, res=r, mutation=mutation)["y"]

    y64 = ref()
    bound, v = gemm_bound(A, w64, b64, case.act, slope, r64)
    if case.act == ACT_GELU:
        assert bool((v < -8).any()), "no GELU input below -8"
    ratio = bound_ratio(got, y64, bound)
    print(f"\n[fp32 gemm] {case.src} path={gemm_path(case.call())}: worst error / bound {ratio:.3f}, "
          f"max |err| {float((got.double() - y64).abs().max()):.2e}")
    muts = {}
    if K % 16:
        w2 = w64.clone()
        w2[:, K // 16 * 16:] = 0
        muts["partial last k tile dropped"] = ref(w=w2)
    if case.conv:
        muts["taps transposed"] = ref(A=im2col(x64, transposed=True))
        muts["padding taps wrap into the previous row / image"] = ref(A=im2col(x64, wrap=True))
    if N > 1:
        nb = torch.arange(N, device=device) + 1
        nb[-1] = N - 2
        muts["bias of the neighbouring column"] = ref(b=b64[nb])
    if r64 is not None:
        r2 = r64.clone()
        r2[(M - 1) // 64 * 64:] = 0
        muts["no residual on the last row tile"] = ref(r=r2)
    if case.act == ACT_GELU:
        muts["tanh-GELU"] = ref(mutation="gelu_tanh")
    missed, old = [], []
    for name, m in muts.items():
        if not report(name, bound_ratio(got, m, bound), 1.0):
            missed.append(name)
        if old_misses(m, y64):
            old.append(name)
    print(f"  the old {OLD_TOL} bound misses {len(old)}: {old}")
    assert ratio <= 1.0, (case, ratio)
    assert not missed, f"mutations the gate does not catch: {missed}"


# ------------------------------------------------------------------------------------------- GPU: LayerNorm residual


HIGH_MEAN_ROWS, LOW_STD_ROWS = (5, 133), (7, 150)


LN_CASES = [(C, with_x, cab) for C in (64, 128, 180) for with_x, cab in ((False, False), (True, False), (True, True))]


@pytest.mark.gpu
@pytest.mark.parametrize("C,with_x,cab", LN_CASES, ids=lambda v: str(v))
def test_ln_residual(lib, device, C, with_x, cab):
    from grl_image_restoration_b200 import capi

    g = torch.Generator().manual_seed(C * 4 + 2 * with_x + cab)
    M = B * L_LN
    u = torch.randn(M, C, generator=g) * torch.exp2(3 * torch.rand(M, 1, generator=g) - 1) + torch.randn(M, 1, generator=g)
    for r in HIGH_MEAN_ROWS:
        u[r] = 100.0 + torch.randn(C, generator=g)
    for r in LOW_STD_ROWS:
        u[r] = 0.3 + 1e-2 * torch.randn(C, generator=g)
    gamma_, beta = 1 + 0.3 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
    x = torch.randn(M, C, generator=g) if with_x else None
    cy = torch.randn(M, C, generator=g) * torch.exp2(2 * torch.rand(M, 1, generator=g) - 1) if cab else None
    gate = torch.sigmoid(torch.randn(B, C, generator=g)) if cab else None
    rs, eps = 0.5, 1e-5
    dv = [t if t is None else t.float().to(device) for t in (u, gamma_, beta, x, cy, gate)]
    out, buf = nan_rows(M, C, device)
    capi.check(lib.grl_ln_residual_f32(ptr(dv[3]) if with_x else None, ptr(dv[0]), ptr(dv[1]), ptr(dv[2]), eps, rs,
                                       ptr(dv[4]) if cab else None, ptr(dv[5]) if cab else None, L_LN, ptr(out), M, C,
                                       stream()))
    torch.cuda.synchronize()
    check_written(buf, C, "output")
    d64 = [t if t is None else t.double() for t in dv]
    ref = ln_reference(d64[0], d64[1], d64[2], eps, rs, d64[3], d64[4], d64[5])
    bound = ln_bound(d64[0], d64[1], d64[2], eps, rs, d64[3], d64[4], d64[5])
    ratio = bound_ratio(out, ref, bound)
    hm = list(HIGH_MEAN_ROWS)
    print(f"\n[fp32 ln_residual] C={C} x={with_x} cab={cab}: worst error / bound {ratio:.3f} "
          f"(high-mean rows {bound_ratio(out[hm], ref[hm], bound[hm]):.3f})")
    names = ["n - 1 variance", "no eps", "naive fp32 E[x^2] - E[x]^2", "res_scale dropped"]
    if cab:
        names.append("CAB gate of the wrong image at the boundary")
    missed, old = [], []
    for name in names:
        m = ln_reference(d64[0], d64[1], d64[2], eps, rs, d64[3], d64[4], d64[5], mutation=name)
        if not report(name, bound_ratio(out, m, bound), 1.0):
            missed.append(name)
        if old_misses(m, ref):
            old.append(name)
    print(f"  the old {OLD_TOL} bound misses {len(old)}: {old}")
    assert ratio <= 1.0, ratio
    assert not missed, f"mutations the gate does not catch: {missed}"


# ------------------------------------------------------------------------------------------------ GPU: channel gate

@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 100, 1000])
def test_channel_gate(lib, device, L):
    from grl_image_restoration_b200 import capi

    C, R = 180, 10  # GRL-Base's CAB: ChannelAttention(180, reduction 18)
    g = torch.Generator().manual_seed(L)
    y = torch.randn(B, L, C, generator=g) + 0.3
    w1, b1 = torch.randn(R, C, generator=g) * 0.1, torch.randn(R, generator=g) * 0.5
    w2, b2 = torch.randn(C, R, generator=g) * 0.3, torch.randn(C, generator=g) * 0.5
    dv = [t.float().to(device).contiguous() for t in (y, w1, b1, w2, b2)]
    nbytes = lib.grl_channel_gate_workspace(B, L, C)
    ws = torch.full((nbytes // 4,), float("nan"), device=device)
    out, buf = nan_rows(B, C, device)
    capi.check(lib.grl_channel_gate_f32(ptr(dv[0]), B, L, C, ptr(dv[1]), ptr(dv[2]), ptr(dv[3]), ptr(dv[4]), R,
                                        ptr(out), ptr(ws), nbytes, stream()))
    torch.cuda.synchronize()
    check_written(buf, C, "gate")
    d64 = [t.double() for t in dv]
    ref = gate_reference(*d64)
    bound = gate_bound(*d64)
    ratio = bound_ratio(out, ref, bound)
    print(f"\n[fp32 channel gate] B={B} L={L} C={C} R={R}: worst error / bound {ratio:.3f}")
    missed, old = [], []
    for name in ("partial last chunk dropped", "division by chunks x 256", "ReLU missing"):
        if name == "division by chunks x 256" and L % POOL_ROWS == 0:
            continue
        m = gate_reference(*d64, mutation=name)
        if not report(name, bound_ratio(out, m, bound), 1.0):
            missed.append(name)
        if old_misses(m, ref):
            old.append(name)
    print(f"  the old {OLD_TOL} bound misses {len(old)}: {old}")
    assert ratio <= 1.0, ratio
    assert not missed, f"mutations the gate does not catch: {missed}"


# ------------------------------------------------------------------------------------ GPU: avgpool, bias table


@pytest.mark.gpu
@pytest.mark.parametrize("df", [1, 2, 4])
def test_avgpool_bit_exact(lib, device, df):
    """The kernel sums the df x df pixels in (dy, dx) order in fp32 and divides by df^2 (exact): bit for bit."""
    from grl_image_restoration_b200 import capi

    H, W, C = 16, 24, 36
    x = (torch.randn(B, H, W, C, generator=torch.Generator().manual_seed(df)) * 3).to(device)
    Ho, Wo = H // df, W // df
    out, buf = nan_rows(B * Ho * Wo, C, device)
    capi.check(lib.grl_avgpool_f32(ptr(x), ptr(out), B, H, W, C, df, stream()))
    torch.cuda.synchronize()
    check_written(buf, C, "output")
    xc = x.cpu().view(B, Ho, df, Wo, df, C)
    s = torch.zeros(B, Ho, Wo, C)
    for dy in range(df):
        for dx in range(df):
            s = s + xc[:, :, dy, :, dx]
    ref = (s / float(df * df)).reshape(-1, C)
    assert torch.equal(out.cpu(), ref), float((out.cpu() - ref).abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("heads", range(1, 9))
def test_bias_table(lib, device, heads):
    from grl_image_restoration_b200 import capi

    hidden = 512
    table = O.coords_table([32, 64], 2).reshape(-1, 2)  # 47 x 95 = 4465 rows: a partial last 128-row block
    rows = table.shape[0]
    g = torch.Generator().manual_seed(heads)
    w1, b1 = torch.randn(hidden, 2, generator=g) * 0.7, torch.randn(hidden, generator=g) * 0.1
    w2 = torch.randn(heads, hidden, generator=g) * 0.15
    dv = [t.float().to(device).contiguous() for t in (table, w1, b1, w2)]
    out, buf = nan_rows(heads, rows, device)
    capi.check(lib.grl_bias_table_f32(ptr(dv[0]), rows, ptr(dv[1]), ptr(dv[2]), ptr(dv[3]), hidden, heads, ptr(out),
                                      stream()))
    torch.cuda.synchronize()
    check_written(buf, rows, "table")
    bound, ref = bias_table_bound(*[t.double() for t in dv])
    ratio = bound_ratio(out, ref, bound)
    print(f"\n[fp32 bias table] heads={heads} hidden={hidden} rows={rows}: worst error / bound {ratio:.3f}")
    assert ratio <= 1.0, ratio


# --------------------------------------------------------------------------------------------- GPU: recorded launches


class Recorder:
    """Stands in for capi.lib(): records the fp32 GEMM and attention calls, forwards every call to the library."""

    def __init__(self, lib):
        self._lib, self.gemm, self.attn = lib, [], []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def grl_linear_f32(self, x, ldx, w, b, res, ldr, y, ldy, M, N, K, act, slope, st):
        self.gemm.append((False, K, N, act, slope, b is not None, res is not None))
        return self._lib.grl_linear_f32(x, ldx, w, b, res, ldr, y, ldy, M, N, K, act, slope, st)

    def grl_conv3x3_f32(self, x, w, b, res, y, Bn, H, W, Cin, Cout, act, slope, st):
        self.gemm.append((True, 9 * Cin, Cout, act, slope, b is not None, res is not None))
        return self._lib.grl_conv3x3_f32(x, w, b, res, y, Bn, H, W, Cin, Cout, act, slope, st)

    def grl_window_attn_f32(self, qkv, ldq, out, ldo, Bn, grid, heads, d, ls, bias, use_mask, st):
        self.attn.append(("window", grid_t(grid), grid_t(grid), heads, d, bool(use_mask)))
        return self._lib.grl_window_attn_f32(qkv, ldq, out, ldo, Bn, grid, heads, d, ls, bias, use_mask, st)

    def grl_stripe_attn_f32(self, qkv, ldq, anc, lda, out, ldo, Bn, tok, ancg, heads, d, s1, b1, s2, b2, use_mask, ws,
                            nbytes, st):
        self.attn.append(("stripe1", grid_t(ancg), grid_t(tok), heads, d, bool(use_mask)))
        self.attn.append(("stripe2", grid_t(tok), grid_t(ancg), heads, d, bool(use_mask)))
        return self._lib.grl_stripe_attn_f32(qkv, ldq, anc, lda, out, ldo, Bn, tok, ancg, heads, d, s1, b1, s2, b2,
                                             use_mask, ws, nbytes, st)


@pytest.mark.gpu
@pytest.mark.parametrize("variant,task,scale", [("tiny", "sr", 2), ("small", "jpeg", 1), ("base", "sr", 4),
                                                ("base", "dm", 1)])
def test_recorded_launches_match_lists(pkg, lib, device, monkeypatch, variant, task, scale):
    """The C-ABI calls of a real fp32 forward (smallest padded size, an input that needs padding) are, one for one and
    in order, the GEMM and attention launches f32_launches lists, and each one's path has a case."""
    from grl_image_restoration_b200 import capi, modules

    cfg = pkg.configs.grl_config(variant, task, scale)
    model = pkg.GRL(**dict(cfg, img_size=archs.smallest_size(cfg)))
    model.set_precision("fp32")
    model = model.to(device).eval()
    S = model.pad_size
    x = torch.rand(1, 3, S - 5, S - 3, generator=torch.Generator().manual_seed(0)).to(device)
    rec = Recorder(lib)
    monkeypatch.setattr(capi, "lib", lambda: rec)
    y = model(x)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert y.shape == (1, 3, (S - 5) * cfg["upscale"], (S - 3) * cfg["upscale"])
    launches = modules.f32_launches(model, tuple(x.shape))
    want_g = launches_of(launches, "GemmF32")
    assert len(rec.gemm) == len(want_g), (len(rec.gemm), len(want_g))
    for got, g in zip(rec.gemm, want_g):
        assert got == (g.conv, g.K, g.N, g.act, g.slope, g.bias, g.res), (g.name, got)
    gemm_have = {gemm_path(c.call()) for c in GEMM_CASES}
    assert all(gemm_path(g) in gemm_have for g in want_g)
    want_a = launches_of(launches, "AttnF32")
    assert len(rec.attn) == len(want_a), (len(rec.attn), len(want_a))
    attn_have = {attn_path(attn_case_launch(c)[1]) for c in ATTN_CASES}
    for got, ln in zip(rec.attn, want_a):
        assert got == (ln.role, grid_t(ln.gq), grid_t(ln.gk), ln.heads, ln.d, bool(ln.use_mask)), (ln.name, got)
        assert attn_path(ln) in attn_have, (got, attn_path(ln))
    print(f"\n{variant}/{task}x{scale}: {len(rec.gemm)} GEMM and {len(rec.attn)} attention launches match the list")


# ------------------------------------------------------------------------------------------------ listing mode


class HostOnly:
    """Stands in for capi.lib() during a listing run: host helpers (`*_host`) run, any other symbol raises."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        if not name.endswith("_host"):
            raise AssertionError(f"a listing run called {name}")
        self.calls.append(name)
        return getattr(self._lib, name)


@pytest.mark.parametrize("input_format", ["rgb", "rggb"])
def test_listing_calls_only_host_helpers(pkg, monkeypatch, input_format):
    """Listing a released config, at a resolution other than the model's own (so the coordinate tables are computed),
    makes no library call but the host helpers and never touches a CUDA stream."""
    from grl_image_restoration_b200 import capi, modules

    cfg = pkg.configs.grl_config("base", "dm", 1)
    model = pkg.GRL(input_format=input_format, **dict(cfg, img_size=archs.smallest_size(cfg)))
    S = model.pad_size
    shape = (2, 4, S // 2 + 3, S - 1) if input_format == "rggb" else (2, 3, S + 5, 2 * S - 1)
    host = HostOnly(capi.lib())
    monkeypatch.setattr(capi, "lib", lambda: host)

    def no_stream(*args, **kw):
        raise AssertionError("a listing run asked for a CUDA stream")

    monkeypatch.setattr(torch.cuda, "current_stream", no_stream)
    launches = modules.f32_launches(model, shape)
    monkeypatch.undo()
    assert set(host.calls) == {"grl_coords_table_host"}
    n_blocks = sum(len(layer.blocks) for layer in model.layers)
    assert len(launches_of(launches, "AttnF32")) == 3 * n_blocks
    assert len(launches_of(launches, "GemmF32")) == 7 * n_blocks + len(model.layers) + 3  # CAB: 2 convs per block


def test_fp32_and_tensor_core_listings_name_the_same_gemms(pkg):
    """Both paths run the same network: their listings name the same GEMMs in the same order, except that a tensor-core
    block runs its CAB convs before the output projection, whose LayerNorm epilogue adds the CAB branch."""
    from grl_image_restoration_b200 import modules, tc

    def no_cab(names):
        return [n for n in names if not n.endswith((".cab1", ".cab2"))]

    for (name, m32, shape), (_, m16, _) in zip(archs.architectures(pkg, "fp32"), archs.architectures(pkg, "fp16")):
        names16 = [ln.name for ln in tc.gemm_launches(m16, shape)]
        names32 = [g.name for g in launches_of(modules.f32_launches(m32, shape), "GemmF32")]
        assert sorted(names32) == sorted(names16), name
        assert no_cab(names32) == no_cab(names16), name


@pytest.mark.gpu
@pytest.mark.parametrize("task,input_format", [("sr", "rgb"), ("dm", "rggb")])
def test_listing_first_leaves_the_forward_unchanged(pkg, device, task, input_format):
    """f32_launches on a fresh fp32 model, then its forward: bitwise the forward of an identical model that was never
    listed.  A listing run packs conv weights on the device, but keeps no meta tensor a forward would use."""
    import copy

    from grl_image_restoration_b200 import modules

    cfg = pkg.configs.grl_config("tiny", task, 2 if task == "sr" else 1)
    cfg = dict(cfg, img_size=archs.smallest_size(cfg), input_format=input_format)
    torch.manual_seed(0)
    listed = pkg.GRL(**cfg)
    fresh = copy.deepcopy(listed)
    S = listed.pad_size
    shape = (1, 4, S // 2, S // 2 - 1) if input_format == "rggb" else (1, 3, S, S)
    x = torch.rand(shape, generator=torch.Generator().manual_seed(0)).to(device)
    ys = []
    for model, list_first in ((fresh, False), (listed, True)):
        model = model.to(device).eval()
        model.set_precision("fp32")
        if list_first:
            assert len(modules.f32_launches(model, tuple(x.shape))) > 0
        ys.append(model(x))
    torch.cuda.synchronize()
    assert torch.equal(ys[0], ys[1])
