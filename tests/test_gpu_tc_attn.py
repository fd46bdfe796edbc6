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

import pytest
import torch

import archs
import grl_oracle as O
from attn_cases import (B, CASES, EXTRAS, GATE_CHAIN, SENTINEL, ZOO_CASES, block_inputs, case_launch, check_pads, compare,
                        cpb_table, fails_gate, operand, path, run)
from support import grid_t

ATTN_VARIANTS = [5, 0]  # grl_tc_attn_variant: 5 = TMA boxes where the geometry has them (default), 0 = cp.async gathers


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


def old_bound_catches(m, exact, d):
    """The bound of the operator tests this file replaces: max-abs 4e-2 * max(1, |ref|), mean 6e-3."""
    err = (m[..., :d] - exact[..., :d]).abs()
    return bool(err.max() > 4e-2 * max(1.0, float(exact[..., :d].abs().max())) or err.mean() > 6e-3)


GATED = ("bias entry read from its neighbour", "shift mask missing for one region pair", "key box taken without the roll",
         "query box taken without the roll", "rescale applied to O only")
_REF = {}  # (case, fmt) -> float64 references, shared by both attention variants


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
