"""The tensor-core GEMM / conv kernel and the attention kernel at the sizes the benchmark launches them, against float64,
and the batch composition of the tensor-core and fp32 forwards, bit for bit.

test_gpu_tc_gemm.py and test_gpu_tc_attn.py run one small instance of every launch path (B = 2, a few dozen CTAs at
most), on the claim that the image size does not enter a launch's path.  This file runs the launches of the benchmark's
workloads at their real size: grids of thousands of CTAs (several waves of two CTAs per SM on 132 SMs), the benchmark's
micro-batch of 16 images, and the non-square window grids of the stripe passes of cfg3 (4 x 2) and cfg5 (10 x 5).

Workloads are read from bench.py's text (WORKLOADS, MICRO_BATCH, CFG5_*; importing bench.py would redirect stdout).  One
launch's batch is min(tiles per GPU, MICRO_BATCH); cfg5 runs the 6 tiles of its frame in one batch, as one GPU does.
Operands follow the seeded recipes of the small-size tests (gemm_cases.instantiate, attn_cases.block_inputs)
at the production batch and image size, and use the same gates.

  GEMM: each distinct launch of tc.gemm_launches (its name modulo the stage / block index) runs on the whole batch;
    every owned element must be written, pads exactly 0 and the guard rows untouched.  Images 0, B // 2 and B - 1 (the
    first, a middle and the last wave of CTAs) are compared with float64; conv and linear rows are image-local, so that
    is exact.
  Attention: each distinct launch of tc.attention_launches (window; stripe pass 1 and 2 through X1) runs on the whole
    batch with the default loader (variant 5); no output slot may keep its sentinel and nothing outside the slots may be
    written.  Every window of images 0 and B - 1 and 32 seeded windows elsewhere are compared with the float64
    emulation; stripe pass 2 also along the chain with the emulated X1.
Mutation controls, derived from the reference (a kernel bug's effect, never an edited kernel), that only show at this
size: a conv halo taken from the vertically adjacent image (a tensor map that merges B and H), every LayerNorm + CAB row
taking image 0's gate, the last image attending to image 0's keys and values, and the window grid decomposed with nwh and
nww swapped (visible on non-square grids only).  Each must fail the gate wherever it applies.

Each GPU test prints its time and peak device memory.
"""
import ast
import os
import re
import time
from functools import lru_cache

import pytest
import torch

import grl_oracle as O
import attn_cases as A
import gemm_cases as G
from support import grid_t

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100_SMS = 132
CTAS_PER_SM = 2  # both kernels are built for two resident CTAs per SM
RUNS = [("cfg4", "fp16"), ("cfg4", "bf16"), ("cfg2", "fp16"), ("cfg3", "fp16"), ("cfg1", "fp16"), ("cfg5", "fp16")]
EXTRA_WINDOWS = 32  # seeded windows outside the first and the last image in the float64 attention check


def bench_constants():
    """WORKLOADS, MICRO_BATCH and CFG5_* as bench.py assigns them, from its syntax tree."""
    with open(os.path.join(ROOT, "bench.py")) as f:
        tree = ast.parse(f.read())
    want = {"WORKLOADS", "MICRO_BATCH", "CFG5_FRAME", "CFG5_TILE", "CFG5_OVERLAP"}
    out = {}
    for node in tree.body:
        if not (isinstance(node, ast.Assign) and len(node.targets) == 1):
            continue
        t = node.targets[0]
        names = [t.id] if isinstance(t, ast.Name) else [e.id for e in getattr(t, "elts", []) if isinstance(e, ast.Name)]
        if want.isdisjoint(names):
            continue
        value = ast.literal_eval(node.value)
        out.update({names[0]: value} if len(names) == 1 else dict(zip(names, value)))
    return out


BENCH = bench_constants()


def frame_tiles():
    from grl_image_restoration_b200 import tiling

    (h, w), tile, overlap = BENCH["CFG5_FRAME"], BENCH["CFG5_TILE"], BENCH["CFG5_OVERLAP"]
    return len(tiling.tile_origins(h, tile, overlap)) * len(tiling.tile_origins(w, tile, overlap))


def batch_of(name):
    """Images per launch of a workload on one GPU."""
    per_gpu = BENCH["WORKLOADS"][name][4]
    return frame_tiles() if name == "cfg5" else min(per_gpu, BENCH["MICRO_BATCH"])


def picks(n):
    """Images compared with float64: the first, a middle and the last."""
    return sorted({0, n // 2, n - 1})


@lru_cache(maxsize=None)
def workload_model(pkg, name, precision):
    """(model on the host, input shape of one launch) of a workload, at bench's tile size."""
    variant, task, scale, tile = BENCH["WORKLOADS"][name][:4]
    m = pkg.GRL(**pkg.configs.grl_config(variant, task, scale, tile))
    assert m.set_precision(precision) == precision
    return m, (batch_of(name), m.in_channels, tile, tile)


def distinct_gemm_launches(tc, model, shape):
    """The first launch of each name modulo the stage / block index."""
    out = {}
    for ln in tc.gemm_launches(model, shape):
        out.setdefault(re.sub(r"(stage|block)\d+", r"\1#", ln.name), ln)
    return list(out.values())


def distinct_attention_units(tc, model, shape):
    """(block, launches) per distinct window launch and per distinct stripe pass pair (pass 1, pass 2)."""
    out = {}
    for layer in model.layers:
        for blk in layer.blocks:
            w, s1, s2 = tc.attention_launches(blk, shape[2:])
            for lns in ((w,), (s1, s2)):
                key = tuple((ln.role, grid_t(ln.gq), grid_t(ln.gk), ln.heads, ln.use_mask, ln.ones_col) for ln in lns)
                out.setdefault(key, (blk, lns))
    return list(out.values())


def window_grid(g):
    return g.H // g.wh, g.W // g.ww


def attn_ctas(ln, batch):
    nwh, nww = window_grid(ln.gq)
    return batch * nwh * nww * ln.heads * -(-(ln.gq.wh * ln.gq.ww) // O.ATTN_Q_TILE)


# ----------------------------------------------------------------------------------------------------------------- CPU


def test_workloads_from_bench(pkg):
    """The workload table parsed from bench.py has the expected entries, and every workload resolves to a model that
    runs the tensor-core path at bench's `auto` precision."""
    assert set(BENCH["WORKLOADS"]) == {"cfg1", "cfg2", "cfg3", "cfg4", "cfg5"}
    assert {n: batch_of(n) for n in BENCH["WORKLOADS"]} == {"cfg4": 16, "cfg2": 16, "cfg3": 8, "cfg1": 1, "cfg5": 6}
    assert BENCH["CFG5_TILE"] == BENCH["WORKLOADS"]["cfg5"][3]
    for name in BENCH["WORKLOADS"]:
        model, shape = workload_model(pkg, name, "fp16")
        assert model.pad_size and shape[2] % model.pad_size == 0, name
        variant, task, scale, tile = BENCH["WORKLOADS"][name][:4]
        assert pkg.GRL(**pkg.configs.grl_config(variant, task, scale, tile)).set_precision("auto") == "fp16", name


def test_production_paths_are_gated(pkg):
    """Every launch this file runs takes a path the small-size tests already gate: this file is about size only.  The
    attention inputs assume as many window heads as stripe heads (the packed layout of test_gpu_tc_attn)."""
    from grl_image_restoration_b200 import capi, tc

    gemm_have = {G.path(G.case_launch(pkg, c)) for c in G.ALL_CASES}
    attn_have = {A.path(capi, A.case_launch(c)[1]) for c in A.CASES + A.EXTRAS + A.ZOO_CASES}
    for name, precision in RUNS:
        model, shape = workload_model(pkg, name, precision)
        for ln in distinct_gemm_launches(tc, model, shape):
            assert G.path(ln) in gemm_have, (name, ln.name, G.path(ln))
        for blk, lns in distinct_attention_units(tc, model, shape):
            assert blk.attn.window_attn.num_heads == blk.attn.stripe_attn.num_heads, name
            for ln in lns:
                assert A.path(capi, ln) in attn_have, (name, ln.role, A.path(capi, ln))


def test_launches_span_waves_and_non_square_grids(pkg):
    """At least one GEMM and one attention launch have more CTAs than 132 SMs hold at two per SM, and at least one
    attention launch has a non-square window grid."""
    from grl_image_restoration_b200 import tc

    gemm_grid = attn_grid = 0
    non_square = []
    for name, precision in RUNS:
        model, shape = workload_model(pkg, name, precision)
        gemm_grid = max([gemm_grid] + [tc.gemm_path(ln).grid for ln in distinct_gemm_launches(tc, model, shape)])
        for _, lns in distinct_attention_units(tc, model, shape):
            attn_grid = max([attn_grid] + [attn_ctas(ln, shape[0]) for ln in lns])
            non_square += [(name, ln.role, window_grid(ln.gq)) for ln in lns if len(set(window_grid(ln.gq))) > 1]
    print(f"largest grids: GEMM {gemm_grid} CTAs, attention {attn_grid} CTAs; non-square window grids: {non_square}")
    assert gemm_grid > CTAS_PER_SM * H100_SMS and attn_grid > CTAS_PER_SM * H100_SMS
    assert non_square


# ----------------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def tc(pkg, device):
    from grl_image_restoration_b200 import capi, tc as T

    if capi.lib().grl_device_ok() != 1:
        pytest.skip("wgmma path needs sm_90")
    prev = capi.lib().grl_tc_attn_variant(5)
    yield T
    capi.lib().grl_tc_attn_variant(prev)


@pytest.fixture
def measured(device):
    """Prints the test's wall time and peak device memory."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(device)
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n  time {time.perf_counter() - t0:.1f} s, peak memory {torch.cuda.max_memory_allocated(device) / 2 ** 30:.2f} GiB "
          f"allocated ({torch.cuda.get_device_name(device)})")
    torch.cuda.empty_cache()


def run_id(r):
    return f"{r[0]}-{r[1]}"


def merge(total, res):
    """Worst statistic and joint verdict per gate over images."""
    for what, (s, ok) in res.items():
        if what in total:
            s0, ok0 = total[what]
            s = tuple(map(max, s0, s)) if isinstance(s, tuple) else max(s0, s)
            ok = ok and ok0
        total[what] = (s, ok)
    return total


def gemm_image(run, b, conv, L):
    """(float64-reference operands, kernel outputs, first row) of image b of a GEMM run."""
    o = dict(run.ops)
    rows = slice(b, b + 1) if conv else slice(b * L, (b + 1) * L)
    for k in ("x", "res", "cab_y"):
        if k in o:
            o[k] = o[k][rows]
    if "cab_gate" in o:
        o["cab_gate"] = o["cab_gate"][b:b + 1]
    got = {k: view[b:b + 1] if conv or k == "out_nchw" else view[rows] for k, (view, _) in run.bufs.items()}
    return o, got, 0 if conv else b * L


def gemm_reference(o, bn, mutation=None):
    o = dict(o)
    return O.gemm_launch_reference(o.pop("x"), o.pop("w"), o.pop("bias"), bn=bn, mutation=mutation, **o)


def halo_reference(run, b, bn):
    """The conv of image b with its halo rows taken from the vertically adjacent images, as if the batch were one tall
    image: what a tensor map that merges B and H loads."""
    o = dict(run.ops)
    x = o["x"]
    n, H, W, _ = x.shape
    top = 1 if b > 0 else 0

    def tall(t):
        parts = ([t[b - 1, -1:]] if b > 0 else []) + [t[b]] + ([t[b + 1, :1]] if b + 1 < n else [])
        return torch.cat(parts, 0)[None]

    o["x"] = tall(x)
    if "res" in o:
        o["res"] = tall(o["res"])
    Ht = o["x"].shape[1]
    if "crop" in o:
        o["crop"] = (Ht * o["nchw_r"], W * o["nchw_r"])
    ref = gemm_reference(o, bn)
    out = {"y": ref["y"][top * W:(top + H) * W]}
    if "ps" in ref:
        r = o["ps_r"]
        out["ps"] = ref["ps"][:, top * r:(top + H) * r]
    if "nchw" in ref:
        r, crop = o["nchw_r"], run.ops["crop"]
        out["nchw"] = ref["nchw"][:, :, top * r:(top + H) * r][:, :, :crop[0], :crop[1]]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("workload", RUNS, ids=run_id)
def test_gemm_at_scale(pkg, tc, device, measured, workload):
    name, precision = workload
    fmt = tc.FMT[precision]
    model, shape = workload_model(pkg, name, precision)
    Bn = shape[0]
    n_sm = torch.cuda.get_device_properties(device).multi_processor_count
    failed, missed = [], []
    for i, launch in enumerate(distinct_gemm_launches(tc, model, shape)):
        a = launch.args
        conv = a["taps"] == 9
        L = 1 if conv else a["M"] // Bn
        assert conv or a["M"] == Bn * L
        size = tuple(a["image"][1:]) if conv else (G.HT, G.WT)
        run = G.instantiate(tc, launch, fmt, device, seed=1000 + 100 * RUNS.index(workload) + i, batch=Bn, size=size, L=L)
        assert run.sig == G.path(launch), (launch.name, run.sig)
        q = tc.gemm_path(launch)
        tc.gemm(**run.kw)
        torch.cuda.synchronize()
        G.check_buffers(tc, run, fmt, q.epi_mode)
        res = {}
        for b in picks(Bn):
            o, got, row0 = gemm_image(run, b, conv, L)
            merge(res, G.evaluate(tc, run, got, gemm_reference(o, q.bn), fmt, row0))
        print(f"\n[{name} {precision}] {launch.name} B={Bn} {'image ' + 'x'.join(map(str, size)) if conv else f'L={L}'}: "
              f"grid {q.grid} CTAs = {q.grid / (CTAS_PER_SM * n_sm):.1f} waves of {CTAS_PER_SM} x {n_sm}; images "
              f"{picks(Bn)} vs float64")
        for what, (s, ok) in res.items():
            print(f"  {what}: {s} {'ok' if ok else 'FAILS'}")
        if not all(ok for _, ok in res.values()):
            failed.append((launch.name, res))

        muts = {}
        if conv and Bn > 1:
            muts["conv halo from the adjacent image"] = [(b, halo_reference(run, b, q.bn)) for b in picks(Bn)]
        elif conv:
            print("  mutation 'conv halo from the adjacent image': does not apply (one image)")
        if a["epi"] == tc.EPI_LN and a["cab_y"] is not None:
            if Bn > 1:
                refs = []
                for b in picks(Bn)[1:]:
                    o = dict(gemm_image(run, b, conv, L)[0], cab_gate=run.ops["cab_gate"][:1])
                    refs.append((b, gemm_reference(o, q.bn)))
                muts["every row takes image 0's CAB gate"] = refs
            else:
                print("  mutation 'every row takes image 0's CAB gate': does not apply (one image)")
        for mname, refs in muts.items():
            mres = {}
            for b, mref in refs:
                o, got, row0 = gemm_image(run, b, conv, L)
                merge(mres, G.evaluate(tc, run, got, mref, fmt, row0))
            caught = not all(ok for _, ok in mres.values())
            print(f"  mutation '{mname}': {'FAILS the gate' if caught else 'passes the gate'} "
                  f"{ {k: v[0] for k, v in mres.items()} }")
            if not caught:
                missed.append((launch.name, mname))
        del run
        torch.cuda.empty_cache()
    assert not failed, failed
    assert not missed, f"mutations the gate does not catch: {missed}"


def window_subset(Bn, nW, seed, device):
    """Every window of the first and the last image and EXTRA_WINDOWS seeded windows of the others (kernel order)."""
    ends = torch.cat([torch.arange(nW), torch.arange((Bn - 1) * nW, Bn * nW)]).unique()
    rest = torch.arange(nW, max(nW, (Bn - 1) * nW))
    g = torch.Generator().manual_seed(seed)
    extra = rest[torch.randperm(rest.numel(), generator=g)[:EXTRA_WINDOWS]]
    return torch.cat([ends, extra]).sort().values.to(device)


def transposed_mutation(emul, sel, ln, dense, sentinel):
    """The emulated output of a kernel that decomposes the window index with nwh and nww swapped: CTA w works on window
    (w // nwh, w % nwh).  A dense output (X1) slot w then holds that window (where it lies in the grid; elsewhere the
    effect is not modelled); a strided output keeps its previous value at every window no CTA maps to.  None where the
    swap changes nothing (a square grid)."""
    nwh, nww = window_grid(ln.gq)
    if nwh == nww:
        return None
    nW = nwh * nww
    w = sel % nW
    r, c = w // nwh, w % nwh
    out = emul.clone()
    if dense:
        pos = {int(s): j for j, s in enumerate(sel)}
        for j in range(sel.numel()):
            src = int(sel[j]) - int(w[j]) + int(r[j]) * nww + int(c[j])
            if r[j] < nwh and c[j] < nww and src in pos:
                out[j] = emul[pos[src]]
    else:
        wr, wc = w // nww, w % nww
        out[(wr >= nww) | (wc >= nwh)] = sentinel
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("workload", RUNS, ids=run_id)
def test_attention_at_scale(pkg, tc, device, measured, workload):
    name, precision = workload
    fmt = tc.FMT[precision]
    dtype = tc.DTYPE[fmt]
    model, shape = workload_model(pkg, name, precision)
    Bn, (H, W) = shape[0], shape[2:]
    n_sm = torch.cuda.get_device_properties(device).multi_processor_count
    sentinel = torch.tensor(A.SENTINEL, dtype=dtype).double().item()
    failed, missed = [], []
    for u, (blk, lns) in enumerate(distinct_attention_units(tc, model, shape)):
        h = lns[-1].heads
        d = blk.dim // 2 // h
        s2 = lns[-1]
        df = s2.gq.wh // s2.gk.wh if s2.role == "stripe2" else blk.attn.anchor.body[0].down_factor
        seed = 2000 + 100 * RUNS.index(workload) + u
        case = A.AttnCase(f"{name}", s2.role, (s2.gq.wh, s2.gq.ww), df, s2.use_mask, h, d)
        qkv, anc = A.block_inputs(case, (H, W), dtype, device, seed, batch=Bn)
        merged = torch.full((Bn * H * W, 2 * h * 32), A.SENTINEL, device=device, dtype=dtype)
        buf = {"qkv": qkv, "anchor": anc, "merged": merged}
        if s2.role == "stripe2":
            ag = lns[0].gq
            buf["x1"] = torch.full((Bn * (ag.H // ag.wh) * (ag.W // ag.ww) * h * ag.wh * ag.ww, 32), A.SENTINEL,
                                   device=device, dtype=dtype)
        tables = {ln.role: A.cpb_table(ln, seed + 10 * k) for k, ln in enumerate(lns)}
        for ln in lns:
            A.run(tc, ln, buf, tables[ln.role], batch=Bn)
        torch.cuda.synchronize()

        # the whole output: every slot written, pads and ones column right, nothing outside the slots
        for ln in lns:
            out = A.operand(buf, ln.out, ln.gq, h, batch=Bn)
            assert not bool((out[..., :d] == A.SENTINEL).any()), f"{ln.role}: an output slot was not written"
            assert bool(out[..., :d].isfinite().all()), f"{ln.role}: non-finite output"
            A.check_pads(out, ln, d, ln.role)
        other = 1 if lns[0].role == "window" else 0
        assert bool((merged.view(Bn * H * W, 2, h * 32)[:, other] == A.SENTINEL).all()), "wrote outside its output slots"

        nW = (lns[0].gq.H // lns[0].gq.wh) * (lns[0].gq.W // lns[0].gq.ww)
        sel = window_subset(Bn, nW, seed, device)
        last = (sel // nW == Bn - 1).nonzero().flatten() if Bn > 1 else None
        first = {int(s): j for j, s in enumerate(sel) if s < nW}
        emulated = {}  # role -> emulated output on the subset (pass 1: the chain's X1)
        for ln in lns:
            index, mask = O.attn_pair_geometry(grid_t(ln.gq), grid_t(ln.gk), ln.use_mask)
            index, mask = index.to(device), None if mask is None else mask.to(device)[sel % nW]
            q, k, v = (A.operand(buf, s, g, h, batch=Bn)[sel] for s, g in ((ln.q, ln.gq), (ln.k, ln.gk), (ln.v, ln.gk)))
            got = A.operand(buf, ln.out, ln.gq, h, batch=Bn)[sel]

            def ref(q, k, v, mask):
                return O.attn_launch_reference(q, k, v, tables[ln.role], index, mask, dtype)

            exact, emul, info = ref(q, k, v, mask)
            emulated[ln.role] = emul
            stats = A.compare(got, emul, d, dtype)
            nwh, nww = window_grid(ln.gq)
            ctas = attn_ctas(ln, Bn)
            print(f"\n[{name} {precision}] {ln.role} {grid_t(ln.gq)} <- {grid_t(ln.gk)} h{h} d{d} mask={ln.use_mask} "
                  f"B={Bn}: window grid {nwh} x {nww}, {ctas} CTAs = {ctas / (CTAS_PER_SM * n_sm):.1f} waves; "
                  f"{sel.numel()} of {Bn * nW} windows vs float64: |got-emulated| {stats[0]:.2f} ulp (gate {A.GATE_ULP}), "
                  f"mismatch {stats[1]:.4f}, |emulated-exact| {float((emul - exact)[..., :d].abs().max()):.2e}, "
                  f"rescales {info['rescales']}")
            if A.fails_gate(stats):
                failed.append((ln.role, stats))
            if ln.role == "stripe2":
                _, em_c, _ = ref(q, k, emulated["stripe1"], mask)
                sc = A.compare(got, em_c, d, dtype)
                print(f"  chain vs chained emulation: {sc[0]:.2f} ulp (gate {A.GATE_CHAIN}), mismatch {sc[1]:.4f}")
                if sc[0] > A.GATE_CHAIN:
                    failed.append(("chain", sc))

            muts = {}
            if last is not None:
                src = torch.tensor([first[int(s) - (Bn - 1) * nW] for s in sel[last]], device=device)
                m_last = ref(q[last], k[src], v[src], None if mask is None else mask[last])[1]
                muts["the last image reads image 0's keys and values"] = (got[last], m_last)
            else:
                print("  mutation 'the last image reads image 0's keys and values': does not apply (one image)")
            m_t = transposed_mutation(emul, sel, ln, ln.o_dense, sentinel)
            if m_t is not None:
                muts["window grid decomposed transposed"] = (got, m_t)
            else:
                print(f"  mutation 'window grid decomposed transposed': does not apply (square {nwh} x {nww} grid)")
            for mname, (g_m, m_emul) in muts.items():
                ms = A.compare(g_m, m_emul, d, dtype)
                print(f"  mutation '{mname}': {ms[0]:.2f} ulp -> {'FAILS the gate' if A.fails_gate(ms) else 'passes the gate'}")
                if not A.fails_gate(ms):
                    missed.append((ln.role, mname))
        del qkv, anc, merged, buf
        torch.cuda.empty_cache()
    assert not failed, failed
    assert not missed, f"mutations the gate does not catch: {missed}"


@lru_cache(maxsize=1)
def bench_model(pkg, name, device):
    """A workload's model with bench's seeded weights, on the device (one at a time)."""
    variant, task, scale, tile = BENCH["WORKLOADS"][name][:4]
    cfg = pkg.configs.grl_config(variant, task, scale, tile)
    m = pkg.GRL(**cfg)
    m.load_state_dict(O.synth_state_dict(cfg, seed=0, style="init"), strict=False)
    return m.to(device).eval()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp16", "bf16", "fp32"])
@pytest.mark.parametrize("name", ["cfg2", "cfg3", "cfg4", "cfg5"])
def test_batch_composition_bitwise(pkg, device, measured, name, precision):
    """One forward of the benchmark's batch: images 0, B // 2 and B - 1 are each bit for bit the forward of that image
    alone.  Rows, pixel patches, windows and CAB chunks are image-local, and at these sizes every image's rows fill
    whole 128-row tiles, except the anchor rows of cfg5 (120 x 120 per image), where rows of two images share a tile:
    there equality also needs a wgmma row's result not to depend on its position in the tile, which it does not."""
    model = bench_model(pkg, name, device)
    model.use_cuda_graph = False
    assert model.set_precision(precision) == precision
    variant, task, scale, tile, _, _, sigma = BENCH["WORKLOADS"][name]
    Bn = batch_of(name)
    g = torch.Generator().manual_seed(1234)
    x = torch.rand(Bn, 3, tile, tile, generator=g)
    if sigma > 0:
        x = x + (sigma / 255.0) * torch.randn(x.shape, generator=g)
    x = x.to(device)
    y = model(x)
    differ = []
    for b in picks(Bn):
        yb = model(x[b:b + 1])
        same = torch.equal(yb[0], y[b])
        print(f"\n[{name} {precision}] B={Bn}: image {b} of the batch == its B = 1 forward: {same}"
              + ("" if same else f" (max |diff| {float((yb[0] - y[b]).abs().max()):.3e})"))
        if not same:
            differ.append(b)
    assert not differ, f"images {differ} of the batch differ from their B = 1 forward"
