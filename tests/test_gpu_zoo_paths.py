"""Launch-path coverage of every released checkpoint (configs.RELEASED): the tensor-core GEMM and attention kernels and the
fp32 kernels, with the paths and cases of test_gpu_tc_gemm.py, test_gpu_tc_attn.py and test_gpu_f32_paths.py.

Those files walk the architectures of configs.grl_config's first tasks with 3 input channels.  The walks here build each
RELEASED entry with its own in_channels (1 for grayscale dn / jpeg, 6 for dual-pixel defocus) at its smallest padded
size and list its launches the same way: tc.gemm_launches, tc.attention_launches per block, modules.f32_launches.
Every path must have a case in the existing files or in the NEW_* lists below, and every new case must be a path a
released config launches that no existing case covers.  The new cases run through the existing GPU tests unchanged
(their float64 references, gates, both attention operand loaders, fp16 and bf16, and the mutation controls that apply),
as extras of those tests' case lists.
"""
import math
from functools import lru_cache

import pytest

import test_gpu_f32_paths as F
import test_gpu_tc_attn as A
import test_gpu_tc_gemm as G
from test_gpu_f32_paths import lib  # noqa: F401  (fixture)
from test_gpu_tc_attn import tc  # noqa: F401  (fixture: once per attention operand loader)

# tensor-core attention: GRL-Base blind SR's stripe pass 1 over 64 x 32 stripes with df 4 (16 x 8 anchor windows)
NEW_TC_ATTN = [
    A.AttnCase("base/bsr/b1", "stripe1", (64, 32), 4, False, 3, 30),
    A.AttnCase("base/bsr/b3", "stripe1", (64, 32), 4, True, 3, 30),
]
# fp32 attention: the same pass in the fp32 kernel's signature (Base head_dim 30 on 8 x 16 anchors, 2048 keys)
NEW_F32_ATTN = [
    F.AttnCase("base/bsr", "stripe1", (32, 64), 4, False, 3, 30),
    F.AttnCase("base/bsr", "stripe1", (32, 64), 4, True, 3, 30),
]
# fp32 GEMM: 1- and 6-channel heads, the 3-channel tail without the input residual, the nearest+conv head's convs
NEW_F32_GEMM = [
    F.GemmCase("tiny/dnx1 c1 conv_first", True, 9, 64),
    F.GemmCase("small/dnx1 c1 conv_first", True, 9, 128),
    F.GemmCase("base/dnx1 c1 conv_first", True, 9, 180),
    F.GemmCase("base/bsrx4 conv_up1", True, 576, 64, F.ACT_LEAKY, slope=0.2),
    F.GemmCase("base/defocus_dual conv_first", True, 54, 180),
    F.GemmCase("base/defocus_dual conv_last", True, 1620, 3),
]


@lru_cache(maxsize=None)
def released_model(pkg, variant, task, upscale, cin, precision):
    """A RELEASED architecture at its smallest padded size, with the input shape of one such image."""
    cfg = pkg.configs.grl_config(variant, task, upscale, in_channels=cin if task in ("dn", "jpeg") else 3)
    S = math.lcm(cfg["window_size"], *cfg["stripe_size"])
    model = pkg.GRL(**dict(cfg, img_size=S))
    model.set_precision(precision)
    return model, (1, model.in_channels, S, S)


def released(pkg, precision):
    """(checkpoint name, model, input shape) of every architecture in RELEASED, once each."""
    seen = set()
    for name, (variant, task, upscale, cin, _, _) in pkg.configs.RELEASED.items():
        key = (variant, task, upscale, cin)
        if key not in seen:
            seen.add(key)
            yield (name, *released_model(pkg, *key, precision))


def check_walk(what, launched, existing, new):
    """launched: (path, first launcher) pairs; existing / new: path -> case.  No path without a case, no new case that
    is not launched or that an existing case already covers."""
    paths = {}
    for s, name in launched:
        paths.setdefault(s, name)
    missing = {s: n for s, n in paths.items() if s not in existing and s not in new}
    for s, n in missing.items():
        print(f"{what} path without a case: {s}, first launched by {n}")
    stale = [c for s, c in new.items() if s not in paths]
    dup = [c for s, c in new.items() if s in existing]
    print(f"{what}: {len(paths)} released paths, {len(new)} new cases, {len(missing)} without a case, "
          f"{len(stale)} stale")
    assert not missing, f"{len(missing)} released {what} paths have no case: {missing}"
    assert not stale, f"new {what} cases that no released config launches: {stale}"
    assert not dup, f"new {what} cases that an existing case already covers: {dup}"


def test_released_zoo_tc_gemm_paths_have_cases(pkg):
    from grl_image_restoration_b200 import tc as T

    existing = {G.path(G.case_launch(pkg, c)): c for c in G.CASES + G.EXTRA_NAMES}
    launched = [(G.path(ln), f"{name} {ln.name}") for name, m, shape in released(pkg, "fp16")
                for ln in T.gemm_launches(m, shape)]
    check_walk("tensor-core gemm", launched, existing, {})


def test_released_zoo_tc_attention_paths_have_cases(pkg):
    from grl_image_restoration_b200 import capi, tc as T

    existing = {A.path(capi, A.case_launch(c)[1]): c for c in A.CASES + A.EXTRAS}
    new = {A.path(capi, A.case_launch(c)[1]): c for c in NEW_TC_ATTN}
    assert len(new) == len(NEW_TC_ATTN), "two new cases share a path"
    launched = [(A.path(capi, ln), f"{name} stage {si} block {bi} {ln.role}") for name, m, shape in released(pkg, "fp16")
                for si, layer in enumerate(m.layers) for bi, blk in enumerate(layer.blocks)
                for ln in T.attention_launches(blk, shape[2:])]
    check_walk("tensor-core attention", launched, existing, new)


def test_released_zoo_f32_paths_have_cases(pkg):
    from grl_image_restoration_b200 import modules

    lists = [(name, modules.f32_launches(m, shape)) for name, m, shape in released(pkg, "fp32")]
    existing = {F.attn_path(F.attn_case_launch(c)[1]): c for c in F.ATTN_CASES}
    new = {F.attn_path(F.attn_case_launch(c)[1]): c for c in NEW_F32_ATTN}
    assert len(new) == len(NEW_F32_ATTN), "two new cases share a path"
    check_walk("fp32 attention", [(F.attn_path(ln), f"{n} {ln.name} {ln.role}") for n, ls in lists
                                  for ln in F.launches_of(ls, "AttnF32")], existing, new)
    existing = {F.gemm_path(c.call()): c for c in F.GEMM_CASES + F.GEMM_EXTRAS}
    new = {F.gemm_path(c.call()): c for c in NEW_F32_GEMM}
    assert len(new) == len(NEW_F32_GEMM), "two new cases share a path"
    check_walk("fp32 gemm", [(F.gemm_path(g), f"{n} {g.name}") for n, ls in lists for g in F.launches_of(ls, "GemmF32")],
               existing, new)


# ----------------------------------------------------------------------------------------------------------------- GPU


def tc_attn_id(c):
    return f"{c.src}-{c.role}-{c.win[0]}x{c.win[1]}-df{c.df}-{'s' if c.shifted else 'u'}-h{c.heads}d{c.d}".replace("/", "-")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", NEW_TC_ATTN, ids=tc_attn_id)
def test_zoo_tc_attention_path(tc, device, monkeypatch, case, fmt):  # noqa: F811
    monkeypatch.setattr(A, "EXTRAS", A.EXTRAS + NEW_TC_ATTN)  # the case's seed is its index in CASES + EXTRAS
    A.test_attention_path(tc, device, case, fmt)


@pytest.mark.gpu
@pytest.mark.parametrize("case", NEW_F32_ATTN, ids=F.attn_id)
def test_zoo_f32_attention_path(lib, device, monkeypatch, case):  # noqa: F811
    monkeypatch.setattr(F, "ATTN_EXTRAS", F.ATTN_EXTRAS + NEW_F32_ATTN)
    F.test_attention_path(lib, device, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", NEW_F32_GEMM, ids=F.gemm_id)
def test_zoo_f32_gemm_path(lib, device, monkeypatch, case):  # noqa: F811
    monkeypatch.setattr(F, "GEMM_EXTRAS", F.GEMM_EXTRAS + NEW_F32_GEMM)
    F.test_gemm_path(lib, device, case)
