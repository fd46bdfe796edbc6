"""The released test commands' forward sizes (tests/command_cases.py), on the CPU: every configs.RELEASED checkpoint has a
command case, each case's forward size is what its evaluation.RECIPES entry makes of its image (crop, SR scale, packed
planes, tile), and at that size the forward takes the same launch paths as at archs.smallest_size, the size the
launch-path tests walk: the tensor-core GEMM (gemm_cases.path) and attention (attn_cases.path) signatures and the fp32
GEMM and attention signatures (f32_cases.gemm_path / attn_path), each set equal and each path with a case
(archs.check_walk)."""
import pytest
import torch

import archs
import attn_cases as A
import command_cases as CC
import f32_cases as C
import gemm_cases as G


def recipe_forward_size(pkg, ckpt, image):
    """(H, W) of the forward's input when the command `ckpt` reads an image of size `image`: the recipe's crop to
    multiples of the SR scale or of 8, the low-resolution file of the cropped ground truth (SR), the packed Bayer
    planes (dm), then a tiled command's t = min(tile, H, W)."""
    from grl_image_restoration_b200 import configs, evaluation

    r = evaluation.RECIPES[ckpt]
    scale = configs.RELEASED[ckpt][2]
    m = {"modcrop": scale, "mod8": 8, "none": 1}[r.crop]
    H, W = (v - v % m for v in image)
    if r.crop == "modcrop":
        H, W = H // scale, W // scale
    if r.input == "mosaic":
        H, W = H // 2, W // 2
    if r.tile:
        H = W = min(r.tile, H, W)
    return H, W


def test_every_released_checkpoint_has_a_command_case(pkg):
    missing = sorted(set(pkg.configs.RELEASED) - {c.ckpt for c in CC.CASES})
    assert not missing, f"released checkpoints without a command case: {missing}"
    unknown = sorted({c.ckpt for c in CC.CASES} - set(pkg.configs.RELEASED))
    assert not unknown, f"command cases of unknown checkpoints: {unknown}"
    assert len(CC.BY_NAME) == len(CC.CASES), "two command cases share a name"


@pytest.mark.parametrize("case", CC.CASES, ids=lambda c: c.name)
def test_case_size_follows_its_recipe(pkg, case):
    got = recipe_forward_size(pkg, case.ckpt, case.image)
    assert got == tuple(case.forward), f"{case.name}: the recipe makes a {got} forward of a {case.image} image"


def signatures(pkg, model16, model32, shape):
    """{family: {signature: first launch}} of one forward on a meta input of `shape`."""
    from grl_image_restoration_b200 import capi, modules, tc

    out = {"tc gemm": {}, "tc attention": {}, "fp32 gemm": {}, "fp32 attention": {}}
    for ln in tc.gemm_launches(model16, shape):
        out["tc gemm"].setdefault(G.path(ln), ln.name)
    h, w = shape[2:]
    if model16.input_format == "rggb":
        h, w = 2 * h, 2 * w
    p = model16.pad_size
    hp, wp = -(-h // p) * p, -(-w // p) * p
    for si, layer in enumerate(model16.layers):
        for bi, blk in enumerate(layer.blocks):
            for ln in tc.attention_launches(blk, (hp, wp)):
                out["tc attention"].setdefault(A.path(capi, ln), f"stage {si} block {bi} {ln.role}")
    launches = modules.f32_launches(model32, shape)
    for g in C.launches_of(launches, "GemmF32"):
        out["fp32 gemm"].setdefault(C.gemm_path(g), g.name)
    for a in C.launches_of(launches, "AttnF32"):
        out["fp32 attention"].setdefault(C.attn_path(a), f"{a.name} {a.role}")
    return out


def command_models(pkg, case):
    """(fp16 model, fp32 model) of the case's checkpoint, with the case's input format."""
    cfg = CC.cfg(pkg, case)
    kw = {"input_format": "rggb"} if CC.is_dm(pkg, case) else {}
    models = []
    for precision in ("fp16", "fp32"):
        m = pkg.GRL(**cfg, **kw)
        m.set_precision(precision)
        models.append(m)
    return models


def smallest_signatures(pkg, case):
    variant, task, scale, cin, _, _ = pkg.configs.RELEASED[case.ckpt]
    key = (variant, task, scale, cin if task in ("dn", "jpeg") else 3)
    (m16, shape), (m32, _) = archs.model(pkg, *key, "fp16"), archs.model(pkg, *key, "fp32")
    return signatures(pkg, m16, m32, shape)


def test_command_sizes_take_the_walked_paths(pkg):
    """Every command case's launch signatures equal those of its architecture at archs.smallest_size (the claim
    archs.py rests on), and every one has a launch-path case."""
    from grl_image_restoration_b200 import capi

    cases = {
        "tc gemm": [(G.path(G.case_launch(pkg, c)), c) for c in G.CASES + G.EXTRA_NAMES],
        "tc attention": [(A.path(capi, A.case_launch(c)[1]), c) for c in A.CASES + A.EXTRAS + A.ZOO_CASES],
        "fp32 gemm": [(C.gemm_path(c.call()), c) for c in C.GEMM_CASES + C.GEMM_ZOO_CASES + C.GEMM_EXTRAS],
        "fp32 attention": [(C.attn_path(C.attn_case_launch(c)[1]), c)
                           for c in C.ATTN_CASES + C.ATTN_ZOO_CASES + C.ATTN_EXTRAS],
    }
    launched = {fam: [] for fam in cases}
    differ = []
    with torch.no_grad():
        for case in CC.CASES:
            m16, m32 = command_models(pkg, case)
            got = signatures(pkg, m16, m32, CC.input_shape(pkg, case))
            want = smallest_signatures(pkg, case)
            for fam, sigs in got.items():
                launched[fam] += [(s, f"{case.name} {first}") for s, first in sigs.items()]
                new, gone = set(sigs) - set(want[fam]), set(want[fam]) - set(sigs)
                if new or gone:
                    differ.append(f"{case.name} {fam}: {len(new)} paths only at the command size "
                                  f"({[sigs[s] for s in new]}), {len(gone)} only at the smallest size")
    print(f"{len(CC.CASES)} command cases: " + ", ".join(f"{len(set(s for s, _ in v))} {fam} paths"
                                                          for fam, v in launched.items()))
    for fam, ln in launched.items():
        archs.check_walk(f"{fam} (command sizes)", ln, [], cases[fam])
    assert not differ, "; ".join(differ)
