"""The architectures the launch-path tests walk (test_gpu_tc_gemm.py, test_gpu_tc_attn.py, test_gpu_f32_paths.py): every
configs.RELEASED entry with its own in_channels, and every grl_config of the VARIANTS x TASKS grid (which also holds
architectures without a released checkpoint, such as GRL-Tiny deblurring).  Each is built once per precision, at the
smallest size its windows and stripes tile: any size they tile gives the same launch paths (test_command_paths.py checks
this at the sizes the released test commands run)."""
import math
from functools import lru_cache

VARIANTS = ("tiny", "small", "base")
TASKS = (("sr", 2), ("sr", 3), ("sr", 4), ("dn", 1), ("deblur", 1), ("jpeg", 1), ("dm", 1))


def smallest_size(cfg):
    return math.lcm(cfg["window_size"], *cfg["stripe_size"])


@lru_cache(maxsize=None)
def model(pkg, variant, task, scale, in_channels, precision):
    """(model, input shape): grl_config(variant, task, scale, in_channels) at its smallest size, one image of it."""
    cfg = pkg.configs.grl_config(variant, task, scale, in_channels=in_channels)
    S = smallest_size(cfg)
    m = pkg.GRL(**dict(cfg, img_size=S))
    m.set_precision(precision)
    return m, (1, m.in_channels, S, S)


def architectures(pkg, precision):
    """(name, model, input shape) once per distinct architecture: the RELEASED checkpoints first, by checkpoint name,
    then the rest of the grid, by variant / task x scale."""
    keys = {}
    for name, (variant, task, scale, cin, _, _) in pkg.configs.RELEASED.items():
        keys.setdefault((variant, task, scale, cin if task in ("dn", "jpeg") else 3), name)
    for variant in VARIANTS:
        for task, scale in TASKS:
            keys.setdefault((variant, task, scale, 3), f"{variant}/{task}x{scale}")
    for key, name in keys.items():
        yield (name, *model(pkg, *key, precision))


def check_walk(what, launched, cases, extras=()):
    """launched: (path, first launcher) pairs of a walk; cases: (path, case) pairs of the cases that stand for launched
    paths; extras: (path, case) pairs of the other cases.  Fails on a launched path without a case and on a case of
    `cases` that nothing launches."""
    paths = {}
    for s, name in launched:
        paths.setdefault(s, name)
    have = {s for s, _ in list(cases) + list(extras)}
    missing = {s: n for s, n in paths.items() if s not in have}
    for s, n in missing.items():
        print(f"{what} path without a case: {s}, first launched by {n}")
    stale = [c for s, c in cases if s not in paths]
    print(f"{what}: {len(paths)} launched paths, {len(missing)} without a case, {len(stale)} stale cases")
    assert not missing, f"{len(missing)} launched {what} paths have no case: " + "; ".join(
        f"{s} ({n})" for s, n in missing.items())
    assert not stale, f"{what} cases that no architecture launches: {stale}"
