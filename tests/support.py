"""Plumbing shared by the test modules: the one model builder and the models built with it, seeded inputs, and the
comparisons.  Like archs.py, nothing here imports the product package at module level: collection runs before the
`pkg` fixture has built and loaded the library."""
import hashlib
import json
import os

import numpy as np
import torch

from engine_oracle import augment, merge_reference

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FMTS = [0, 1]  # 16-bit operand formats: 0 = fp16, 1 = bf16


def build(pkg, oracle, cfg, device, precision, *, style, seed=0, **kw):
    """GRL(**cfg, **kw) with oracle.synth_state_dict(cfg, seed, style), on `device`, in eval mode, at `precision`.  The
    non-strict load may leave out only the coordinate tables, which the model computes itself."""
    m = pkg.GRL(**cfg, **kw)
    missing, unexpected = m.load_state_dict(oracle.synth_state_dict(cfg, seed=seed, style=style), strict=False)
    assert not unexpected and set(missing) <= {"table_w", "table_sh", "table_sv"}, (missing, unexpected)
    m = m.to(device).eval()
    assert m.set_precision(precision) == precision
    return m


MICRO = {  # configs.micro_config kwargs: upscaling with CAB, denoising with the input residual, grayscale, 6 channels in
    # (dual-pixel views) and 3 out
    "micro_cab_x2": dict(),
    "micro_pad_dn": dict(embed_dim=36, stripe=(8, 16), df=2, upsampler="", upscale=1, img_size=32),
    "micro_gray": dict(embed_dim=32, heads=1, window=6, stripe=(6, 12), df=3, local_connection=False, upsampler="",
                       upscale=1, img_size=24, in_channels=1),
    "micro_dual": dict(upsampler="", upscale=1, in_channels=6),
}


def micro(pkg, oracle, name, device, precision, **kw):
    cfg = pkg.configs.micro_config(**MICRO[name])
    if name == "micro_dual":
        cfg["out_channels"] = 3
    return build(pkg, oracle, cfg, device, precision, style="init", **kw)


def dm_cases():
    with open(os.path.join(GOLD, "dm_cases.json")) as f:
        return json.load(f)


def dm_model(pkg, oracle, device, precision, input_format="rggb", **kw):
    """The architecture of the dm goldens (tests/golden/dm_cases.json)."""
    return build(pkg, oracle, dm_cases()["cfg"], device, precision, style="init", input_format=input_format, **kw)


def ensemble_cases():
    with open(os.path.join(GOLD, "ensemble_cases.json")) as f:
        return json.load(f)


def loop_ensemble(m, x):
    """What a user writes without the feature: 8 plain forwards of the module, mapped back and averaged."""
    flag, m.self_ensemble = m.self_ensemble, False
    try:
        return merge_reference([m(augment(x, mode).contiguous()) for mode in range(8)])
    finally:
        m.self_ensemble = flag


SHAPES = {  # BASELINE.json's native shapes: (variant, task, scale, img_size, input size, noise sigma); must match
    # oracle/make_golden_native.py
    "cfg2": ("small", "sr", 4, 256, (256, 256), 0.0),
    "cfg3": ("base", "dn", 1, 256, (256, 256), 50.0),
    "cfg4": ("base", "sr", 4, 256, (256, 256), 0.0),
    "cfg5": ("base", "deblur", 1, 480, (480, 480), 0.0),
}


def native_model(pkg, oracle, shape_name, style, device, precision):
    """(model, input, scale) of a native shape, as oracle/make_golden_native.py seeds them."""
    variant, task, scale, img_size, hw, sigma = SHAPES[shape_name]
    cfg = pkg.configs.grl_config(variant, task, scale, img_size)
    m = build(pkg, oracle, cfg, device, precision, style=style)
    x = oracle.synth_input((1, 3, *hw), seed=1234, noise_sigma=sigma)
    return m, x, scale


with open(os.path.join(GOLD, "zoo_cases.json")) as _f:
    ZOO = json.load(_f)["cases"]


def zoo_model(pkg, oracle, name, device, precision):
    """(model, golden arrays) of a zoo golden (tests/golden/zoo_*.npz)."""
    c = ZOO[name]
    gold = np.load(os.path.join(GOLD, f"zoo_{name}.npz"))
    return build(pkg, oracle, c["kwargs"], device, precision, style=c["style"], seed=c["weight_seed"]), gold


def random_images(shape_of, sizes, seed, device, dtype=torch.float32):
    """One torch.rand image of shape_of(h, w) per size, from one seeded generator."""
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(shape_of(h, w), generator=g).to(device=device, dtype=dtype) for h, w in sizes]


def round8_ref(v):
    """(C, H, W) or (B, C, H, W) float -> (H, W, C) or (B, H, W, C) uint8: tensor_round times 255, NaN -> 0
    (grl_image_u8.h)."""
    return (v.nan_to_num(nan=0.0).clamp(0, 1) * 255).round().byte().movedim(-3, -1)


def assert_equal_lists(got, want):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and a.dtype == b.dtype, (i, a.shape, b.shape, a.dtype, b.dtype)
        assert torch.equal(a, b), (i, (a.float() - b.float()).abs().max().item())


def count_calls(obj, attr):
    """Wraps obj.attr so that each call records the shape of its first argument; returns the list of shapes."""
    calls = []
    inner = getattr(obj, attr)

    def wrapped(x, *args, **kw):
        calls.append(tuple(x.shape))
        return inner(x, *args, **kw)

    setattr(obj, attr, wrapped)
    return calls


def grid_t(g):
    return (g.H, g.W, g.wh, g.ww, g.sh, g.sw)


def sha(t):
    return hashlib.sha256(np.ascontiguousarray(t.numpy()).tobytes()).hexdigest()


def ulp(x, dtype):
    """Spacing of `dtype` at |x| (float64), subnormal spacing at the bottom."""
    fi = torch.finfo(dtype)
    e = torch.frexp(x.abs())[1]
    return torch.clamp(fi.eps * torch.exp2((e - 1).double()), min=fi.tiny * fi.eps)


def bound_ratio(got, ref, bound):
    """max |got - ref| / bound (inf where either side is NaN)."""
    return float(((got.double() - ref).abs() / bound).nan_to_num(float("inf")).max())


def same_bits(a, b):
    """Asserts that two 8, 16, 32 or 64-bit tensors have one shape, one dtype and the same bits everywhere, except that a
    NaN matches a NaN at the same position (any payload).  +0 and -0 differ."""
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    nan_a, nan_b = a.isnan(), b.isnan()
    assert torch.equal(nan_a, nan_b), "NaN positions differ"
    ib = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    ai, bi = a.contiguous().view(ib), b.contiguous().view(ib)
    bad = (ai != bi) & ~nan_a
    assert not bad.any(), f"{int(bad.sum())} of {a.numel()} differ, first at {bad.nonzero()[0].tolist()}: " \
                          f"{a[tuple(bad.nonzero()[0])].item()!r} vs {b[tuple(bad.nonzero()[0])].item()!r}"
