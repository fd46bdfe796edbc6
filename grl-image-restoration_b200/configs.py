"""Effective ("released") GRL hyper-parameters: the model yamls overridden by the experiment yamls
and the evaluation commands (SURVEY.md Appendix B).

Cites (reference): config/model/grl/grl_{tiny,small,base}.yaml, config/experiment/sr/grl/grl_p256.yaml:31-41,
config/experiment/dn/grl/grl_p256.yaml:34-45, config/experiment/db_motion/grl_p480.yaml:33-44,
config/experiment/bsr/grl.yaml:51-64, config/model/grl/grl_base_bsr.yaml:1-34,
config/experiment/db_defocus/grl_p480.yaml:32-43,
scripts/grl/grl_test.md:35-128.
"""
import copy

_COMMON = dict(
    in_channels=3, img_range=1.0, stripe_shift=True, mlp_ratio=2, qkv_proj_type="linear",
    anchor_proj_type="avgpool", anchor_one_stage=True, out_proj_type="linear", conv_type="1conv",
    init_method="n", fairscale_checkpoint=False, offload_to_cpu=False, euclidean_dist=False,
)

_VARIANT = {
    "tiny": dict(embed_dim=64, depths=[4, 4, 4, 4], num_heads_window=[2] * 4, num_heads_stripe=[2] * 4,
                 local_connection=False, upsampler="pixelshuffledirect"),
    "small": dict(embed_dim=128, depths=[4, 4, 4, 4], num_heads_window=[2] * 4, num_heads_stripe=[2] * 4,
                  local_connection=False, upsampler="pixelshuffle"),
    "base": dict(embed_dim=180, depths=[4, 4, 8, 8, 8, 4, 4], num_heads_window=[3] * 7, num_heads_stripe=[3] * 7,
                 local_connection=True, upsampler="pixelshuffle"),
}


def grl_config(variant, task="sr", upscale=4, img_size=256, yaml_default=False, in_channels=3):
    """Constructor kwargs for GRL(**cfg).  task in {sr, dn, deblur, jpeg, dm, bsr, defocus, defocus_dual}.

    in_channels: 1 for the grayscale dn / jpeg checkpoints (model.in_channels is data_module.num_channels,
    dn/grl/grl_p256.yaml:36, jpeg/grl/grl_p288.yaml:37; grl_test.md:24,:87 select 1 or 3); the other tasks take 3.
    out_channels is left to the model's default, in_channels (grl.py:259), except for defocus_dual.
    bsr (GRL-Base only): real-world x4 SR with the nearest+conv head, window 16, stripes 32 x 64, df 4 (the released
    model's img_size is the 128 patch).  defocus: window 16, stripes 48 x 96, df 4 (img_size 480).
    defocus_dual is INFERRED, not read from a yaml (the reference has no db_defocus/grl_dual_p480.yaml): defocus with
    the left and right dual-pixel views concatenated into 6 input channels (engines/base.py:119-120) and the RGB target
    as output, so in_channels=6, out_channels=3; the model's mean is then zero (grl.py:267-271).  Nobody here has
    confirmed it against the checkpoint's conv_first.weight shape (180, 6, 3, 3)."""
    if task not in ("dn", "jpeg") and in_channels != 3:
        raise ValueError(f"task {task!r} takes 3 input channels, got in_channels={in_channels}")
    cfg = dict(_COMMON)
    cfg.update(copy.deepcopy(_VARIANT[variant]))
    cfg["img_size"] = img_size
    if yaml_default:  # bare config/model/grl/*.yaml: window 8, stripe [8, W/4], df 4
        cfg.update(window_size=8, stripe_size=[8, None], stripe_groups=[None, 4], anchor_window_down_factor=4,
                   upscale=upscale)
        return cfg
    big = variant == "base"
    if task == "sr":
        cfg.update(window_size=32, stripe_size=[64, 64], stripe_groups=[None, None],
                   anchor_window_down_factor=2 if big else 4, upscale=upscale)
    elif task == "dn":
        cfg.update(window_size=32 if big else 16, stripe_size=[64, 128], stripe_groups=[None, None],
                   anchor_window_down_factor=2 if big else 4, upscale=1, upsampler="", in_channels=in_channels)
    elif task == "deblur":
        cfg.update(window_size=12, stripe_size=[48, 96], stripe_groups=[None, None],
                   anchor_window_down_factor=4, upscale=1, upsampler="")
    elif task == "jpeg":
        cfg.update(window_size=36, stripe_size=[72, 144], stripe_groups=[None, None],
                   anchor_window_down_factor=4, upscale=1, upsampler="", in_channels=in_channels)
    elif task == "dm":
        cfg.update(window_size=8, stripe_size=[32, 32], stripe_groups=[None, None],
                   anchor_window_down_factor=4, upscale=1, upsampler="")
    elif task == "bsr":
        if not big:
            raise ValueError("the released blind SR model is GRL-Base (config/model/grl/grl_base_bsr.yaml)")
        cfg.update(window_size=16, stripe_size=[32, 64], stripe_groups=[None, None], anchor_window_down_factor=4,
                   upscale=upscale, upsampler="nearest+conv")
    elif task in ("defocus", "defocus_dual"):
        cfg.update(window_size=16, stripe_size=[48, 96], stripe_groups=[None, None], anchor_window_down_factor=4,
                   upscale=1, upsampler="")
        if task == "defocus_dual":
            cfg.update(in_channels=6, out_channels=3)
    else:
        raise ValueError(task)
    return cfg


def micro_config(embed_dim=36, depth=4, stages=1, heads=2, window=8, stripe=(8, 16), groups=(None, None), df=2,
                 local_connection=True, upsampler="pixelshuffle", upscale=2, img_size=32, in_channels=3):
    """Small test architecture that still walks all four block personalities (i % 4)."""
    cfg = dict(_COMMON)
    cfg.update(embed_dim=embed_dim, depths=[depth] * stages, num_heads_window=[heads] * stages,
               num_heads_stripe=[heads] * stages, window_size=window, stripe_size=list(stripe),
               stripe_groups=list(groups), anchor_window_down_factor=df, local_connection=local_connection,
               upsampler=upsampler, upscale=upscale, img_size=img_size, in_channels=in_channels)
    return cfg


# BASELINE.json configs (SURVEY.md 8d)
BASELINE_CONFIGS = {
    "cfg1": dict(model=("tiny", "sr", 2, 64), batch=1, size=(64, 64)),
    "cfg2": dict(model=("small", "sr", 4, 256), batch=16, size=(256, 256)),
    "cfg3": dict(model=("base", "dn", 1, 256), batch=8, size=(256, 256)),
    "cfg4": dict(model=("base", "sr", 4, 256), batch=128, size=(256, 256)),
    "cfg5": dict(model=("base", "deblur", 1, 480), batch=1, size=(720, 1280)),
}


# The released checkpoints (scripts/grl/grl_test.md) -> (variant, task, upscale, in_channels, tile, tile_overlap) of
# their evaluation.  tile / tile_overlap are what tiling.forward_tile takes (0: the whole image): the test command's
# tile= override where it has one (grl_test.md:49 dn base 256 / 32, :96 jpeg 288 / 36, :62,:70,:78 sr and :128 motion
# deblurring 0), else the experiment yaml's (db_defocus/grl_p480.yaml:9-10: 480 / 48), else config/defaults.yaml:25-26
# (0: dn tiny / small, dm, bsr).  The commands pick one noise level (SIGMA=15, :29) and one quality factor (QUALITY=10,
# :91); checkpoints of other levels share the architecture of these.
RELEASED = {
    **{f"sr_grl_{v}_c3x{s}.ckpt": (v, "sr", s, 3, 0, 0) for v in ("tiny", "small", "base") for s in (2, 3, 4)},
    **{f"dn_grl_{v}_c{c}s15.ckpt": (v, "dn", 1, c, 256 if v == "base" else 0, 32 if v == "base" else 0)
       for v in ("tiny", "small", "base") for c in (1, 3)},
    **{f"jpeg_grl_small_c{c}q10.ckpt": ("small", "jpeg", 1, c, 288, 36) for c in (1, 3)},
    "dm_grl_small.ckpt": ("small", "dm", 1, 3, 0, 0),
    "bsr_grl_base.ckpt": ("base", "bsr", 4, 3, 0, 0),
    "db_defocus_single_pixel_grl_base.ckpt": ("base", "defocus", 1, 3, 480, 48),
    "db_defocus_dual_pixel_grl_base.ckpt": ("base", "defocus_dual", 1, 6, 480, 48),
    **{f"db_motion_grl_base_{d}.ckpt": ("base", "deblur", 1, 3, 0, 0) for d in ("gopro", "realblur_j", "realblur_r")},
}


def released_config(name, img_size=256):
    """grl_config of a RELEASED checkpoint."""
    variant, task, upscale, cin, _, _ = RELEASED[name]
    return grl_config(variant, task, upscale, img_size, in_channels=cin if task in ("dn", "jpeg") else 3)
