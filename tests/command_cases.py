"""The forwards the released checkpoints' test commands run (evaluation.evaluate), at the sizes they run them: one or more
CommandCase per configs.RELEASED checkpoint, shared by test_command_paths.py (CPU: the sizes follow each recipe, and no
size takes a launch path the launch-path tests lack) and the two replay files (`command:` cases of
replay_base.replay_case).  Like support.py, nothing here imports the product package at module level.

A case's `image` is a test-set size class, not a file: the clean image the dataset reads (for SR, the ground truth
whose low-resolution file the command loads; for dm, the RGB image it mosaics).  Its `forward` is what the network's
forward really sees: after the recipe's crop (modcrop by the SR scale, or mod 8), the SR scale, the packed Bayer planes
(dm: half the size, 4 planes) and t = min(tile, H, W) of a tiled command.  Inputs follow the recipe: sigma 15 Gaussian
noise for dn (synth_input(noise_sigma=15)), "spread" weights everywhere."""
from typing import NamedTuple

import torch

import archs

DN_SIGMA = 15.0


class CommandCase(NamedTuple):
    ckpt: str        # configs.RELEASED key
    image: tuple     # (H, W) of the image the command reads
    forward: tuple   # (H, W) of the forward's input (dm: of the packed planes)
    what: str        # what the size exercises
    tc: tuple = ()   # precisions the tensor-core replay runs it in
    f32: bool = False  # the fp32 replay runs it

    @property
    def name(self):
        """The replay case name without its precision: command:<checkpoint>@<H>x<W> (the forward's size)."""
        return f"command:{self.ckpt[:-len('.ckpt')]}@{self.forward[0]}x{self.forward[1]}"


FP16, BOTH = ("fp16",), ("fp16", "bf16")
CASES = [
    *[CommandCase(f"sr_grl_{v}_c3x2.ckpt", (1170, 827), (585, 413), "crop on both sides, pad 640 x 448", FP16,
                  f32=v == "base") for v in ("tiny", "small", "base")],
    *[CommandCase(f"sr_grl_{v}_c3x3.ckpt", (768, 1024), (256, 341), "crop on W, ps_r / nchw_r = 3 at real width",
                  FP16, f32=v == "tiny") for v in ("tiny", "small", "base")],
    *[CommandCase(f"sr_grl_{v}_c3x4.ckpt", (1170, 827), (292, 206), "crop on both sides, non-square", FP16)
      for v in ("tiny", "small", "base")],
    *[CommandCase(f"dn_grl_{v}_c{c}s15.ckpt", (321, 481), (320, 480), "mod 8, pad to 384 x 512, crop", FP16,
                  f32=(v, c) == ("small", 3)) for v in ("tiny", "small") for c in (1, 3)],
    CommandCase("dn_grl_small_c3s15.ckpt", (768, 1024), (768, 1024), "a whole 768 x 1024 image", FP16),
    CommandCase("dn_grl_base_c1s15.ckpt", (321, 481), (256, 256), "256 tile: the 1-channel Base head and tail", FP16),
    # the 3-channel Base denoiser's 256 tile is native:cfg3's architecture and geometry, which both replays run
    CommandCase("dn_grl_base_c3s15.ckpt", (321, 481), (256, 256), "256 tile (native:cfg3 replays it)"),
    CommandCase("jpeg_grl_small_c1q10.ckpt", (512, 512), (288, 288), "288 tile: window 36, generic-KW attention", FP16,
                f32=True),
    CommandCase("jpeg_grl_small_c1q10.ckpt", (256, 400), (256, 256), "an image under the tile: 256 tile, pad to 288",
                f32=True),
    CommandCase("jpeg_grl_small_c3q10.ckpt", (512, 512), (288, 288), "288 tile: window 36, generic-KW attention", FP16),
    CommandCase("jpeg_grl_small_c3q10.ckpt", (256, 400), (256, 256), "an image under the tile: 256 tile, pad to 288",
                BOTH),
    CommandCase("dm_grl_small.ckpt", (500, 500), (248, 248), "mod 8 to 496, rggb head, pad 512, crop", FP16, f32=True),
    CommandCase("bsr_grl_base.ckpt", (375, 500), (375, 500), "nearest+conv tail, crop", BOTH, f32=True),
    CommandCase("db_defocus_single_pixel_grl_base.ckpt", (1120, 1680), (480, 480), "window 16 / stripes 48 x 96, 480 tile",
                FP16, f32=True),
    CommandCase("db_defocus_dual_pixel_grl_base.ckpt", (1120, 1680), (480, 480), "480 tile, 6 channels in", FP16),
    CommandCase("db_motion_grl_base_gopro.ckpt", (720, 1280), (720, 1280),
                "a whole frame, 768 x 1344 padded: the largest single forward of any command", FP16, f32=True),
    # the RealBlur checkpoints share GoPro's architecture and whole-image recipe
    CommandCase("db_motion_grl_base_realblur_j.ckpt", (720, 1280), (720, 1280), "as GoPro"),
    CommandCase("db_motion_grl_base_realblur_r.ckpt", (720, 1280), (720, 1280), "as GoPro"),
]
BY_NAME = {c.name: c for c in CASES}


def tc_names():
    return [f"{c.name}-{p}" for c in CASES for p in c.tc]


def f32_names():
    return [f"{c.name}-fp32" for c in CASES if c.f32]


def cfg(pkg, case):
    """The checkpoint's constructor kwargs (configs.released_config), with the img_size archs.py builds it at (the
    forward pads any input to model.pad_size)."""
    c = pkg.configs.released_config(case.ckpt)
    return dict(c, img_size=archs.smallest_size(c))


def input_shape(pkg, case):
    """(1, C, H, W) of the forward's input: 4 packed planes for dm, else the model's in_channels."""
    return (1, 4 if is_dm(pkg, case) else cfg(pkg, case)["in_channels"], *case.forward)


def is_dm(pkg, case):
    return pkg.configs.RELEASED[case.ckpt][1] == "dm"


def model_and_input(pkg, oracle, case, device, precision, style="spread"):
    """(model, input, rggb) of a command case: "spread" weights (or `style`); dm takes packed Bayer planes
    (input_format "rggb"); dn adds sigma 15 noise."""
    from support import build

    rggb = is_dm(pkg, case)
    m = build(pkg, oracle, cfg(pkg, case), device, precision, style=style,
              **({"input_format": "rggb"} if rggb else {}))
    sigma = DN_SIGMA if pkg.configs.RELEASED[case.ckpt][1] == "dn" else 0.0
    x = oracle.synth_input(input_shape(pkg, case), seed=1234, noise_sigma=sigma)
    return m, x, rggb


@torch.no_grad()
def oracle_output(pkg, oracle, case, x, rggb, style, dtype=torch.float32):
    """oracle.grl_forward of the case in `dtype` on x's device (weights of `style`), with TF32 off for its convs and
    matmuls; dm runs on the library's host demosaic of the planes (bit-exact against the kernel)."""
    from grl_image_restoration_b200 import functional as K

    c = cfg(pkg, case)
    sd = {k: v.to(x.device, dtype) for k, v in oracle.synth_state_dict(c, seed=0, style=style).items()}
    xin = K.demosaic_host(x.cpu()).to(x.device) if rggb else x
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return oracle.grl_forward(sd, c, xin.to(dtype))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags


GT_SEED = 9  # the uniform "ground truth" of the 16-bit PSNR gates (test_gpu_zoo_model.py, test_gpu_native_shapes.py)


def _stats(oracle, y, ref):
    """(max-abs, PSNR(cand, ref), |PSNR(cand, GT) - PSNR(ref, GT)|) over the whole output."""
    y, ref = y.double().cpu(), ref.double().cpu()
    gt = torch.rand(ref.shape, generator=torch.Generator().manual_seed(GT_SEED)).double()
    return (float((y - ref).abs().max()), float(-10 * torch.log10(((y - ref) ** 2).mean())),
            float((oracle.psnr(y, gt) - oracle.psnr(ref, gt)).abs().max()))


@torch.no_grad()
def end_to_end(pkg, oracle, case, device, precision, y, x, rggb):
    """(passes, report) of the case's forward against oracle.grl_forward on the device, with the gates of
    test_gpu_native_shapes.py in the regimes it applies them:
      y (the replayed forward of x, "spread" weights): fp32 within 1e-3 max-abs of the fp32 oracle.  Where it is not,
        the oracle's own fp32 error is measured against the float64 oracle, and y passes if it is no farther from
        float64 than max(1e-3, twice that error): a near-chaotic network amplifies any fp32 rounding, the oracle's too.
        fp16 / bf16 outputs are reported: the 16-bit gates are defined on "init" weights;
      a forward on "init" weights, every precision: max-abs <= 1e-3 in fp32, PSNR(cand, ref) >= 56 / 40 dB and
        |dPSNR vs GT| <= 0.01 dB in fp16 / bf16."""
    ok = bool(torch.isfinite(y).all())
    err, p_cr, d_psnr = _stats(oracle, y, oracle_output(pkg, oracle, case, x, rggb, "spread"))
    msg = f"spread: max-abs vs oracle {err:.3e}, PSNR(cand, ref) {p_cr:.1f} dB, |dPSNR vs GT| {d_psnr:.2e} dB"
    if precision == "fp32" and err > 1e-3:
        ref64 = oracle_output(pkg, oracle, case, x, rggb, "spread", torch.float64)
        own = _stats(oracle, oracle_output(pkg, oracle, case, x, rggb, "spread"), ref64)[0]
        err64 = _stats(oracle, y, ref64)[0]
        del ref64
        ok = ok and err64 <= max(1e-3, 2 * own)
        msg += f"; vs the float64 oracle {err64:.3e}, the fp32 oracle's own error {own:.3e}"
    m, xi, rggb = model_and_input(pkg, oracle, case, device, precision, style="init")
    xi = xi.to(device)
    m.use_cuda_graph = False
    yi = m(xi)
    del m
    err, p_cr, d_psnr = _stats(oracle, yi, oracle_output(pkg, oracle, case, xi, rggb, "init"))
    msg += f"; init: max-abs {err:.3e}, PSNR(cand, ref) {p_cr:.1f} dB, |dPSNR vs GT| {d_psnr:.2e} dB"
    if precision == "fp32":
        ok = ok and err <= 1e-3
    else:
        ok = ok and p_cr >= (56.0 if precision == "fp16" else 40.0) and d_psnr <= 0.01
    return ok and bool(torch.isfinite(yi).all()), msg


def expected_mutations(model, case, rggb):
    """(the tail / crop pitch control applies: Wc < Wp, the transposed-grid control applies: a non-square window grid)
    of a command case."""
    h, w = (2 * v for v in case.forward) if rggb else case.forward
    p = model.pad_size
    hp, wp = -(-h // p) * p, -(-w // p) * p
    wh, ww = model.layers[0].blocks[0].attn.window_attn.window_size
    return w < wp, hp // wh != wp // ww
