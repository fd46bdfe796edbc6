"""A released checkpoint's test command as one call: the clean image the dataset crops, the model input it makes, the
forward the command runs and the metric collection it reports, all on the device.

RECIPES maps every configs.RELEASED name to its Recipe; evaluate(model, name, gts, ...) runs it over a test set of
decoded 8-bit images with the package's own device calls only (crop views, the degradation kernels, forward_list /
forward_tile_list and their _u8 forms, psnr_fused / ssim_fused / psnrb_fused / niqe) and returns the per-image scores
under the reference's metric names and their means as average_metric (utils/metrics/psnr.py:19-41) forms them.  Under
an initialised process group every rank restores a contiguous slice of the images (sharding.shard_range) and the
per-image scores are all-gathered (sharding.gather_metric), as the reference's gpus=2 commands do.

Reference lines (all paths in the reference checkout):
  crop (VAL)   data/datasets/base_image.py:404-405 (modcrop by the SR scale when a low-quality image is given; scale 1
               for the JPEG and paired deblurring sets: no crop), :419-423 (clean image alone: top-left crop to multiples
               of data_module.modulo, default 8: dn, dm)
  inputs       restoration_sr.py:100-115 (LR file; with synthesize_lr the online LR of :127-141, imresize(modcrop(img_gt)
               / 255, 1 / scale), utils/matlab_functions.py:92-188), restoration_dn.py:134-143 (AWGN keyed on img_info[index][0],
               base_image.py:47-53), restoration_jpeg.py:38-42 + :62-79 (JPEG round trip, colour via BGR),
               base_image.py:233-241 (gray JPEG on live1 / bsds500 / urban100: rgb2ycbcr_np luma of the colour read),
               restoration_dm.py:33-37 (mosaic_CFA_Bayer(img)[1]), restoration_bsr.py:111-118 (uint2single of the image
               itself, no ground truth), restoration_paired_dataset.py:140-147 + engines/base.py:119-120 (LQ file; dual
               pixel: left and right concatenated on channels)
  forward      configs.RELEASED's tile / tile_overlap (scripts/grl/grl_test.md)
  metrics      config/metric/restorer*.yaml (restorer_perceptual through the metric= override); engines/base.py:255-268
               (tensor_round, shave by the scale for SR), engines/base_gan.py:149-168 (bsr: no shave)
"""
import collections
import math

import torch

from . import configs, functional as K, metrics, sharding, tiling

# The metric collections (config/metric/<name>.yaml) -> the reference's metric names, in the yaml's order.
COLLECTIONS = {
    "restorer": ("val_psnr", "val_psnr_y", "val_ssim", "val_ssim_y"),
    "restorer_gray": ("val_psnr", "val_ssim"),
    "restorer_jpeg": ("val_psnr", "val_psnr_y", "val_ssim", "val_ssim_y", "val_psnrb", "val_psnrb_y"),
    "restorer_jpeg_gray": ("val_psnr", "val_ssim", "val_psnrb"),
    "restorer_niqe": ("val_niqe",),
}

# The collections a test command's metric= override may select instead of its recipe's, each for recipes whose own
# collection is "restorer" (config/metric/restorer_perceptual.yaml).
PERCEPTUAL_COLLECTIONS = {
    "restorer_perceptual": ("val_psnr", "val_psnr_y", "val_ssim", "val_ssim_y", "val_lpips", "val_niqe"),
}

# The dtype each metric's per-image value has: psnr_fused gives float32, ssim_fused / psnrb_fused / niqe float64.
METRIC_DTYPES = {"val_psnr": torch.float32, "val_psnr_y": torch.float32, "val_ssim": torch.float64,
                 "val_ssim_y": torch.float64, "val_psnrb": torch.float64, "val_psnrb_y": torch.float64,
                 "val_niqe": torch.float64, "val_lpips": torch.float64}

# The test sets' directory names, which start the reference's image names (img_info[index][0], the denoising seed key),
# from the lower-case names its configs use (data/datasets/restoration_dn.py:72-88).
TEST_SETS = {"set12": "Set12", "bsd68": "BSD68", "cbsd68": "CBSD68", "kodak24": "Kodak24", "mcmaster": "McMaster",
             "urban100": "Urban100", "classic5": "Classic5", "live1": "LIVE1", "bsds500": "BSDS500",
             "icb_gray": "ICB_Gray", "icb_rgb": "ICB_RGB", "realsr": "RealSRSetPlus5images"}


def seed_keys(dataset, filenames):
    """The denoising seed keys of a test set's files, img_info[index][0] = "<test set directory>/<file name>": the set
    name is looked up case-insensitively in TEST_SETS, so "cbsd68" and "CBSD68" both key on "CBSD68/...".  A name the
    reference does not know is refused: its noise stream would silently differ."""
    d = TEST_SETS.get(str(dataset).lower())
    if d is None:
        raise ValueError(f"grl_b200: unknown denoising test set {dataset!r}; the reference keys its noise on one of "
                         f"{sorted(TEST_SETS.values())}")
    return [f"{d}/{f}" for f in filenames]


# The gray JPEG sets whose clean image is the MATLAB luma of the colour file (base_image.py:233-237); every other gray set
# is cv2's IMREAD_GRAYSCALE decode (:239).
LUMA_SETS = ("live1", "bsds500", "urban100")

Recipe = collections.namedtuple("Recipe", [
    "task",         # configs task name
    "crop",         # clean image: "modcrop" (to a multiple of the scale), "mod8" (to multiples of 8) or "none"
    "input",        # model input: "lq" (the LQ file as is), "lq_dual" (left || right), "awgn", "jpeg", "mosaic",
                    # "self" (the image itself, no ground truth)
    "level",        # the degradation's parameter: noise sigma (awgn) or JPEG quality, else None
    "channels",     # the clean image's channels
    "tile",         # tile, tile_overlap of the forward (0: the whole image)
    "tile_overlap",
    "collection",   # metric collection (COLLECTIONS)
    "border",       # pixels shaved on every side before the metrics
])


def _recipe(name):
    _, task, scale, cin, tile, overlap = configs.RELEASED[name]
    if task == "sr":  # grl_test.md:55-78 (tile=0); config/experiment/sr/grl/grl_p256.yaml:23
        return Recipe(task, "modcrop", "lq", None, 3, tile, overlap, "restorer", scale)
    if task == "dn":  # grl_test.md:23-29 (SIGMA=15, METRIC=(restorer_gray restorer)), :49
        return Recipe(task, "mod8", "awgn", 15, cin, tile, overlap, "restorer" if cin == 3 else "restorer_gray", 0)
    if task == "jpeg":  # grl_test.md:84-96 (QUALITY=10, METRIC=(restorer_jpeg_gray restorer_jpeg))
        return Recipe(task, "none", "jpeg", 10, cin, tile, overlap, "restorer_jpeg" if cin == 3 else "restorer_jpeg_gray", 0)
    if task == "dm":  # config/experiment/dm/grl.yaml:21
        return Recipe(task, "mod8", "mosaic", None, 3, tile, overlap, "restorer", 0)
    if task == "bsr":  # config/experiment/bsr/grl.yaml:26, :49 (with_gt: False)
        return Recipe(task, "none", "self", None, 3, tile, overlap, "restorer_niqe", 0)
    if task in ("defocus", "defocus_dual", "deblur"):  # db_defocus/grl_p480.yaml:24, db_motion/grl_p480.yaml:25
        return Recipe(task, "none", "lq_dual" if task == "defocus_dual" else "lq", None, 3, tile, overlap, "restorer", 0)
    raise ValueError(task)


RECIPES = {name: _recipe(name) for name in configs.RELEASED}


def _images(xs, what, channels=None):
    xs = list(xs)
    for i, t in enumerate(xs):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.dim() != 3 or not t.is_cuda:
            raise ValueError(f"grl_b200: evaluate: {what}[{i}] must be an (H, W, C) uint8 CUDA tensor, got "
                             f"{type(t).__name__} {getattr(t, 'dtype', '')} {tuple(getattr(t, 'shape', ()))}")
        if channels is not None and t.shape[2] != channels:
            raise ValueError(f"grl_b200: evaluate: {what}[{i}] has {t.shape[2]} channels, the recipe needs {channels}")
    return xs


def _crop(g, recipe, scale):
    H, W = g.shape[:2]
    m = scale if recipe.crop == "modcrop" else 8 if recipe.crop == "mod8" else 1
    return g[: H - H % m, : W - W % m]


def clean_images(name, gts, dataset=None):
    """The recipe's clean images of decoded 8-bit images (views where they are crops): the dataset's VAL crop, and for the
    gray JPEG command on LIVE1 / BSDS500 / Urban100 the device luma of the RGB images."""
    r = RECIPES[name]
    scale = configs.RELEASED[name][2]
    luma = r.task == "jpeg" and r.channels == 1 and (dataset or "").lower() in LUMA_SETS
    gts = _images(gts, "gts", 3 if luma else r.channels)
    if luma:
        gts = K.luma_list(gts)
    return [_crop(g, r, scale) for g in gts]


def _check_synthesize_lr(name, lqs, synthesize_lr):
    if synthesize_lr and (RECIPES[name].task != "sr" or lqs is not None):
        raise ValueError(f"grl_b200: evaluate: synthesize_lr=True makes the LR input of an SR recipe from its HR images and "
                         f"takes no lqs; got {name} ({RECIPES[name].task}) with lqs {'given' if lqs is not None else 'None'}")


def model_inputs(name, clean, lqs=None, keys=None, synthesize_lr=False):
    """The recipe's model inputs: (H, W, C) uint8 for the u8 forwards, (C, H, W) float32 for awgn, the mosaic and, with
    synthesize_lr (SR recipes, no lqs), the bicubic downscale of the modcropped clean images."""
    r = RECIPES[name]
    _check_synthesize_lr(name, lqs, synthesize_lr)
    if synthesize_lr:
        return K.imresize_list(clean, 1 / configs.RELEASED[name][2])
    if r.input == "awgn":
        if keys is None or len(keys) != len(clean):
            raise ValueError("grl_b200: evaluate: the denoising recipe needs one seed key per image (the reference keys "
                             "on img_info[index][0], '<dataset>/<file name>')")
        return K.awgn_list([c.contiguous() for c in clean], r.level, keys)
    if r.input == "jpeg":
        return K.jpeg_roundtrip_list([c.contiguous() for c in clean], r.level)
    if r.input == "mosaic":
        return K.mosaic_list(clean)
    if r.input == "self":
        return [c.contiguous() for c in clean]
    if lqs is None or len(lqs) != len(clean):
        raise ValueError(f"grl_b200: evaluate: the {r.task} recipe needs one low-quality image per clean image")
    if r.input == "lq_dual":
        pairs = list(lqs)
        left = _images([p[0] for p in pairs], "lqs (left)", 3)
        right = _images([p[1] for p in pairs], "lqs (right)", 3)
        return [torch.cat([a, b], 2) for a, b in zip(left, right)]
    return [t.contiguous() for t in _images(lqs, "lqs", r.channels)]


def restore(model, name, inputs):
    """The command's forward over the model inputs -> (H, W, C) uint8 outputs (f32_to_u8 of the float forwards: the
    validation step's tensor_round)."""
    r = RECIPES[name]
    if (r.input == "mosaic") != (getattr(model, "input_format", "rgb") == "rggb"):
        raise ValueError(f"grl_b200: evaluate: {name} needs a model with input_format="
                         f"{'rggb' if r.input == 'mosaic' else 'rgb'}")
    if not inputs:
        return []
    if inputs[0].dtype == torch.uint8:
        return (tiling.forward_tile_list_u8(model, inputs, r.tile, r.tile_overlap) if r.tile
                else model.forward_list_u8(inputs))
    outs = tiling.forward_tile_list(model, inputs, r.tile, r.tile_overlap) if r.tile else model.forward_list(inputs)
    return [K.f32_to_u8(o[None])[0] for o in outs]


def collection(name, metric=None):
    """The metric names `name`'s test command reports: its recipe's collection, or the collection `metric` names (the
    command's metric= override; PERCEPTUAL_COLLECTIONS, for recipes whose collection is restorer)."""
    r = RECIPES[name]
    if metric is None:
        return COLLECTIONS[r.collection]
    if metric not in PERCEPTUAL_COLLECTIONS:
        raise ValueError(f"grl_b200: evaluate: metric={metric!r} is not supported; None keeps the recipe's collection, or "
                         f"one of {sorted(PERCEPTUAL_COLLECTIONS)} (restorer_gray_perceptual needs a grayscale NIQE, which "
                         "is not built)")
    if r.collection != "restorer":
        raise ValueError(f"grl_b200: evaluate: metric={metric!r} needs a recipe whose collection is restorer; {name} "
                         f"reports {r.collection}")
    return PERCEPTUAL_COLLECTIONS[metric]


def score(name, restored, clean, niqe_params=None, metric=None, lpips_weights=None):
    """{metric name: 0-d tensor} of one (H, W, C) uint8 output against its clean image (None for the blind recipe), for
    the collection of collection(name, metric)."""
    r = RECIPES[name]
    names = collection(name, metric)
    a = restored[None]
    if r.collection == "restorer_niqe":
        if niqe_params is None:
            raise ValueError("grl_b200: evaluate: the blind SR recipe scores NIQE and needs niqe_params (the reference's "
                             "niqe_pris_params.npz)")
        return {"val_niqe": metrics.niqe(a, niqe_params, r.border)[0]}
    b = clean[None]
    out = {}
    p, py = metrics.psnr_fused(a, b, r.border)
    s, sy = metrics.ssim_fused(a, b, r.border)
    out.update(val_psnr=p[0], val_psnr_y=py[0], val_ssim=s[0], val_ssim_y=sy[0])
    if r.collection.startswith("restorer_jpeg"):
        pb, pby = metrics.psnrb_fused(a, b)
        out.update(val_psnrb=pb[0], val_psnrb_y=pby[0])
    if "val_lpips" in names:
        out.update(val_lpips=metrics.lpips(a, b, lpips_weights, r.border)[0],
                   val_niqe=metrics.niqe(a, niqe_params, r.border)[0])
    return {k: out[k] for k in names}


def mean(values):
    """average_metric's mean of per-image values in index order: a running sum of the 0-d tensors in their dtype, over
    the count."""
    acc = 0
    for v in values:
        acc = acc + v
    return acc / len(values)


@torch.no_grad()
def evaluate(model, name, gts, lqs=None, keys=None, dataset=None, niqe_params=None, metric=None, lpips_weights=None,
             synthesize_lr=False):
    """The test command of the released checkpoint `name` (a configs.RELEASED key) on `model`, over one test set.

    gts: decoded (H, W, C) uint8 CUDA images (RGB, or one channel for the gray sets; for the gray JPEG command on
    LIVE1 / BSDS500 / Urban100 the RGB images, whose luma this takes); for the blind SR command the images themselves.
    lqs: the low-quality images of the SR and deblurring commands, (H, W, 3) uint8, and for defocus_dual (left, right)
    pairs.  keys: the denoising noise's seed per image, a dataset-relative path such as "CBSD68/0001.png" (dn_seed).
    dataset: the set's name (selects the luma for the gray JPEG command).  niqe_params: the NIQE pristine model (bsr, and
    restorer_perceptual).  metric: the command's metric= override: None keeps the recipe's collection; "restorer_perceptual"
    (recipes whose collection is restorer) adds val_lpips and val_niqe on the same shaved 8-bit images and needs
    lpips_weights (metrics.lpips_weights accepts it) and niqe_params.  synthesize_lr: for an SR recipe without lqs, make
    each LR input on the device from its modcropped HR image as the SR dataset's online branch does, imresize(img / 255,
    1 / scale) (functional.imresize_list), instead of reading an LR file; the scores may differ slightly from those on
    MATLAB-made LR files.  model.precision and model.self_ensemble apply as they are set.

    Returns {"scores": {metric: (N,) CPU tensor in image order}, "means": {metric: float}} with the reference's metric
    names (val_psnr, val_psnr_y, val_ssim, ...)."""
    if name not in RECIPES:
        raise ValueError(f"grl_b200: evaluate: unknown checkpoint name {name!r} (configs.RELEASED)")
    names = collection(name, metric)
    _check_synthesize_lr(name, lqs, synthesize_lr)
    if metric is not None and (lpips_weights is None or niqe_params is None):
        raise ValueError(f"grl_b200: evaluate: metric={metric!r} scores LPIPS and NIQE and needs lpips_weights and "
                         "niqe_params")
    if lpips_weights is not None:
        lpips_weights = metrics.lpips_weights(lpips_weights)
    gts = list(gts)
    n = len(gts)
    if n == 0:
        raise ValueError("grl_b200: evaluate: no images")
    lqs = None if lqs is None else list(lqs)
    keys = None if keys is None else list(keys)
    lo, hi = 0, n
    distributed = torch.distributed.is_available() and torch.distributed.is_initialized()
    if distributed:
        lo, hi = sharding.shard_range(n, torch.distributed.get_rank(), torch.distributed.get_world_size())
    clean = clean_images(name, gts[lo:hi], dataset)
    inputs = model_inputs(name, clean, None if lqs is None else lqs[lo:hi], None if keys is None else keys[lo:hi],
                          synthesize_lr)
    outs = restore(model, name, inputs)
    per = [score(name, o, c, niqe_params, metric, lpips_weights) for o, c in zip(outs, clean)]
    return gather_scores(per, names, lo, hi, gts[0].device)


def gather_scores(per, names, lo, hi, device):
    """evaluate's result from this rank's per-image scores `per` (images lo..hi-1, a list of {metric: 0-d tensor}):
    every rank's scores all-gathered (sharding.gather_metric) and put back in image order, and their means.  Each metric
    has one dtype (METRIC_DTYPES) on every rank, also on a rank whose slice is empty, so the collective's buffers agree."""
    scores, means = {}, {}
    idx = torch.arange(lo, hi, device=device, dtype=torch.int64)
    for m in names:
        dtype = METRIC_DTYPES[m]
        vals = torch.stack([p[m].to(device=device, dtype=dtype) for p in per]) if per else \
            torch.empty(0, device=device, dtype=dtype)
        gv, gi = sharding.gather_metric(vals, idx)
        v = gv[torch.argsort(gi)].cpu()
        scores[m] = v
        means[m] = float(mean(list(v.unbind(0))))
    return {"scores": scores, "means": means}


def table(result, title=None):
    """A plain text table of evaluate's result: one row per metric, its mean and the number of images."""
    lines = [title] if title else []
    for m, v in result["means"].items():
        lines.append(f"{m:<14} {v:>10.4f}   ({len(result['scores'][m])} images)" if math.isfinite(v)
                     else f"{m:<14} {v!r:>10}   ({len(result['scores'][m])} images)")
    return "\n".join(lines)
