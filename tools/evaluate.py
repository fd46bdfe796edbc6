"""Score a released checkpoint on one test set, as its test command does (evaluation.evaluate), from image files:

    python tools/evaluate.py CKPT NAME --gt DIR [--lq DIR | --bicubic-lr | --lq-left DIR --lq-right DIR] [--dataset NAME]
                             [--niqe-params FILE] [--precision fp32|fp16|bf16] [--self-ensemble]
                             [--metric restorer_perceptual --lpips-weights FILE]

NAME is the configs.RELEASED key of the checkpoint (e.g. dn_grl_base_c3s15.ckpt); CKPT the file to load
(checkpoint.load_reference_checkpoint).  Files are paired by sorted name and decoded with cv2 as the reference's
base_image.imread does (data/datasets/base_image.py:227-245): colour reads converted BGR -> RGB, IMREAD_GRAYSCALE for the
gray sets, and for the gray JPEG command on LIVE1 / BSDS500 / Urban100 the colour read, whose luma evaluate takes on the
device.  --metric restorer_perceptual is the test commands' metric= override: PSNR, SSIM, LPIPS and NIQE of a command
whose collection is restorer, with LPIPS(net="vgg")'s state dict (or torchvision's vgg16 features merged with LPIPS's
lin weights) from --lpips-weights and NIQE's pristine model from --niqe-params.  The denoising noise is keyed on
"<test set directory>/<file name>" (evaluation.seed_keys, the reference's img_info[index][0]; --dataset cbsd68 and CBSD68
name the same set).  --bicubic-lr scores an SR checkpoint from HR images alone: each LR input is the bicubic downscale
of the modcropped HR image made on the device, as the SR dataset's online branch makes it (evaluate's synthesize_lr),
instead of an LR file from --lq.  Prints one table.
Under torchrun each process takes its slice of the images and rank 0 prints the gathered means.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

IMAGE_EXT = (".png", ".jpg", ".jpeg", ".bmp", ".tif", ".tiff")


def _cv2():
    try:
        import cv2
    except ImportError:
        sys.exit("tools/evaluate.py reads image files with OpenCV: install opencv-python (the package itself never needs "
                 "it)")
    return cv2


def list_images(d):
    names = sorted(f for f in os.listdir(d) if f.lower().endswith(IMAGE_EXT))
    if not names:
        sys.exit(f"no images in {d}")
    return names


def read(path, gray):
    """(H, W, C) uint8 numpy array as base_image.imread reads it."""
    cv2 = _cv2()
    if gray:
        img = cv2.imread(path, cv2.IMREAD_GRAYSCALE)
        return None if img is None else img[:, :, None]
    img = cv2.imread(path)
    return None if img is None else cv2.cvtColor(img, cv2.COLOR_BGR2RGB)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("checkpoint")
    ap.add_argument("name", help="configs.RELEASED key of the checkpoint")
    ap.add_argument("--gt", required=True)
    ap.add_argument("--lq")
    ap.add_argument("--bicubic-lr", action="store_true",
                    help="SR names: make each LR input from its HR image on the device (MATLAB bicubic, as the SR "
                         "dataset's online branch) instead of reading --lq")
    ap.add_argument("--lq-left")
    ap.add_argument("--lq-right")
    ap.add_argument("--dataset", default=None, help="the set's name, e.g. CBSD68, live1 (seed keys, gray JPEG luma)")
    ap.add_argument("--niqe-params", default=None, help="the reference's niqe_pris_params.npz (blind SR)")
    ap.add_argument("--metric", default=None, choices=("restorer_perceptual",),
                    help="metric collection override (default: the command's own)")
    ap.add_argument("--lpips-weights", default=None, help="LPIPS(net='vgg') state dict (restorer_perceptual)")
    ap.add_argument("--precision", default="fp16", choices=("fp32", "fp16", "bf16"))
    ap.add_argument("--self-ensemble", action="store_true")
    args = ap.parse_args()

    import torch

    from _pkgload import load_package

    pkg = load_package()
    from grl_image_restoration_b200 import checkpoint, configs, evaluation

    if args.name not in evaluation.RECIPES:
        sys.exit(f"unknown checkpoint name {args.name!r}; one of: {', '.join(sorted(evaluation.RECIPES))}")
    if not torch.cuda.is_available():
        sys.exit("tools/evaluate.py needs a CUDA device")
    _cv2()
    if torch.distributed.is_available() and "RANK" in os.environ and not torch.distributed.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        torch.distributed.init_process_group("nccl")
    r = evaluation.RECIPES[args.name]
    try:
        evaluation.collection(args.name, args.metric)
    except ValueError as e:
        sys.exit(str(e))
    if args.metric and not (args.lpips_weights and args.niqe_params):
        sys.exit(f"--metric {args.metric} needs --lpips-weights and --niqe-params")
    dataset = args.dataset or os.path.basename(os.path.normpath(args.gt))
    luma = r.task == "jpeg" and r.channels == 1 and dataset.lower() in evaluation.LUMA_SETS
    gray = r.channels == 1 and not luma

    dev = torch.device("cuda", torch.cuda.current_device())
    names = list_images(args.gt)

    def load_dir(d, names, gray):
        out = []
        for n in names:
            a = read(os.path.join(d, n), gray)
            if a is None:
                sys.exit(f"cannot read {os.path.join(d, n)}")
            out.append(torch.from_numpy(a).to(dev))
        return out

    t0 = time.perf_counter()
    gts = load_dir(args.gt, names, gray)
    lqs = None
    if args.bicubic_lr and (r.task != "sr" or args.lq):
        sys.exit("--bicubic-lr makes the LR inputs of an SR checkpoint and takes no --lq"
                 if r.task == "sr" else f"--bicubic-lr applies to SR checkpoints, not {args.name}")
    if r.input == "lq" and not args.bicubic_lr:
        if not args.lq:
            sys.exit(f"{args.name} needs --lq")
        lq_names = list_images(args.lq)
        if len(lq_names) != len(names):
            sys.exit(f"{len(names)} images in --gt but {len(lq_names)} in --lq")
        lqs = load_dir(args.lq, lq_names, False)
    elif r.input == "lq_dual":
        if not (args.lq_left and args.lq_right):
            sys.exit(f"{args.name} needs --lq-left and --lq-right")
        left, right = (load_dir(d, list_images(d), False) for d in (args.lq_left, args.lq_right))
        if not len(left) == len(right) == len(gts):
            sys.exit("--gt, --lq-left and --lq-right hold different numbers of images")
        lqs = list(zip(left, right))
    try:
        keys = evaluation.seed_keys(dataset, names) if r.input == "awgn" else None
    except ValueError as e:
        sys.exit(str(e))
    t_read = time.perf_counter() - t0

    img_size = {"jpeg": 288, "defocus": 480, "defocus_dual": 480, "deblur": 480}.get(r.task, 256)
    cfg = configs.released_config(args.name, img_size=img_size)
    model = pkg.GRL(**cfg, input_format="rggb" if r.input == "mosaic" else "rgb")
    checkpoint.load_reference_checkpoint(model, args.checkpoint)
    model = model.to(dev).eval()
    model.set_precision(args.precision)
    model.self_ensemble = args.self_ensemble

    torch.cuda.synchronize()
    t1 = time.perf_counter()
    result = evaluation.evaluate(model, args.name, gts, lqs, keys, dataset, args.niqe_params, args.metric,
                                 args.lpips_weights, synthesize_lr=args.bicubic_lr)
    torch.cuda.synchronize()
    t_eval = time.perf_counter() - t1
    if not torch.distributed.is_initialized() or torch.distributed.get_rank() == 0:
        print(evaluation.table(result, f"{args.name} on {dataset} ({len(gts)} images, {args.precision}"
                                       f"{', x8 self-ensemble' if args.self_ensemble else ''}); read {t_read:.2f} s, "
                                       f"evaluate {t_eval:.2f} s on {torch.cuda.get_device_name(dev)}"))
    if torch.distributed.is_initialized():
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
