"""A list of differently sized images restored in a few batched forwards (GRL.forward_list / forward_list_u8).

The reference's forward takes one (B, C, H, W) tensor, so a test set of differently sized images runs as a loop of B = 1
forwards, which leaves most of the GPU idle at test-set sizes.  A forward's arithmetic depends only on the padded size
(Hp, Wp) that check_image_size gives: reflect padding, normalisation, the CAB pool, windows, stripes and the final crop
all act per image.  So the images of one padded size share a forward: one kernel pads them into a batch
(functional.list_gather), the unchanged forward runs on it and pads and crops nothing, one kernel cuts each image's
output out of the batch's (functional.list_crop).  Each output equals the image's own B = 1 forward bit for bit.
"""
from typing import NamedTuple

import torch

from . import capi
from . import functional as K
from .tc import round_up

FLOAT_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


class Chunk(NamedTuple):
    """One batched forward: the padded size and the input indices of its images, in input order."""
    hp: int
    wp: int
    index: list


def network_sizes(shapes, input_format="rgb", u8=False):
    """The (H, W) the network runs on for each image shape: (C, H, W), (H, W, C) with u8, or the (2h, 2w) of the packed
    Bayer planes (4, h, w) of an input_format="rggb" model."""
    if u8:
        return [(s[0], s[1]) for s in shapes]
    k = 2 if input_format == "rggb" else 1
    return [(k * s[1], k * s[2]) for s in shapes]


def plan(sizes, pad_size, max_batch_tokens):
    """Chunks of a list of images with network sizes `sizes`: the images are grouped by padded size (round_up(H,
    pad_size), round_up(W, pad_size)), groups in order of their first image, images in input order within a group; each
    group is cut into consecutive chunks of at most max_batch_tokens padded pixels (an image larger than that runs
    alone).  Needs no device."""
    groups = {}
    for i, (h, w) in enumerate(sizes):
        groups.setdefault((round_up(h, pad_size), round_up(w, pad_size)), []).append(i)
    chunks = []
    for (hp, wp), index in groups.items():
        n = max(1, int(max_batch_tokens) // (hp * wp))
        chunks += [Chunk(hp, wp, index[k:k + n]) for k in range(0, len(index), n)]
    return chunks


def _check(model, images, u8, what, floats=FLOAT_DTYPES):
    """Refuses a bad list before anything launches; float images must have one of the dtypes `floats`."""
    rggb = model.input_format == "rggb"
    cdim, C, least = (2, model.in_channels, 1) if u8 else (0, 4, 2) if rggb else (0, model.in_channels, 1)
    layout = f"(H, W, {C}) uint8" if u8 else f"({C}, {'h, w' if rggb else 'H, W'}) float"
    for i, x in enumerate(images):
        if not isinstance(x, torch.Tensor):
            raise ValueError(f"{what}: element {i} is a {type(x).__name__}, not a tensor")
        capi.require_device(x)
        if x.dtype not in ((torch.uint8,) if u8 else floats):
            names = [str(d).replace("torch.", "") for d in floats]
            raise ValueError(f"{what}: element {i} has dtype {x.dtype}; it takes {layout} images"
                             + ("" if u8 else f" ({' or '.join([', '.join(names[:-1]), names[-1]] if names[:-1] else names)})"))
        hw = [d for j, d in enumerate(x.shape) if j != cdim]
        if x.dim() != 3 or x.shape[cdim] != C or min(hw) < least:
            raise ValueError(f"{what}: element {i} has shape {tuple(x.shape)}; it takes {layout} images"
                             + (" with h, w >= 2" if rggb else ""))
    if len({x.dtype for x in images}) > 1:
        raise ValueError(f"{what}: the images have different dtypes {sorted({str(x.dtype) for x in images})}")


@torch.no_grad()
def forward_list(model, images, u8=False):
    """GRL.forward_list (u8=False) / GRL.forward_list_u8 (u8=True) of GRL `model`."""
    what = "forward_list_u8" if u8 else "forward_list"
    rggb = model.input_format == "rggb"
    if u8 and rggb:
        raise ValueError("forward_list_u8 takes (H, W, C) 8-bit images; packed 8-bit Bayer input (input_format='rggb') is "
                         "not supported")
    images = list(images)
    _check(model, images, u8, what)
    if not images:
        return []
    if model.self_ensemble:
        # every view of the x8 ensemble is padded on its own and each image's 8 views already form a batch: padding the
        # image first would change the views
        one = model.forward_u8 if u8 else model
        return [one(x[None])[0] for x in images]
    dtype = images[0].dtype
    kind = capi.IMAGE_U8 if u8 else capi.IMAGE_RGGB if rggb else capi.IMAGE_F32
    # the gather reads float32: other float inputs are converted, and their batch converted back below, so that the
    # forward sees what the image's own forward sees (rggb: forward converts the packed planes to float32 itself)
    src = [x.contiguous() if dtype in (torch.uint8, torch.float32) else x.float().contiguous() for x in images]
    sizes = network_sizes([tuple(x.shape) for x in images], model.input_format, u8)
    s = model.upscale
    outs = [None] * len(images)
    for ch in plan(sizes, model.pad_size, model.max_batch_tokens):
        batch = K.list_gather([src[i] for i in ch.index], kind, model.in_channels, ch.hp, ch.wp)
        if not (u8 or rggb):
            batch = batch.to(dtype)
        y = model._forward_once(batch)
        out_dtype = dtype if rggb else y.dtype
        crops = K.list_crop(y.float(), [(sizes[i][0] * s, sizes[i][1] * s) for i in ch.index], u8)
        for i, o in zip(ch.index, crops):
            outs[i] = o if u8 else o.to(out_dtype)
    return outs
