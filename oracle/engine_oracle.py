"""The reference's code around the network, restated: the datasets' to_tensor, the model's check_image_size, the x8
self-ensemble's augment_img_tensor4 and merge, and the engine's forward_tile.  Each is written with the same torch ops
as the reference, on the CPU unless its inputs are elsewhere."""
import numpy as np
import torch
import torch.nn.functional as F

INVERSE = {3: 5, 5: 3}  # augment mode -> the mode that maps its view back (every other mode is its own inverse)


def to_tensor(img):
    """uint8 (..., H, W, C), NumPy or torch -> (..., C, H, W) float32 k / 255 on the CPU, as the datasets compute it.
    On a CUDA tensor torch divides by a Python scalar as a multiply by its reciprocal, 1 ulp off for 126 of the 256
    bytes, so the division stays on the CPU; callers move the result."""
    t = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img.cpu()
    return t.movedim(-1, -3).float().div(255)


def check_image_size(x, Hp, Wp):
    """check_image_size of x (B, C, H, W) padded to (Hp, Wp) (grl.py:479-489): reflect, or zeros when F.pad refuses."""
    pads = (0, Wp - x.shape[3], 0, Hp - x.shape[2])
    try:
        return F.pad(x, pads, "reflect")
    except BaseException:
        return F.pad(x, pads, "constant")


def augment(img, mode):
    """augment_img_tensor4 (utils/utils_bsr/utils_image.py:444-460) restated with the same torch ops."""
    ops = [lambda t: t, lambda t: t.rot90(1, [2, 3]).flip([2]), lambda t: t.flip([2]), lambda t: t.rot90(3, [2, 3]),
           lambda t: t.rot90(2, [2, 3]).flip([2]), lambda t: t.rot90(1, [2, 3]), lambda t: t.rot90(2, [2, 3]),
           lambda t: t.rot90(3, [2, 3]).flip([2])]
    return ops[mode](img)


def merge_reference(outs):
    """outs[m] = view m's output: 0.125 * sequential fp32 sum of the mapped-back views in mode order."""
    acc = None
    for mode, o in enumerate(outs):
        back = augment(o, INVERSE.get(mode, mode))
        acc = back.clone() if acc is None else acc + back
    return acc * 0.125


def forward_tile(fn, x, tile, overlap, scale):
    """engines/base.py:90-116 restated with `fn` as the model call; the blend runs on the CPU."""
    b, c, h, w = x.shape
    tile = min(tile, h, w)
    stride = tile - overlap
    h_idx = list(range(0, h - tile, stride)) + [h - tile]
    w_idx = list(range(0, w - tile, stride)) + [w - tile]
    E = W = None
    for hi in h_idx:
        for wi in w_idx:
            out = fn(x[..., hi:hi + tile, wi:wi + tile])
            if E is None:
                E = torch.zeros(b, out.shape[1], h * scale, w * scale)
                W = torch.zeros_like(E)
            E[..., hi * scale:(hi + tile) * scale, wi * scale:(wi + tile) * scale] += out
            W[..., hi * scale:(hi + tile) * scale, wi * scale:(wi + tile) * scale] += 1
    return E / W
