"""Thin functional layer over the C ABI (capi.py): allocates outputs with torch, passes raw device pointers +
the current CUDA stream, raises RuntimeError on a non-zero status.  Activations are channels-last fp32."""
import ctypes

import torch

from . import capi

ACT_NONE, ACT_GELU, ACT_LEAKY = 0, 1, 2


class KernelTimer:
    """Optional CUDA-event timer around the attention launches (bench.py's roofline leg).  Events are recorded on
    the stream the kernels are launched on (torch's current stream)."""

    def __init__(self):
        self.pairs = {}

    def wrap(self, tag, fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        self.pairs.setdefault(tag, []).append((e0, e1))
        return out

    def totals_ms(self):
        """{tag: (total ms, launches)} -- call after a synchronize."""
        return {k: (sum(a.elapsed_time(b) for a, b in v), len(v)) for k, v in self.pairs.items()}


timer = None  # set to a KernelTimer to time attention kernels


def _timed(tag, fn):
    return fn() if timer is None else timer.wrap(tag, fn)


def _f32c(t, name):
    capi.require_device(t)
    if t.dtype != torch.float32:
        raise RuntimeError(f"grl_b200: {name} must be float32, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def linear(x, weight, bias=None, act=ACT_NONE, slope=0.0, res=None, out=None):
    """x (..., K) -> (..., N): y = act(x W^T + b) (+ res)."""
    x = _f32c(x, "x")
    K = x.shape[-1]
    N = weight.shape[0]
    M = x.numel() // K
    y = out if out is not None else torch.empty(*x.shape[:-1], N, device=x.device, dtype=torch.float32)
    if res is not None:
        res = _f32c(res, "res")
    capi.check(capi.lib().grl_linear_f32(capi.ptr(x), K, capi.ptr(_f32c(weight, "weight")), capi.ptr(bias),
                                         capi.ptr(res), N, capi.ptr(y), N, M, N, K, act, slope, capi.stream()))
    return y


def pack_conv_weight(weight):
    """(Cout, Cin, 3, 3) -> (Cout, 9*Cin) with k = (ky*3+kx)*Cin + c (the im2col order of the kernels)."""
    co, ci, kh, kw = weight.shape
    if (kh, kw) != (3, 3):
        raise RuntimeError("grl_b200: only 3x3 convolutions are on this path")
    return weight.detach().permute(0, 2, 3, 1).reshape(co, 9 * ci).contiguous()


def conv3x3(x, wpacked, bias=None, act=ACT_NONE, slope=0.0, res=None, out=None):
    """x (B, H, W, Cin) channels-last -> (B, H, W, Cout); stride 1, zero pad 1."""
    x = _f32c(x, "x")
    B, H, W, Cin = x.shape
    Cout = wpacked.shape[0]
    y = out if out is not None else torch.empty(B, H, W, Cout, device=x.device, dtype=torch.float32)
    if res is not None:
        res = _f32c(res, "res")
    capi.check(capi.lib().grl_conv3x3_f32(capi.ptr(x), capi.ptr(wpacked), capi.ptr(bias), capi.ptr(res), capi.ptr(y),
                                          B, H, W, Cin, Cout, act, slope, capi.stream()))
    return y


def avgpool(x, df, out=None):
    x = _f32c(x, "x")
    B, H, W, C = x.shape
    y = out if out is not None else torch.empty(B, H // df, W // df, C, device=x.device, dtype=torch.float32)
    capi.check(capi.lib().grl_avgpool_f32(capi.ptr(x), capi.ptr(y), B, H, W, C, df, capi.stream()))
    return y


def ln_residual(x, u, gamma, beta, eps=1e-5, res_scale=1.0, cab_y=None, cab_gate=None, out=None):
    """(x or 0) + res_scale * LN(u) (+ cab_y * gate[b]); x, u (B, L, C)."""
    u = _f32c(u, "u")
    B, L, C = u.shape
    out = torch.empty_like(u) if out is None else out
    capi.check(capi.lib().grl_ln_residual_f32(
        capi.ptr(_f32c(x, "x")) if x is not None else None, capi.ptr(u), capi.ptr(gamma), capi.ptr(beta), eps,
        res_scale, capi.ptr(_f32c(cab_y, "cab_y")) if cab_y is not None else None,
        capi.ptr(cab_gate) if cab_gate is not None else None, L, capi.ptr(out), B * L, C, capi.stream()))
    return out


def channel_gate(y, w1, b1, w2, b2, out=None):
    """y (B, L, C) -> gate (B, C) = sigmoid(W2 relu(W1 mean_L(y) + b1) + b2)."""
    y = _f32c(y, "y")
    B, L, C = y.shape
    R = w1.shape[0]
    nbytes = capi.lib().grl_channel_gate_workspace(B, L, C)
    ws = torch.empty(max(nbytes, 4) // 4, device=y.device, dtype=torch.float32)
    gate = out if out is not None else torch.empty(B, C, device=y.device, dtype=torch.float32)
    capi.check(capi.lib().grl_channel_gate_f32(capi.ptr(y), B, L, C, capi.ptr(w1), capi.ptr(b1), capi.ptr(w2),
                                               capi.ptr(b2), R, capi.ptr(gate), capi.ptr(ws), nbytes, capi.stream()))
    return gate


def bias_table(table, w1, b1, w2, out=None):
    """table (..., 2) -> activated bias (heads, rows) = 16*sigmoid(cpb_mlp(table))."""
    t = _f32c(table, "table").reshape(-1, 2)
    heads, hidden = w2.shape
    out = out if out is not None else torch.empty(heads, t.shape[0], device=t.device, dtype=torch.float32)
    capi.check(capi.lib().grl_bias_table_f32(capi.ptr(t), t.shape[0], capi.ptr(_f32c(w1, "w1")), capi.ptr(b1),
                                             capi.ptr(_f32c(w2, "w2")), hidden, heads, capi.ptr(out), capi.stream()))
    return out


def affine_(attn, logit_scale, bias, index, mask):
    """In-place AffineTransform on a materialised (B_, heads, n1, n2) map."""
    attn = _f32c(attn, "attn")
    B_, H, n1, n2 = attn.shape
    nW = mask.shape[0] if mask is not None else 0
    capi.check(capi.lib().grl_affine_f32(capi.ptr(attn), B_, H, n1, n2, capi.ptr(logit_scale.reshape(-1)),
                                         capi.ptr(bias), bias.shape[1], capi.ptr(index.contiguous()),
                                         capi.ptr(_f32c(mask, "mask")) if mask is not None else None, nW,
                                         capi.stream()))
    return attn


def _token_rows(t, name):
    capi.require_device(t)
    if t.dtype != torch.float32 or t.dim() != 3 or t.stride(2) != 1 or t.stride(0) != t.shape[1] * t.stride(1):
        raise RuntimeError(f"grl_b200: {name} must be float32 (B, L, c) with unit channel stride and packed rows")
    return ctypes.c_void_p(t.data_ptr()), t.stride(1)


def window_attention(qkv, B, grid, heads, logit_scale, bias, use_mask, out=None):
    """qkv (B, L, 3c) view (window half) -> (B, L, c)."""
    qp, ldq = _token_rows(qkv, "qkv")
    c = qkv.shape[2] // 3
    if out is None:
        out = torch.empty(B, qkv.shape[1], c, device=qkv.device, dtype=torch.float32)
    op, ldo = _token_rows(out, "out")
    _timed("window_attn", lambda: capi.check(capi.lib().grl_window_attn_f32(
        qp, ldq, op, ldo, B, grid, heads, c // heads, capi.ptr(logit_scale.reshape(-1)), capi.ptr(bias),
        int(use_mask), capi.stream())))
    return out


def d8_index(mode, H, W, inverse=False):
    """Host expansion of the self-ensemble's view maps (CPU, no device needed).  inverse=False: (H', W') int32 flat
    source index y*W + x of every position of view `mode` = augment_img_tensor4(., mode) of an (H, W) image; inverse=True:
    (H, W) int32 flat index into the (H', W') view of every image pixel."""
    Hv, Wv = (W, H) if mode & 1 else (H, W)
    out = torch.empty((H, W) if inverse else (Hv, Wv), dtype=torch.int32)
    capi.check(capi.lib().grl_d8_index_host(int(mode), int(H), int(W), int(bool(inverse)),
                                            ctypes.c_void_p(out.data_ptr())))
    return out


def ens_gather(x, group, out=None):
    """x (B, C, H, W) fp32 -> the 4 views augment_img_tensor4(x, 2*i + group), i = 0..3, as (4B, C, H', W') view-major
    (index i*B + b); (H', W') = (W, H) for group 1."""
    x = _f32c(x, "x")
    B, C, H, W = x.shape
    shape = (4 * B, C) + ((W, H) if group else (H, W))
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    elif tuple(out.shape) != shape or out.dtype != torch.float32 or not out.is_contiguous():
        raise RuntimeError(f"grl_b200: ens_gather output must be contiguous float32 {shape}")
    capi.check(capi.lib().grl_ens_gather_f32(capi.ptr(x), B, C, H, W, int(group), capi.ptr(out), capi.stream()))
    return out


def ens_merge(ya, yb, B):
    """Self-ensemble average: ya (4B, C, Hs, Ws) outputs of views 0, 2, 4, 6 and yb (4B, C, Ws, Hs) of views 1, 3, 5, 7
    -> (B, C, Hs, Ws) = 0.125 * (V_0 + ... + V_7) in mode order, V_m = view m's output mapped back."""
    ya, yb = _f32c(ya, "ya"), _f32c(yb, "yb")
    n, C, Hs, Ws = ya.shape
    if n != 4 * B or tuple(yb.shape) != (n, C, Ws, Hs):
        raise RuntimeError(f"grl_b200: ens_merge needs (4B, C, Hs, Ws) and (4B, C, Ws, Hs) view outputs, got "
                           f"{tuple(ya.shape)} / {tuple(yb.shape)} for B={B}")
    y = torch.empty(B, C, Hs, Ws, device=ya.device, dtype=torch.float32)
    capi.check(capi.lib().grl_ens_merge_f32(capi.ptr(ya), capi.ptr(yb), B, C, Hs, Ws, capi.ptr(y), capi.stream()))
    return y


def _cfa4(x):
    x = _f32c(x, "cfa4")
    if x.dim() != 4 or x.shape[1] != 4 or x.shape[2] < 2 or x.shape[3] < 2:
        raise ValueError(f"grl_b200: packed RGGB Bayer planes must be (B, 4, h, w) with h, w >= 2, got {tuple(x.shape)}")
    return x


def demosaic(x, out=None):
    """The reference's dm_matlab (utils/utils_mosaic.py:36-111), the dm task's input transform (engines/base.py:127-128):
    packed RGGB planes x (B, 4, h, w) float32 on the GPU (R, G of the even rows, G of the odd rows, B) -> RGB
    (B, 3, 2h, 2w) float32.  One sm_90a kernel; GRL(input_format="rggb") fuses the same arithmetic into its head."""
    x = _cfa4(x)
    B, _, h, w = x.shape
    y = out if out is not None else torch.empty(B, 3, 2 * h, 2 * w, device=x.device, dtype=torch.float32)
    capi.check(capi.lib().grl_demosaic_f32(capi.ptr(x), B, h, w, capi.ptr(y), capi.stream()))
    return y


def demosaic_host(x):
    """demosaic evaluated on the CPU by the library's host copy of the same closed form (tests)."""
    x = x.float().contiguous()
    B, _, h, w = x.shape
    y = torch.empty(B, 3, 2 * h, 2 * w, dtype=torch.float32)
    capi.check(capi.lib().grl_demosaic_host(ctypes.c_void_p(x.data_ptr()), B, h, w, ctypes.c_void_p(y.data_ptr())))
    return y


def u8_to_f32(img):
    """Decoded 8-bit images (B, H, W, C) uint8 on the GPU, 1 <= C <= 8 -> (B, C, H, W) float32 = k / 255, correctly
    rounded: what every dataset's transforms.functional.to_tensor gives (img.float().div(255) on the CPU).  One kernel."""
    capi.require_device(img)
    if img.dtype != torch.uint8 or img.dim() != 4 or not 1 <= img.shape[3] <= 8:
        raise RuntimeError(f"grl_b200: u8_to_f32 needs (B, H, W, C) uint8 images with 1 <= C <= 8, got {img.dtype} "
                           f"{tuple(img.shape)}")
    img = img.contiguous()
    B, H, W, C = img.shape
    y = torch.empty(B, C, H, W, device=img.device, dtype=torch.float32)
    capi.check(capi.lib().grl_u8_to_f32(capi.ptr(img), B, H, W, C, capi.ptr(y), capi.stream()))
    return y


def f32_to_u8(y):
    """(B, C, H, W) float32 on the GPU, 1 <= C <= 8 -> (B, H, W, C) uint8 = round(clamp(v, 0, 1) * 255) with ties to
    even: the validation step's tensor_round times 255, the bytes of a saved image.  NaN gives 0.  One kernel."""
    y = _f32c(y, "y")
    if y.dim() != 4 or not 1 <= y.shape[1] <= 8:
        raise RuntimeError(f"grl_b200: f32_to_u8 needs (B, C, H, W) float32 images with 1 <= C <= 8, got {tuple(y.shape)}")
    B, C, H, W = y.shape
    img = torch.empty(B, H, W, C, device=y.device, dtype=torch.uint8)
    capi.check(capi.lib().grl_f32_to_u8(capi.ptr(y), B, C, H, W, capi.ptr(img), capi.stream()))
    return img


def u8_to_f32_host(img):
    """u8_to_f32 evaluated on the CPU by the library's host copy of the same closed form (tests)."""
    img = img.contiguous()
    B, H, W, C = img.shape
    y = torch.empty(B, C, H, W, dtype=torch.float32)
    capi.check(capi.lib().grl_u8_to_f32_host(ctypes.c_void_p(img.data_ptr()), B, H, W, C, ctypes.c_void_p(y.data_ptr())))
    return y


def f32_to_u8_host(y):
    """f32_to_u8 evaluated on the CPU by the library's host copy of the same closed form (tests)."""
    y = y.float().contiguous()
    B, C, H, W = y.shape
    img = torch.empty(B, H, W, C, dtype=torch.uint8)
    capi.check(capi.lib().grl_f32_to_u8_host(ctypes.c_void_p(y.data_ptr()), B, C, H, W, ctypes.c_void_p(img.data_ptr())))
    return img


def _image_refs(images, kind):
    refs = (capi.GrlImageRef * max(1, len(images)))()
    for r, t in zip(refs, images):
        h, w = t.shape[:2] if kind == capi.IMAGE_U8 else t.shape[1:]
        r.data, r.H, r.W, r.kind = t.data_ptr(), h, w, kind
    return refs


def list_gather(images, kind, C, Hp, Wp):
    """check_image_size of every image into one padded batch (n, C, Hp, Wp) float32: reflect padding on the bottom /
    right, zeros on both axes when a pad is not smaller than its axis (grl.py:479-489).  images: contiguous tensors on
    the GPU, all of `kind`: capi.IMAGE_F32 (C, H, W) float32, capi.IMAGE_U8 (H, W, C) uint8 (k / 255 as u8_to_f32) or
    capi.IMAGE_RGGB (4, h, w) float32 packed Bayer planes (demosaiced as K.demosaic, C = 3).  Needs (H, W) <= (Hp, Wp)."""
    want = torch.uint8 if kind == capi.IMAGE_U8 else torch.float32
    want_c = {capi.IMAGE_U8: (2, C), capi.IMAGE_RGGB: (0, 4)}.get(kind, (0, C))  # (channel dim, channels)
    for t in images:
        capi.require_device(t)
        if t.dtype != want or t.dim() != 3 or not t.is_contiguous() or t.shape[want_c[0]] != want_c[1]:
            raise RuntimeError(f"grl_b200: list_gather needs contiguous {want} images of {C} channels (kind {kind}), got "
                               f"{t.dtype} {tuple(t.shape)}")
    dev = torch.device("cuda", torch.cuda.current_device()) if not images else images[0].device
    out = torch.empty(len(images), C, Hp, Wp, device=dev, dtype=torch.float32)
    capi.check(capi.lib().grl_list_gather(_image_refs(images, kind), len(images), C, Hp, Wp, capi.ptr(out), capi.stream()))
    return out


def list_crop(y, sizes, u8=False):
    """The top-left (H_i, W_i) corner of every image of a batch y (n, C, Hy, Wy) float32 on the GPU, as a list of
    (C, H_i, W_i) float32 tensors, or with u8 of (H_i, W_i, C) uint8 tensors as f32_to_u8 gives them."""
    y = _f32c(y, "y")
    n, C, Hy, Wy = y.shape
    if len(sizes) != n:
        raise RuntimeError(f"grl_b200: list_crop got {len(sizes)} sizes for a batch of {n}")
    outs = [torch.empty((h, w, C) if u8 else (C, h, w), device=y.device, dtype=torch.uint8 if u8 else torch.float32)
            for h, w in sizes]
    kind = capi.IMAGE_U8 if u8 else capi.IMAGE_F32
    capi.check(capi.lib().grl_list_crop(capi.ptr(y), n, C, Hy, Wy, _image_refs(outs, kind), capi.stream()))
    return outs


def tile_gather(tiles, kind, C, Hp, Wp):
    """check_image_size of tile windows into one padded batch (n, C, Hp, Wp) float32, as list_gather pads whole images.
    tiles: (image, y0, x0, t) with image a contiguous tensor on the GPU of `kind` (see list_gather) and the t x t window
    at (y0, x0) of the frame the network sees (capi.IMAGE_RGGB: of the demosaiced (2h, 2w) frame).  Hp = Wp = t cuts."""
    refs = (capi.GrlTileRef * max(1, len(tiles)))()
    for r, (img, y0, x0, t) in zip(refs, tiles):
        capi.require_device(img)
        if not img.is_contiguous() or img.dtype != (torch.uint8 if kind == capi.IMAGE_U8 else torch.float32):
            raise RuntimeError(f"grl_b200: tile_gather needs contiguous sources of kind {kind}, got {img.dtype}")
        h, w = img.shape[:2] if kind == capi.IMAGE_U8 else img.shape[1:]
        r.src.data, r.src.H, r.src.W, r.src.kind = img.data_ptr(), h, w, kind
        r.y0, r.x0, r.t = y0, x0, t
    dev = torch.device("cuda", torch.cuda.current_device()) if not tiles else tiles[0][0].device
    out = torch.empty(len(tiles), C, Hp, Wp, device=dev, dtype=torch.float32)
    capi.check(capi.lib().grl_tile_gather(refs, len(tiles), C, Hp, Wp, capi.ptr(out), capi.stream()))
    return out


def _tile_images(blends, C, scale, outs_u8=None):
    refs = (capi.GrlTileImage * max(1, len(blends)))()
    for j, (r, (E, t, overlap, k0, k1, slot)) in enumerate(zip(refs, blends)):
        capi.require_device(E)
        if (E.dtype != torch.float32 or E.dim() != 3 or not E.is_contiguous() or E.shape[0] != C or E.shape[1] % scale
                or E.shape[2] % scale):
            raise RuntimeError(f"grl_b200: a tile accumulator must be contiguous float32 ({C}, H*{scale}, W*{scale}), got "
                               f"{E.dtype} {tuple(E.shape)}")
        r.E, r.H, r.W = E.data_ptr(), E.shape[1] // scale, E.shape[2] // scale
        r.t, r.overlap, r.k0, r.k1, r.slot = t, overlap, k0, k1, slot
        if outs_u8 is not None:
            o = outs_u8[j]
            capi.require_device(o)
            if o.dtype != torch.uint8 or not o.is_contiguous() or tuple(o.shape) != (E.shape[1], E.shape[2], E.shape[0]):
                raise RuntimeError(f"grl_b200: tile_finish needs contiguous uint8 (H*s, W*s, C) outputs, got {o.dtype} "
                                   f"{tuple(o.shape)} for an accumulator {tuple(E.shape)}")
            r.out_u8 = o.data_ptr()
    return refs


def tile_accumulate(y, blends, scale):
    """Adds the tile outputs of a batch y (n, C, Hy, Wy) float32 (the forward of a tile_gather batch) to their images'
    accumulators, as the reference's E[...].add_(o) in origin order.  blends: (E, t, overlap, k0, k1, slot) per image with
    tiles in the batch: E (C, H*scale, W*scale) float32, the image's tiles k0..k1-1 (row-major over its origin grid) at
    batch indices slot, slot + 1, ...; tile k's output is the top-left (t*scale)^2 of its entry."""
    y = _f32c(y, "y")
    n, C, Hy, Wy = y.shape
    capi.check(capi.lib().grl_tile_accumulate(capi.ptr(y), n, C, Hy, Wy, int(scale), _tile_images(blends, C, scale),
                                              len(blends), capi.stream()))


def tile_finish(blends, scale, outs_u8=None):
    """E / W of the reference for every image: blends (E, t, overlap) per image; E becomes E / (number of tiles covering
    the pixel), IEEE division, in place, or with outs_u8 the (H*s, W*s, C) uint8 outputs receive round8 of it."""
    C = blends[0][0].shape[0] if blends else 1
    refs = _tile_images([(E, t, overlap, 0, 0, 0) for E, t, overlap in blends], C, scale, outs_u8)
    capi.check(capi.lib().grl_tile_finish(refs, len(blends), C, int(scale), capi.stream()))


def tile_cover_host(size, tile, overlap, scale=1):
    """(size*scale, 2) int32: the first and last tile, in origin order, covering each output row (CPU, no device)."""
    out = torch.empty(size * scale, 2, dtype=torch.int32)
    capi.check(capi.lib().grl_tile_cover_host(int(size), int(tile), int(overlap), int(scale), ctypes.c_void_p(out.data_ptr())))
    return out


def _jpeg_quality(quality):
    if isinstance(quality, bool) or not isinstance(quality, int) or not 1 <= quality <= 100:
        raise ValueError(f"grl_b200: JPEG quality must be an int in 1..100, got {quality!r}")
    return quality


def _jpeg_images(images, what):
    """The list checks of jpeg_roundtrip_list and awgn_list: (H, W, C) uint8 on the current CUDA device, one C in
    {1, 3}."""
    C = None
    for i, t in enumerate(images):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"grl_b200: {what}: element {i} is a {type(t).__name__}, not a tensor")
        capi.require_device(t)
        if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] not in (1, 3) or t.shape[0] < 1 or t.shape[1] < 1:
            raise ValueError(f"grl_b200: {what} needs (H, W, C) uint8 images with C in {{1, 3}}, got element {i}: {t.dtype} "
                             f"{tuple(t.shape)}")
        if C is not None and t.shape[2] != C:
            raise ValueError(f"grl_b200: {what}: element {i} has {t.shape[2]} channels, element 0 {C}: one C per call")
        C = t.shape[2]
    return C


def _jpeg_launch(srcs, dsts, C, quality):
    src, dst = _image_refs(srcs, capi.IMAGE_U8), _image_refs(dsts, capi.IMAGE_U8)
    nbytes = capi.lib().grl_jpeg_workspace(src, len(srcs), C)
    ws = torch.empty(max(nbytes, 1), device=srcs[0].device, dtype=torch.uint8)
    capi.check(capi.lib().grl_jpeg_roundtrip_u8(src, dst, len(srcs), C, quality, capi.ptr(ws), nbytes, capi.stream()))


def jpeg_roundtrip(img, quality):
    """The JPEG test command's degraded input (JPEGDataset.jpeg_compress, data/datasets/restoration_jpeg.py:62-79):
    (B, H, W, C) uint8 images on the GPU, C = 1 (gray) or 3 (RGB) -> new (B, H, W, C) uint8 tensor, each image equal byte
    for byte to cv2.imdecode(cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, quality])) (colour via BGR, as the dataset
    does): libjpeg's baseline 4:2:0 encode and default decode.  quality: int in 1..100.  Two kernels (one for gray)."""
    quality = _jpeg_quality(quality)
    if not isinstance(img, torch.Tensor):
        raise ValueError(f"grl_b200: jpeg_roundtrip needs a tensor, got {type(img).__name__}")
    capi.require_device(img)
    if img.dtype != torch.uint8 or img.dim() != 4 or img.shape[3] not in (1, 3) or min(img.shape[1:3]) < 1:
        raise ValueError(f"grl_b200: jpeg_roundtrip needs (B, H, W, C) uint8 images with C in {{1, 3}}, got {img.dtype} "
                         f"{tuple(img.shape)}")
    img = img.contiguous()
    out = torch.empty_like(img)
    if img.shape[0]:
        _jpeg_launch(list(img.unbind(0)), list(out.unbind(0)), img.shape[3], quality)
    return out


def jpeg_roundtrip_list(images, quality):
    """jpeg_roundtrip of a list of differently sized (H_i, W_i, C) uint8 images on the GPU, all with the same C in {1, 3}
    -> list of new tensors in input order.  The whole list runs in two kernels per 80 images (one for gray)."""
    quality = _jpeg_quality(quality)
    images = list(images)
    C = _jpeg_images(images, "jpeg_roundtrip_list")
    if not images:
        return []
    srcs = [t.contiguous() for t in images]
    outs = [torch.empty_like(t) for t in srcs]
    _jpeg_launch(srcs, outs, C, quality)
    return outs


def jpeg_roundtrip_host(img, quality):
    """jpeg_roundtrip of one (H, W, C) uint8 CPU image, evaluated by the library's host copy of the same closed forms
    (tests)."""
    quality = _jpeg_quality(quality)
    if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] not in (1, 3):
        raise ValueError(f"grl_b200: jpeg_roundtrip_host needs an (H, W, C) uint8 image with C in {{1, 3}}, got {img.dtype} "
                         f"{tuple(img.shape)}")
    img = img.contiguous()
    out = torch.empty_like(img)
    H, W, C = img.shape
    capi.check(capi.lib().grl_jpeg_roundtrip_host(ctypes.c_void_p(img.data_ptr()), H, W, C, quality,
                                                  ctypes.c_void_p(out.data_ptr())))
    return out


def jpeg_quant_tables(quality):
    """(2, 64) int32 CPU tensor: the luma and chroma quantisation tables the round trip uses at this quality
    (jpeg_set_quality with baseline limits), natural row-major order."""
    out = torch.empty(2, 64, dtype=torch.int32)
    capi.check(capi.lib().grl_jpeg_quant_tables_host(_jpeg_quality(quality), ctypes.c_void_p(out.data_ptr())))
    return out


def dn_seed(path):
    """The RandomState key of the denoising test command's noise for one image (DnDataset.__getitem__,
    data/datasets/restoration_dn.py:136-140): (8,) uint32 numpy array = the words of sha256(path.split("_")[0]), as
    np.frombuffer(digest, dtype="uint32") gives them.  `path` is the dataset-relative path the reference keys on, e.g.
    "CBSD68/0001.png".  The reference cuts the path at its first "_", and so does this: every Urban100 image
    ("Urban100/img_001.png", "Urban100/img_092.png", ...) gets the key of "Urban100/img", so all of them draw the same
    noise stream."""
    import hashlib

    import numpy as np

    if not isinstance(path, str):
        raise ValueError(f"grl_b200: dn_seed needs a path string, got {type(path).__name__}")
    return np.frombuffer(hashlib.sha256(path.split("_")[0].encode("utf-8")).digest(), dtype="uint32").copy()


def _awgn_scale(noise_sigma):
    """noise_sigma / 255 in Python double, as the reference divides the config's sigma."""
    import math
    import numbers

    if isinstance(noise_sigma, bool) or not isinstance(noise_sigma, numbers.Real) or not math.isfinite(noise_sigma) \
            or noise_sigma < 0:
        raise ValueError(f"grl_b200: noise_sigma must be a finite real >= 0, got {noise_sigma!r}")
    return noise_sigma / 255


def _awgn_keys(seeds, n, what):
    """(n, 8) uint32 host array of RandomState keys: a path string goes through dn_seed, anything else must be 8 integers
    in [0, 2^32)."""
    import numpy as np

    seeds = list(seeds)
    if len(seeds) != n:
        raise ValueError(f"grl_b200: {what}: {len(seeds)} seeds for {n} images")
    keys = np.empty((n, 8), dtype=np.uint32)
    for i, s in enumerate(seeds):
        if isinstance(s, str):
            keys[i] = dn_seed(s)
            continue
        a = np.asarray(s.cpu() if isinstance(s, torch.Tensor) else s)
        if a.shape != (8,) or a.dtype.kind not in "iu" or (a.astype(np.int64) < 0).any() or (a.astype(np.int64) >> 32).any():
            raise ValueError(f"grl_b200: {what}: seed {i} must be a path string or 8 integers in [0, 2^32), got {s!r}")
        keys[i] = a
    return keys


def _awgn_launch(srcs, dsts, keys, C, scale):
    src, dst = _image_refs(srcs, capi.IMAGE_U8), _image_refs(dsts, capi.IMAGE_F32)
    capi.check(capi.lib().grl_awgn_u8(src, dst, keys.ctypes.data_as(ctypes.c_void_p), len(srcs), C, scale,
                                      capi.stream()))


def awgn(img, noise_sigma, seeds):
    """The denoising test command's noisy input (DnDataset.__getitem__, validation branch,
    data/datasets/restoration_dn.py:134-143): (B, H, W, C) uint8 images on the GPU, C = 1 or 3 -> new (B, C, H, W) float32
    tensor, image b equal bit for bit to to_tensor(img[b]) + torch.from_numpy(np.random.RandomState(key_b).normal(0,
    noise_sigma / 255, (C, H, W))).float().  noise_sigma: the config's sigma (15 for the released checkpoints), a finite
    real >= 0.  seeds: one per image, a dataset-relative path (through dn_seed) or 8 uint32 words.  The reference's crop
    to multiples of 8 stays with the caller: g[:H // 8 * 8, :W // 8 * 8].  One kernel per 64 images."""
    scale = _awgn_scale(noise_sigma)
    if not isinstance(img, torch.Tensor):
        raise ValueError(f"grl_b200: awgn needs a tensor, got {type(img).__name__}")
    capi.require_device(img)
    if img.dtype != torch.uint8 or img.dim() != 4 or img.shape[3] not in (1, 3) or min(img.shape[1:3]) < 1:
        raise ValueError(f"grl_b200: awgn needs (B, H, W, C) uint8 images with C in {{1, 3}}, got {img.dtype} "
                         f"{tuple(img.shape)}")
    keys = _awgn_keys(seeds, img.shape[0], "awgn")
    img = img.contiguous()
    B, H, W, C = img.shape
    out = torch.empty(B, C, H, W, device=img.device, dtype=torch.float32)
    if B:
        _awgn_launch(list(img.unbind(0)), list(out.unbind(0)), keys, C, scale)
    return out


def awgn_list(images, noise_sigma, seeds):
    """awgn of a list of differently sized (H_i, W_i, C) uint8 images on the GPU, all with the same C in {1, 3}, one seed
    per image -> list of new (C, H_i, W_i) float32 tensors in input order.  The whole list runs in one kernel per 64
    images, one CTA per image."""
    scale = _awgn_scale(noise_sigma)
    images = list(images)
    C = _jpeg_images(images, "awgn_list")
    keys = _awgn_keys(seeds, len(images), "awgn_list")
    if not images:
        return []
    srcs = [t.contiguous() for t in images]
    outs = [torch.empty(C, t.shape[0], t.shape[1], device=t.device, dtype=torch.float32) for t in srcs]
    _awgn_launch(srcs, outs, keys, C, scale)
    return outs


def awgn_noise_host(seed, count, noise_sigma):
    """The noise alone, from the library's host copy of the same closed forms with libm's log, as numpy's (tests):
    (count,) float64 CPU tensor = np.random.RandomState(key).normal(0, noise_sigma / 255, count)."""
    scale = _awgn_scale(noise_sigma)
    key = _awgn_keys([seed], 1, "awgn_noise_host")
    if isinstance(count, bool) or not isinstance(count, int) or count < 0:
        raise ValueError(f"grl_b200: awgn_noise_host: count must be an int >= 0, got {count!r}")
    out = torch.empty(count, dtype=torch.float64)
    capi.check(capi.lib().grl_awgn_noise_host(key.ctypes.data_as(ctypes.c_void_p), count, scale,
                                              ctypes.c_void_p(out.data_ptr())))
    return out


def awgn_log_host(x):
    """The device's double-double log of the polar method (awgn_log_cr, csrc/grl_awgn.h), evaluated on the CPU (tests):
    x float64 CPU tensor of positive normal numbers -> log(x), correctly rounded but for inputs within about 2^-100 of a
    rounding midpoint."""
    x = x.to(torch.float64).contiguous()
    out = torch.empty_like(x)
    capi.check(capi.lib().grl_awgn_log_host(ctypes.c_void_p(x.data_ptr()), x.numel(), ctypes.c_void_p(out.data_ptr())))
    return out


def _rgb_u8_images(images, what):
    """The list checks of mosaic_list and luma_list: (H, W, 3) uint8 on the current CUDA device."""
    for i, t in enumerate(images):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"grl_b200: {what}: element {i} is a {type(t).__name__}, not a tensor")
        capi.require_device(t)
        if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3 or t.shape[0] < 1 or t.shape[1] < 1:
            raise ValueError(f"grl_b200: {what} needs (H, W, 3) uint8 RGB images, got element {i}: {t.dtype} "
                             f"{tuple(t.shape)}")


def _rgb_u8_batch(img, what):
    if not isinstance(img, torch.Tensor):
        raise ValueError(f"grl_b200: {what} needs a tensor, got {type(img).__name__}")
    capi.require_device(img)
    if img.dtype != torch.uint8 or img.dim() != 4 or img.shape[3] != 3 or min(img.shape[1:3]) < 1:
        raise ValueError(f"grl_b200: {what} needs (B, H, W, 3) uint8 RGB images, got {img.dtype} {tuple(img.shape)}")
    return img.contiguous()


def _mosaic_launch(srcs, outs):
    capi.check(capi.lib().grl_mosaic_u8(_image_refs(srcs, capi.IMAGE_U8), _image_refs(outs, capi.IMAGE_RGGB), len(srcs),
                                        capi.stream()))


def mosaic(img):
    """The demosaicking test command's input (DemosaicDataset.__getitem__, data/datasets/restoration_dm.py:33-37):
    (B, H, W, 3) uint8 RGB images on the GPU -> new (B, 4, H // 2, W // 2) float32 packed RGGB planes (R, G of the even
    rows, G of the odd rows, B), equal bit for bit to to_tensor(mosaic_CFA_Bayer(img[b])[1]); an odd last row or column is
    dropped.  What GRL(input_format="rggb") takes.  One kernel per 128 images."""
    img = _rgb_u8_batch(img, "mosaic")
    B, H, W, _ = img.shape
    out = torch.empty(B, 4, H // 2, W // 2, device=img.device, dtype=torch.float32)
    if B:
        _mosaic_launch(list(img.unbind(0)), list(out.unbind(0)))
    return out


def mosaic_list(images):
    """mosaic of a list of differently sized (H_i, W_i, 3) uint8 images on the GPU -> list of new (4, H_i // 2, W_i // 2)
    float32 tensors in input order, what GRL(input_format="rggb").forward_list takes.  One kernel per 128 images."""
    images = list(images)
    _rgb_u8_images(images, "mosaic_list")
    if not images:
        return []
    srcs = [t.contiguous() for t in images]
    outs = [torch.empty(4, t.shape[0] // 2, t.shape[1] // 2, device=t.device, dtype=torch.float32) for t in srcs]
    _mosaic_launch(srcs, outs)
    return outs


def mosaic_host(img):
    """mosaic of one (H, W, 3) uint8 CPU image, evaluated by the library's host copy of the same closed form (tests)."""
    if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
        raise ValueError(f"grl_b200: mosaic_host needs an (H, W, 3) uint8 image, got {img.dtype} {tuple(img.shape)}")
    img = img.contiguous()
    H, W, _ = img.shape
    out = torch.empty(4, H // 2, W // 2, dtype=torch.float32)
    capi.check(capi.lib().grl_mosaic_host(ctypes.c_void_p(img.data_ptr()), H, W, ctypes.c_void_p(out.data_ptr())))
    return out


def _luma_launch(srcs, outs):
    capi.check(capi.lib().grl_luma_u8(_image_refs(srcs, capi.IMAGE_U8), _image_refs(outs, capi.IMAGE_U8), len(srcs),
                                      capi.stream()))


def luma(img):
    """The gray JPEG test command's clean image on LIVE1 / BSDS500 / Urban100 (base_image.imread,
    data/datasets/base_image.py:233-241): (B, H, W, 3) uint8 RGB images on the GPU -> new (B, H, W, 1) uint8, equal byte for
    byte to rgb2ycbcr_np(img[b], y_only=True) (MATLAB's rgb2ycbcr luma of k / 255, rounded half to even).  One kernel per
    128 images."""
    img = _rgb_u8_batch(img, "luma")
    out = torch.empty(*img.shape[:3], 1, device=img.device, dtype=torch.uint8)
    if img.shape[0]:
        _luma_launch(list(img.unbind(0)), list(out.unbind(0)))
    return out


def luma_list(images):
    """luma of a list of differently sized (H_i, W_i, 3) uint8 images on the GPU -> list of new (H_i, W_i, 1) uint8
    tensors in input order.  One kernel per 128 images."""
    images = list(images)
    _rgb_u8_images(images, "luma_list")
    if not images:
        return []
    srcs = [t.contiguous() for t in images]
    outs = [torch.empty(t.shape[0], t.shape[1], 1, device=t.device, dtype=torch.uint8) for t in srcs]
    _luma_launch(srcs, outs)
    return outs


def luma_host(rgb):
    """luma of (..., 3) uint8 CPU pixels -> (..., 1) uint8, evaluated by the library's host copy of the same closed form
    (tests)."""
    if rgb.dtype != torch.uint8 or rgb.dim() < 1 or rgb.shape[-1] != 3:
        raise ValueError(f"grl_b200: luma_host needs (..., 3) uint8 pixels, got {rgb.dtype} {tuple(rgb.shape)}")
    rgb = rgb.contiguous()
    out = torch.empty(*rgb.shape[:-1], 1, dtype=torch.uint8)
    capi.check(capi.lib().grl_luma_host(ctypes.c_void_p(rgb.data_ptr()), out.numel(), ctypes.c_void_p(out.data_ptr())))
    return out


def stripe_attention(qkv, anchor, B, tok_grid, anc_grid, heads, scale1, bias1, scale2, bias2, use_mask, out=None):
    """qkv (B, L, 3c) view (stripe half), anchor (B, Ha, Wa, c) -> (B, L, c)."""
    qp, ldq = _token_rows(qkv, "qkv")
    c = qkv.shape[2] // 3
    anchor = _f32c(anchor, "anchor")
    if out is None:
        out = torch.empty(B, qkv.shape[1], c, device=qkv.device, dtype=torch.float32)
    op, ldo = _token_rows(out, "out")
    d = c // heads
    nbytes = capi.lib().grl_stripe_attn_workspace(B, tok_grid, anc_grid, heads, d)
    ws = torch.empty(max(nbytes, 4) // 4, device=qkv.device, dtype=torch.float32)
    _timed("stripe_attn", lambda: capi.check(capi.lib().grl_stripe_attn_f32(
        qp, ldq, capi.ptr(anchor), c, op, ldo, B, tok_grid, anc_grid, heads, d, capi.ptr(scale1.reshape(-1)),
        capi.ptr(bias1), capi.ptr(scale2.reshape(-1)), capi.ptr(bias2), int(use_mask), capi.ptr(ws), nbytes,
        capi.stream())))
    return out
