"""Tiled inference with overlap averaging -- the engine's `forward_tile` (engines/base.py:90-116) with all tiles of the
image(s) batched into a few forwards instead of a Python double loop of single-tile forwards, and (forward_tile_sharded)
with the tiles of one frame spread over the ranks of a process group (SURVEY.md 8e: BASELINE cfg5, one 1280x720 frame
on 8 GPUs).

Semantics are the reference's exactly: tile = min(tile, h, w); origins range(0, h - tile, stride) + [h - tile] with
stride = tile - overlap (same for w); every tile is restored independently (so per-tile operators such as the CAB
global pool see the same data as in the reference), outputs are summed into E, a ones mask into W, result E / W.

forward_tile_list / forward_tile_list_u8 do the same for a list of differently sized images, with the tiles of the
whole list sharing forwards and the cut and blend on the device (csrc/image_list.cu, csrc/grl_tiles.h).
"""
import torch

from . import capi, image_list
from . import functional as K


def _rgb_frame(model, x):
    """A model that takes packed Bayer planes (GRL input_format="rggb") is tiled on the demosaiced frame, the engine's
    order (engines/base.py:127-128 before :90-116): demosaicing each tile on its own would reflect at the tile edges and
    change the pixels there.  Returns the per-tile callable and the frame to cut."""
    if getattr(model, "input_format", "rgb") == "rggb":
        return model.forward_rgb, K.demosaic(x.float().contiguous()).to(x.dtype)
    return model, x


def tile_origins(size, tile, overlap):
    stride = tile - overlap
    return list(range(0, size - tile, stride)) + [size - tile]


def _origins(b, h, w, tile, tile_overlap):
    hs, ws = tile_origins(h, tile, tile_overlap), tile_origins(w, tile, tile_overlap)
    return [(bi, hi, wi) for bi in range(b) for hi in hs for wi in ws]


def _accumulate(E, W, origins, outs, tile, scale):
    for (bi, hi, wi), o in zip(origins, outs):
        E[bi, :, hi * scale:(hi + tile) * scale, wi * scale:(wi + tile) * scale].add_(o)
        W[bi, :, hi * scale:(hi + tile) * scale, wi * scale:(wi + tile) * scale].add_(1.0)


@torch.no_grad()
def forward_tile(model, x, tile, tile_overlap, scale=None, max_batch=16):
    """x (B, C, H, W) on the GPU -> (B, C_out, H*scale, W*scale); for an input_format="rggb" model x is (B, 4, H/2, W/2)
    and the result is that of the demosaiced (H, W) frame."""
    scale = model.upscale if scale is None else scale
    fn, x = _rgb_frame(model, x)
    b, _, h, w = x.shape
    tile = min(tile, h, w)
    origins = _origins(b, h, w, tile, tile_overlap)
    E = W = None
    for i in range(0, len(origins), max_batch):
        chunk = origins[i:i + max_batch]
        patches = torch.stack([x[bi, :, hi:hi + tile, wi:wi + tile] for bi, hi, wi in chunk])
        out = fn(patches)
        if E is None:
            E = torch.zeros(b, out.shape[1], h * scale, w * scale, device=x.device, dtype=out.dtype)
            W = torch.zeros_like(E)
        _accumulate(E, W, chunk, out, tile, scale)
    return E.div_(W)


def shard_tiles(n_tiles, rank, world):
    """Round-robin assignment of tile indices to ranks (tiles of one frame cost the same: balanced to within one)."""
    return list(range(rank, n_tiles, world))


@torch.no_grad()
def forward_tile_sharded(model, x, tile, tile_overlap, scale=None, max_batch=16, group=None):
    """forward_tile with the tiles spread round-robin over the ranks of `group` (one process per GPU; every rank holds
    the whole input frame x and the replicated weights).  Each rank restores its tiles, one all-gather moves the
    restored tiles (NCCL over NVLink; 6 x 3 x 480^2 fp32 = 16.6 MB for the 1280x720 deblur frame), and every rank
    assembles E / W, so the result is identical on all ranks and identical to forward_tile.  `model` is any callable
    (B', C, t, t) -> (B', C_out, t*scale, t*scale); without an initialised process group this is forward_tile."""
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return forward_tile(model, x, tile, tile_overlap, scale=scale, max_batch=max_batch)
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    scale = model.upscale if scale is None else scale
    c_model = getattr(model, "out_channels", None)
    fn, x = _rgb_frame(model, x)
    b, _, h, w = x.shape
    tile = min(tile, h, w)
    origins = _origins(b, h, w, tile, tile_overlap)
    mine = shard_tiles(len(origins), rank, world)
    per_rank = (len(origins) + world - 1) // world
    outs = []
    for i in range(0, len(mine), max_batch):
        chunk = [origins[j] for j in mine[i:i + max_batch]]
        patches = torch.stack([x[bi, :, hi:hi + tile, wi:wi + tile] for bi, hi, wi in chunk])
        outs.append(fn(patches))
    if outs:
        local = torch.cat(outs)
        c_out, dtype = local.shape[1], local.dtype
    else:  # more ranks than tiles: this rank only takes part in the exchange
        c_out, dtype = c_model if c_model is not None else x.shape[1], x.dtype
        local = torch.zeros(0, c_out, tile * scale, tile * scale, device=x.device, dtype=dtype)
    send = torch.zeros(per_rank, c_out, tile * scale, tile * scale, device=x.device, dtype=dtype)
    send[: local.shape[0]] = local
    recv = torch.empty(world * per_rank, c_out, tile * scale, tile * scale, device=x.device, dtype=dtype)
    dist.all_gather_into_tensor(recv, send, group=group)
    E = torch.zeros(b, c_out, h * scale, w * scale, device=x.device, dtype=dtype)
    W = torch.zeros_like(E)
    for r in range(world):
        idx = shard_tiles(len(origins), r, world)
        _accumulate(E, W, [origins[j] for j in idx], recv[r * per_rank: r * per_rank + len(idx)], tile, scale)
    return E.div_(W)


@torch.no_grad()
def forward_tile_u8(model, img, tile, tile_overlap, scale=None, max_batch=16, group=None):
    """forward_tile_sharded on decoded 8-bit images: img (B, H, W, C) uint8 on the GPU -> (B, H*scale, W*scale, C_out)
    uint8 = f32_to_u8(forward_tile_sharded(model, u8_to_f32(img), ...)); without a process group that is forward_tile.
    Packed 8-bit Bayer input (a model with input_format="rggb") is not supported."""
    if getattr(model, "input_format", "rgb") == "rggb":
        raise ValueError("forward_tile_u8 takes (B, H, W, C) 8-bit images; packed 8-bit Bayer input "
                         "(input_format='rggb') is not supported")
    y = forward_tile_sharded(model, K.u8_to_f32(img), tile, tile_overlap, scale=scale, max_batch=max_batch, group=group)
    return K.f32_to_u8(y)


def tile_plan(model, sizes, tile, tile_overlap):
    """The tiles of a list of images of network sizes `sizes` (image_list.network_sizes) and the forwards that restore
    them; needs no device.  Returns (tiles, chunks): tiles are (image, y0, x0, t), t = min(tile, H, W), in forward_tile's
    order: image, then row origin, then column origin (tile_origins).  chunks are image_list.plan of the tiles' (t, t)
    sizes, chunk.index indexing `tiles`: by model.pad_size, so that tiles of one padded size share a forward of at most
    model.max_batch_tokens padded pixels; with self_ensemble by exact size (pad size 1), because forward_rgb pads each of
    a tile's 8 views on its own.
    The blend is exact only if each image's tiles reach it in origin order, and they do: all tiles of an image have one
    size, so they fall in one group, and plan keeps input order within a group and cuts it into consecutive chunks."""
    tiles = []
    for i, (h, w) in enumerate(sizes):
        t = min(tile, h, w)
        tiles += [(i, y0, x0, t) for y0 in tile_origins(h, t, tile_overlap) for x0 in tile_origins(w, t, tile_overlap)]
    pad = 1 if model.self_ensemble else model.pad_size
    return tiles, image_list.plan([(t, t) for *_, t in tiles], pad, model.max_batch_tokens)


def _check_tiles(sizes, tile, tile_overlap, what):
    if tile < 1 or tile_overlap < 0:
        raise ValueError(f"{what}: tile = {tile}, tile_overlap = {tile_overlap}: needs tile >= 1 and tile_overlap >= 0")
    for i, (h, w) in enumerate(sizes):
        t = min(tile, h, w)
        if t <= tile_overlap:  # stride <= 0, or pixels no tile covers
            raise ValueError(f"{what}: element {i} ({h} x {w}) is tiled with side min(tile, H, W) = {t}, which needs to be "
                             f"larger than tile_overlap = {tile_overlap}")


@torch.no_grad()
def _forward_tile_list(model, images, tile, tile_overlap, u8):
    what = "forward_tile_list_u8" if u8 else "forward_tile_list"
    rggb = model.input_format == "rggb"
    if u8 and rggb:
        raise ValueError(f"{what} takes (H, W, C) 8-bit images; packed 8-bit Bayer input (input_format='rggb') is not "
                         "supported")
    images = list(images)
    image_list._check(model, images, u8, what, floats=(torch.float32,))
    sizes = image_list.network_sizes([tuple(x.shape) for x in images], model.input_format, u8)
    _check_tiles(sizes, tile, tile_overlap, what)
    if not images:
        return []
    kind = capi.IMAGE_U8 if u8 else capi.IMAGE_RGGB if rggb else capi.IMAGE_F32
    src = [x.contiguous() for x in images]
    s = model.upscale
    tiles, chunks = tile_plan(model, sizes, tile, tile_overlap)
    first, last = {}, {}
    for j, (i, *_) in enumerate(tiles):
        first.setdefault(i, j)
        last[i] = j
    E, outs = [None] * len(images), [None] * len(images)
    for ch in chunks:
        batch = K.tile_gather([(src[tiles[j][0]],) + tiles[j][1:] for j in ch.index], kind, model.in_channels, ch.hp,
                              ch.wp)
        y = model.forward_rgb(batch)  # what forward_tile's model(patches) runs
        blends, done = [], []  # one run of consecutive tiles per image in this batch
        for slot, j in enumerate(ch.index):
            i, t = tiles[j][0], tiles[j][3]
            if E[i] is None:
                # zeros like forward_tile's E: the first tile is added to +0, not written (0 + -0 = +0)
                E[i] = torch.zeros(y.shape[1], sizes[i][0] * s, sizes[i][1] * s, device=y.device, dtype=torch.float32)
            if blends and blends[-1][0] is E[i]:
                blends[-1][4] += 1
            else:
                blends.append([E[i], t, tile_overlap, j - first[i], j - first[i] + 1, slot])
            if j == last[i]:
                done.append(i)
        K.tile_accumulate(y, [tuple(b) for b in blends], s)
        if not done:
            continue
        fin = [(E[i], tiles[last[i]][3], tile_overlap) for i in done]
        if u8:
            o8 = [torch.empty(E[i].shape[1], E[i].shape[2], E[i].shape[0], device=y.device, dtype=torch.uint8) for i in done]
            K.tile_finish(fin, s, o8)
        else:
            o8 = [E[i] for i in done]
            K.tile_finish(fin, s)
        for i, o in zip(done, o8):
            outs[i], E[i] = o, None
    return outs


def forward_tile_list(model, images, tile, tile_overlap):
    """forward_tile over a list of differently sized images, as a tiled test set comes: images[i] is (in_channels, H_i,
    W_i) float32 on the GPU (a model with input_format "rggb": packed Bayer planes (4, h_i, w_i) float32).  Returns the
    outputs in input order; element i equals forward_tile(model, images[i][None], tile, tile_overlap)[0] bit for bit for
    every precision, use_cuda_graph, self_ensemble and input_format.  The tiles of the whole list share forwards
    (tile_plan); one kernel cuts each batch of tiles out of their images, one adds the batch's outputs to the images'
    accumulators in forward_tile's order, one divides an image by its tile counts after its last tile."""
    return _forward_tile_list(model, images, tile, tile_overlap, u8=False)


def forward_tile_list_u8(model, images, tile, tile_overlap):
    """forward_tile_list of decoded 8-bit images (H_i, W_i, in_channels) uint8 on the GPU -> (H_i*s, W_i*s, out_channels)
    uint8; element i equals forward_tile_u8(model, images[i][None], tile, tile_overlap)[0] (no process group) bit for
    bit.  Packed 8-bit Bayer input (input_format="rggb") is not supported."""
    return _forward_tile_list(model, images, tile, tile_overlap, u8=True)
