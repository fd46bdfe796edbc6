"""Tiled inference with overlap averaging -- the engine's `forward_tile` (engines/base.py:90-116) with all tiles of the
image(s) batched into a few forwards instead of a Python double loop of single-tile forwards, and (forward_tile_sharded)
with the tiles of one frame spread over the ranks of a process group (SURVEY.md 8e: BASELINE cfg5, one 1280x720 frame
on 8 GPUs).

Semantics are the reference's exactly: tile = min(tile, h, w); origins range(0, h - tile, stride) + [h - tile] with
stride = tile - overlap (same for w); every tile is restored independently (so per-tile operators such as the CAB
global pool see the same data as in the reference), outputs are summed into E, a ones mask into W, result E / W.
"""
import torch

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
