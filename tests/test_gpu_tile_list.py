"""Tiled inference over a list of images on the GPU: the tile gather (csrc/image_list.cu) bit-exact against slicing and
check_image_size, the overlap blend bit-exact against forward_tile's slice add_ and E.div_(W), and
tiling.forward_tile_list / forward_tile_list_u8 equal, bit for bit, to the per-image forward_tile / forward_tile_u8 loop
they replace, on every precision, input format, CUDA-graph and self-ensemble setting."""
import pytest
import torch

from engine_oracle import check_image_size, to_tensor
from support import (MICRO, assert_equal_lists, build, count_calls, dm_model, micro, random_images, round8_ref,
                     same_bits)

pytestmark = pytest.mark.gpu


def windows(sizes, n, seed, k=1):
    """n random (image, y0, x0, t) windows of the frames (k*h, k*w), t from 1 up to 16 (the batch side), so that small
    windows take the zero fallback of check_image_size and larger ones reflect."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for j in range(n):
        i = j % len(sizes)
        H, W = k * sizes[i][0], k * sizes[i][1]
        t = int(torch.randint(1, min(16, H, W) + 1, (1,), generator=g))
        out.append((i, int(torch.randint(0, H - t + 1, (1,), generator=g)), int(torch.randint(0, W - t + 1, (1,), generator=g)), t))
    return out


SRC = [(40, 30), (17, 23), (16, 16), (9, 50), (64, 20)]


@pytest.mark.parametrize("kind", ["f32", "u8", "rggb"])
def test_tile_gather_bit_exact(pkg, device, kind):
    """130 windows (two launches' worth of descriptors) into a 16 x 16 batch, then every window cut at its own size."""
    from grl_image_restoration_b200 import capi, functional as K

    g = torch.Generator().manual_seed(7)
    C = 3 if kind == "rggb" else 4
    if kind == "u8":
        imgs = [torch.randint(0, 256, (h, w, C), dtype=torch.uint8, generator=g).to(device) for h, w in SRC]
        frames = [to_tensor(x) for x in imgs]
        code = capi.IMAGE_U8
    elif kind == "rggb":
        imgs = [torch.rand(4, h, w, generator=g).to(device) for h, w in SRC]
        frames = [K.demosaic(x[None])[0].cpu() for x in imgs]  # forward_tile cuts the demosaiced frame
        code = capi.IMAGE_RGGB
    else:
        imgs = [(torch.randn(C, h, w, generator=g) * 2).to(device) for h, w in SRC]
        imgs[0][0, 0, :4] = torch.tensor([-0.0, float("nan"), float("inf"), float("-inf")])
        frames = [x.cpu() for x in imgs]
        code = capi.IMAGE_F32
    wins = windows(SRC, 130, 3, 2 if kind == "rggb" else 1)
    assert any(t <= 8 for *_, t in wins) and any(t > 8 for *_, t in wins)  # both padding rules
    out = K.tile_gather([(imgs[i], y0, x0, t) for i, y0, x0, t in wins], code, C, 16, 16).cpu()
    assert out.shape == (130, C, 16, 16)
    for j, (i, y0, x0, t) in enumerate(wins):
        want = check_image_size(frames[i][None, :, y0:y0 + t, x0:x0 + t], 16, 16)[0]
        assert torch.equal(out[j].view(torch.int32), want.contiguous().view(torch.int32)), (j, i, y0, x0, t)
    for t in (1, 5, 16):  # Hp = Wp = t: a plain cut
        cut = [w for w in wins if w[3] == t][:3] or [(2, 0, 0, t)]
        got = K.tile_gather([(imgs[i], y0, x0, tt) for i, y0, x0, tt in cut], code, C, t, t).cpu()
        for j, (i, y0, x0, _) in enumerate(cut):
            assert torch.equal(got[j].view(torch.int32), frames[i][:, y0:y0 + t, x0:x0 + t].contiguous().view(torch.int32))


@pytest.mark.parametrize("scale", [1, 2])
def test_blend_bit_exact(pkg, device, scale):
    """Random tile outputs with -0, NaN and inf, a batch split so that one image's tiles span two accumulate calls, against
    tiling._accumulate and E.div_(W) on the same outputs; fp32 in place and uint8."""
    from grl_image_restoration_b200 import functional as K, tiling

    C, overlap = 3, 5
    sizes = [(40, 37), (12, 30), (16, 16), (57, 21)]
    tile = 16
    per = []  # (image, origins, t)
    for h, w in sizes:
        t = min(tile, h, w)
        per.append((tiling._origins(1, h, w, t, overlap), t))
    n = sum(len(o) for o, _ in per)
    g = torch.Generator().manual_seed(scale)
    y = torch.randn(n, C, 16 * scale + 3, 16 * scale + 1, generator=g)
    flat = y.view(-1)
    pick = torch.randint(0, flat.numel(), (4, 400), generator=g)
    flat[pick[0]], flat[pick[1]], flat[pick[2]], flat[pick[3]] = -0.0, float("nan"), float("inf"), float("-inf")
    y[0, :, :4, :4] = -0.0  # a corner only image 0's first tile covers: +0 + -0 = +0, where writing the tile gives -0
    y = y.to(device)
    refs, Es, slot = [], [], 0
    spans = []
    for (origins, t), (h, w) in zip(per, sizes):
        E = torch.zeros(1, C, h * scale, w * scale, device=device)
        W = torch.zeros_like(E)
        outs = [y[slot + k, :, :t * scale, :t * scale] for k in range(len(origins))]
        tiling._accumulate(E, W, origins, outs, t, scale)
        refs.append(E.div_(W)[0])
        Es.append(torch.zeros(C, h * scale, w * scale, device=device))
        spans.append((slot, len(origins), t))
        slot += len(origins)
    # two batches: the first holds every tile of images 0 to 2 and the first 3 of image 3's 10, the second the rest
    cut = spans[3][0] + 3
    for lo, hi in ((0, cut), (cut, n)):
        blends = []
        for E, (s0, cnt, t) in zip(Es, spans):
            k0, k1 = max(lo, s0) - s0, min(hi, s0 + cnt) - s0
            if k0 < k1:
                blends.append((E, t, overlap, k0, k1, s0 + k0 - lo))
        K.tile_accumulate(y[lo:hi].contiguous(), blends, scale)
    acc = [E.clone() for E in Es]
    outs8 = [torch.empty(E.shape[1], E.shape[2], C, dtype=torch.uint8, device=device) for E in acc]
    K.tile_finish([(E, s[2], overlap) for E, s in zip(acc, spans)], scale, outs8)
    K.tile_finish([(E, s[2], overlap) for E, s in zip(Es, spans)], scale)
    for i, (E, o8, ref) in enumerate(zip(Es, outs8, refs)):
        same_bits(E.cpu(), ref.cpu())
        assert torch.equal(o8.cpu(), round8_ref(ref.cpu())), i


# ------------------------------------------------------------------------------------------ end to end
# tile 24, overlap 6: several tile rows and columns, images smaller than the tile on one or both axes (t = 17, 12, 9),
# repeats of one size, both orientations
SIZES = [(40, 52), (17, 30), (24, 24), (52, 40), (12, 12), (33, 45), (40, 52), (9, 30)]
TILE, OVERLAP = 24, 6


def loop(tiling, m, xs, tile=TILE, overlap=OVERLAP):
    return [tiling.forward_tile(m, x[None], tile, overlap)[0] for x in xs]


@pytest.mark.parametrize("name", list(MICRO))
@pytest.mark.parametrize("precision,ensemble,graph", [("fp32", False, False), ("fp16", False, False),
                                                      ("fp16", False, True), ("fp16", True, False)])
def test_forward_tile_list_equals_loop(pkg, oracle, device, name, precision, ensemble, graph):
    from grl_image_restoration_b200 import image_list, tiling

    m = micro(pkg, oracle, name, device, precision, self_ensemble=ensemble)
    m.use_cuda_graph = graph
    xs = random_images(lambda h, w: (m.in_channels, h, w), SIZES, list(MICRO).index(name), device)
    kept = [x.clone() for x in xs]
    want = loop(tiling, m, xs)
    calls = count_calls(m, "forward_rgb")
    got = tiling.forward_tile_list(m, xs, TILE, OVERLAP)
    assert_equal_lists(got, want)
    assert all(torch.equal(a, b) for a, b in zip(xs, kept)), "forward_tile_list changed its inputs"
    tiles, chunks = tiling.tile_plan(m, image_list.network_sizes([tuple(x.shape) for x in xs]), TILE, OVERLAP)
    assert calls == [(len(c.index), m.in_channels, c.hp, c.wp) for c in chunks] and len(chunks) < len(xs)
    if graph:
        assert any(k[0][0] > 1 for k in m._graphs), "the batched forward must have replayed a captured graph"
        assert_equal_lists(tiling.forward_tile_list(m, xs, TILE, OVERLAP), want)


@pytest.mark.parametrize("precision,ensemble", [("fp32", False), ("fp16", False), ("fp16", True)])
def test_forward_tile_list_u8_equals_loop(pkg, oracle, device, precision, ensemble):
    from grl_image_restoration_b200 import tiling

    for name in ("micro_cab_x2", "micro_gray", "micro_dual"):
        m = micro(pkg, oracle, name, device, precision, self_ensemble=ensemble)
        g = torch.Generator().manual_seed(8)
        xs = [torch.randint(0, 256, (h, w, m.in_channels), dtype=torch.uint8, generator=g).to(device) for h, w in SIZES]
        kept = [x.clone() for x in xs]
        want = [tiling.forward_tile_u8(m, x[None], TILE, OVERLAP)[0] for x in xs]
        assert_equal_lists(tiling.forward_tile_list_u8(m, xs, TILE, OVERLAP), want)
        assert all(torch.equal(a, b) for a, b in zip(xs, kept))


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_small_budget_splits_images_across_forwards(pkg, oracle, device, precision):
    from grl_image_restoration_b200 import image_list, tiling

    m = micro(pkg, oracle, "micro_cab_x2", device, precision)
    xs = random_images(lambda h, w: (3, h, w), SIZES, 11, device)
    want = loop(tiling, m, xs)
    m.max_batch_tokens = 5 * 32 * 32  # 5 tiles of 24 (padded to 32) per forward: images of 3 x 3 tiles span several
    calls = count_calls(m, "forward_rgb")
    assert_equal_lists(tiling.forward_tile_list(m, xs, TILE, OVERLAP), want)
    tiles, chunks = tiling.tile_plan(m, image_list.network_sizes([tuple(x.shape) for x in xs]), TILE, OVERLAP)
    assert all(n * h * w <= m.max_batch_tokens for n, _, h, w in calls) and (5, 3, 32, 32) in calls
    assert len(calls) == len(chunks)
    assert any(len({k for k, c in enumerate(chunks) if any(tiles[j][0] == i for j in c.index)}) > 1 for i in range(len(xs)))


@pytest.mark.parametrize("precision,ensemble,graph", [("fp32", False, False), ("fp16", False, False),
                                                      ("fp16", False, True), ("fp16", True, False)])
def test_forward_tile_list_rggb(pkg, oracle, device, precision, ensemble, graph):
    from grl_image_restoration_b200 import tiling

    m = dm_model(pkg, oracle, device, precision, self_ensemble=ensemble)
    m.use_cuda_graph = graph
    packed = [(20, 26), (9, 13), (12, 12), (26, 20), (5, 16)]  # demosaiced: 40 x 52, 18 x 26, 24 x 24, 52 x 40, 10 x 32
    xs = random_images(lambda h, w: (4, h, w), packed, 4, device)
    want = loop(tiling, m, xs)
    got = tiling.forward_tile_list(m, xs, TILE, OVERLAP)
    assert_equal_lists(got, want)
    assert got[0].shape == (3, 40, 52)


def test_released_jpeg_small_at_288_36(pkg, oracle, device):
    """jpeg_grl_small_c3q10 as its test command tiles it (288 / 36), fp16, on BSDS500- and LIVE1-like sizes, one smaller
    than the tile."""
    from grl_image_restoration_b200 import tiling

    *_, tile, overlap = pkg.configs.RELEASED["jpeg_grl_small_c3q10.ckpt"]
    assert (tile, overlap) == (288, 36)
    cfg = pkg.configs.released_config("jpeg_grl_small_c3q10.ckpt", tile)
    m = build(pkg, oracle, cfg, device, "fp16", style="init")
    xs = random_images(lambda h, w: (3, h, w), [(481, 321), (321, 481), (512, 512), (500, 375), (256, 300), (481, 321)], 31,
                device)
    want = loop(tiling, m, xs, tile, overlap)
    calls = count_calls(m, "forward_rgb")
    assert_equal_lists(tiling.forward_tile_list(m, xs, tile, overlap), want)
    assert len(calls) < len(xs)


def test_rejects_bad_input_before_launching(pkg, oracle, device):
    from grl_image_restoration_b200 import capi, tiling

    m = micro(pkg, oracle, "micro_cab_x2", device, "fp16")
    good = torch.rand(3, 30, 30, device=device)
    bad = {
        "wrong rank": (ValueError, "shape", [good, torch.rand(1, 3, 20, 20, device=device)], TILE, OVERLAP),
        "wrong channel count": (ValueError, "shape", [good, torch.rand(4, 20, 20, device=device)], TILE, OVERLAP),
        "half input": (ValueError, "dtype.*float32", [good, good.half()], TILE, OVERLAP),
        "bfloat16 input": (ValueError, "dtype", [good.bfloat16()], TILE, OVERLAP),
        "cpu tensor": (RuntimeError, "CUDA device", [good, torch.rand(3, 20, 20)], TILE, OVERLAP),
        "tile 0": (ValueError, "tile = 0", [good], 0, 0),
        "overlap = tile": (ValueError, "tile_overlap", [good], 16, 16),
        "image not wider than the overlap": (ValueError, "element 1", [good, torch.rand(3, 30, 6, device=device)], TILE,
                                             OVERLAP),
    }
    for what, (exc, msg, xs, tile, overlap) in bad.items():
        before = capi.lib().grl_launch_count()
        with pytest.raises(exc, match=msg):
            tiling.forward_tile_list(m, xs, tile, overlap)
        assert capi.lib().grl_launch_count() == before, what
    with pytest.raises(ValueError, match="dtype"):
        tiling.forward_tile_list_u8(m, [good], TILE, OVERLAP)
    with pytest.raises(ValueError, match="input_format='rggb'"):
        tiling.forward_tile_list_u8(dm_model(pkg, oracle, device, "fp16"), [], TILE, OVERLAP)
    assert tiling.forward_tile_list(m, [], TILE, OVERLAP) == [] and tiling.forward_tile_list_u8(m, [], TILE, OVERLAP) == []
