"""Tiled inference over a list of images on the CPU: the coverage closed form of csrc/grl_tiles.h against the enumeration
of tiling.tile_origins, the tile enumeration and batch plan of tiling.forward_tile_list, its list checks, and the argument
checks of grl_tile_gather / grl_tile_accumulate / grl_tile_finish, which refuse a bad call on the host before anything
launches."""
import ctypes

import numpy as np
import pytest
import torch


def T():
    from grl_image_restoration_b200 import tiling

    return tiling


def test_coverage_closed_form_exhaustive(pkg):
    """Every axis size H <= 200, tile t <= H, overlap < t and scale 1..4: the first and last covering tile of every output
    row against the enumeration.  tile_origins strictly increases and every tile has side t, so the tiles with origin
    <= r are a prefix [0, A) and those ending at or before r a prefix [0, B): the covering tiles are exactly [B, A), in
    origin order, and there are A - B of them."""
    from grl_image_restoration_b200 import capi

    lib = capi.lib()
    for H in range(1, 201):
        for t in range(1, H + 1):
            origins = [T().tile_origins(H, t, ov) for ov in range(t)]
            o = np.concatenate(origins)
            ov = np.repeat(np.arange(t), [len(x) for x in origins])
            same = ov[1:] == ov[:-1]
            assert (np.diff(o)[same] > 0).all() and (o[~np.r_[False, same]] == 0).all()
            # a[ov, r]: tiles with origin <= r; b[ov, r]: tiles with origin + t <= r
            a = np.bincount(ov * (H + 1) + o, minlength=t * (H + 1)).reshape(t, H + 1).cumsum(1)[:, :H]
            b = np.bincount(ov * (H + 1) + o + t, minlength=t * (H + 1)).reshape(t, H + 1).cumsum(1)[:, :H]
            assert (a - b >= 1).all()  # every row is covered
            want = np.stack([b, a - 1], 2)  # (overlaps, H, 2)
            for s in (1, 2, 3, 4):
                got = np.empty((t, H * s, 2), dtype=np.int32)
                base, step = got.ctypes.data, H * s * 8
                for k in range(t):
                    assert lib.grl_tile_cover_host(H, t, k, s, base + k * step) == 0
                assert np.array_equal(got, np.repeat(want, s, axis=1)), (H, t, s)


def test_coverage_refuses_bad_axes(pkg):
    from grl_image_restoration_b200 import capi, functional as K

    for size, tile, overlap, scale in ((10, 0, 0, 1), (10, 11, 0, 1), (10, 4, 4, 1), (10, 4, -1, 1), (10, 4, 1, 0)):
        with pytest.raises(RuntimeError, match="tile_cover"):
            K.tile_cover_host(size, tile, overlap, scale)
    assert capi.lib().grl_tile_cover_host(10, 4, 1, 1, None) == -1


class _Model:  # what tile_plan reads of a GRL
    def __init__(self, pad_size=16, max_batch_tokens=10 ** 9, self_ensemble=False):
        self.pad_size, self.max_batch_tokens, self.self_ensemble = pad_size, max_batch_tokens, self_ensemble


def test_tiles_in_forward_tile_order(pkg):
    sizes = [(40, 30), (12, 50), (20, 20)]
    tiles, chunks = T().tile_plan(_Model(), sizes, 16, 4)
    want = []
    for i, (h, w) in enumerate(sizes):
        t = min(16, h, w)
        for bi, y0, x0 in T()._origins(1, h, w, t, 4):  # forward_tile's own enumeration of one image
            want.append((i, y0, x0, t))
    assert tiles == want
    assert [i for i, *_ in tiles] == sorted(i for i, *_ in tiles)
    # image 1 is 12 high: its tiles are 12 x 12 (one row of 6), image 0 has 3 x 3 tiles of 16, image 2 2 x 2
    assert [t for *_, t in tiles].count(12) == 6 and len(tiles) == 9 + 6 + 4
    # 16 and 12 both pad to 16: one forward takes every tile, in order
    assert [(c.hp, c.wp, c.index) for c in chunks] == [(16, 16, list(range(len(tiles))))]


def test_chunk_budget_splits_an_image_in_order(pkg):
    sizes = [(40, 40), (64, 64), (40, 40)]
    tiles, chunks = T().tile_plan(_Model(pad_size=32, max_batch_tokens=5 * 32 * 32), sizes, 32, 8)
    assert len(tiles) == 4 + 9 + 4
    assert [len(c.index) for c in chunks] == [5, 5, 5, 2]
    flat = [j for c in chunks for j in c.index]
    assert flat == list(range(len(tiles)))  # one group: every tile, every image's in origin order
    # image 1's tiles (4 .. 12) span three chunks
    assert {k for k, c in enumerate(chunks) for j in c.index if tiles[j][0] == 1} == {0, 1, 2}
    for c in chunks:  # consecutive runs per image within a chunk
        imgs = [tiles[j][0] for j in c.index]
        assert imgs == sorted(imgs)


def test_mixed_tile_sizes_and_images_smaller_than_the_tile(pkg):
    sizes = [(100, 100), (20, 30), (100, 60), (9, 9), (30, 20)]
    tiles, chunks = T().tile_plan(_Model(pad_size=16), sizes, 48, 8)
    side = {i: t for i, _, _, t in tiles}
    assert side == {0: 48, 1: 20, 2: 48, 3: 9, 4: 20}
    # groups by padded size in order of their first tile: 48 (images 0, 2), 32 (1, 4), 16 (3)
    assert [(c.hp, [tiles[j][0] for j in c.index][0]) for c in chunks] == [(48, 0), (32, 1), (16, 3)]
    for c in chunks:
        js = c.index
        assert js == sorted(js) and all(-(-tiles[j][3] // 16) * 16 == c.hp == c.wp for j in js)
    # images smaller than the tile are one tile each, their whole frame
    assert [x for x in tiles if x[0] in (1, 3, 4)] == [(1, 0, 0, 20), (1, 0, 10, 20), (3, 0, 0, 9), (4, 0, 0, 20),
                                                        (4, 10, 0, 20)]


def test_self_ensemble_groups_by_exact_size(pkg):
    sizes = [(40, 40), (20, 30), (18, 18), (30, 20)]
    _, chunks = T().tile_plan(_Model(pad_size=16), sizes, 24, 4)
    assert [(c.hp, c.wp) for c in chunks] == [(32, 32)]  # 24, 20 and 18 all pad to 32
    tiles, chunks = T().tile_plan(_Model(pad_size=16, self_ensemble=True), sizes, 24, 4)
    assert [(c.hp, c.wp) for c in chunks] == [(24, 24), (20, 20), (18, 18)]
    for c in chunks:
        assert {tiles[j][3] for j in c.index} == {c.hp}
    assert sorted(j for c in chunks for j in c.index) == list(range(len(tiles)))


def test_list_checks_without_a_device(pkg):
    m = pkg.GRL(**pkg.configs.micro_config())
    assert T().forward_tile_list(m, [], 16, 4) == [] and T().forward_tile_list_u8(m, [], 16, 4) == []
    with pytest.raises(ValueError, match="not a tensor"):
        T().forward_tile_list(m, [[1.0]], 16, 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        T().forward_tile_list(m, [torch.rand(3, 8, 8)], 16, 4)
    with pytest.raises(ValueError, match="tile = 0"):
        T().forward_tile_list(m, [], 0, 0)
    with pytest.raises(ValueError, match="tile_overlap = -1"):
        T().forward_tile_list(m, [], 8, -1)
    bayer = pkg.GRL(input_format="rggb", **pkg.configs.micro_config(upsampler="", upscale=1))
    with pytest.raises(ValueError, match="input_format='rggb'"):
        T().forward_tile_list_u8(bayer, [], 16, 4)


def test_overlap_checks_on_network_sizes(pkg):
    from grl_image_restoration_b200 import image_list

    check = T()._check_tiles
    check([(40, 40), (5, 40)], 16, 4, "f")
    with pytest.raises(ValueError, match=r"element 1 \(4 x 40\).*min\(tile, H, W\) = 4.*tile_overlap = 4"):
        check([(40, 40), (4, 40)], 16, 4, "f")
    with pytest.raises(ValueError, match="tile_overlap = 16"):
        check([(40, 40)], 16, 16, "f")
    # packed Bayer planes (4, 3, 3) are a 6 x 6 frame: a 6-pixel tile with overlap 5 is fine, with 6 it is not
    sizes = image_list.network_sizes([(4, 3, 3)], "rggb")
    check(sizes, 16, 5, "f")
    with pytest.raises(ValueError, match="= 6"):
        check(sizes, 16, 6, "f")


# ------------------------------------------------------------------------------------------ C ABI argument checks
P = 0x2000  # a non-NULL data pointer, never dereferenced: every refusal happens on the host
FAKE = ctypes.c_void_p(0x1000)


def gather(tiles, C, Hp, Wp, n=None):
    from grl_image_restoration_b200 import capi

    arr = (capi.GrlTileRef * max(1, len(tiles)))(
        *[capi.GrlTileRef(capi.GrlImageRef(d, h, w, k), y0, x0, t) for (d, h, w, k), y0, x0, t in tiles])
    rc = capi.lib().grl_tile_gather(arr, len(tiles) if n is None else n, C, Hp, Wp, FAKE, None)
    return rc, capi.lib().grl_last_error().decode()


BAD_GATHER = [
    ([((P, 20, 20, 0), 0, 0, 16)], 0, 16, 16, "outside 1..8"),
    ([((P, 20, 20, 0), 0, 0, 16)], 9, 16, 16, "outside 1..8"),
    ([((P, 20, 20, 3), 0, 0, 16)], 3, 16, 16, "unknown kind"),
    ([((P, 20, 20, 0), 0, 0, 16), ((P, 20, 20, 1), 0, 0, 16)], 3, 16, 16, "one kind per call"),
    ([((None, 20, 20, 0), 0, 0, 16)], 3, 16, 16, "null data"),
    ([((P, 20, 20, 0), 0, 0, 17)], 3, 16, 32, "side 17 outside"),
    ([((P, 20, 20, 0), 0, 0, 0)], 3, 16, 16, "side 0 outside"),
    ([((P, 20, 20, 0), 5, 0, 16)], 3, 16, 16, "outside the 20 x 20 image"),
    ([((P, 20, 20, 0), 0, -1, 16)], 3, 16, 16, "outside"),
    ([((P, 20, 30, 1), 0, 15, 16)], 3, 16, 16, "outside the 20 x 30 image"),
    ([((P, 10, 10, 2), 0, 5, 16)], 3, 16, 16, "outside the 20 x 20 image"),  # RGGB 10 x 10 planes: a 20 x 20 frame
    ([((P, 10, 10, 2), 0, 0, 16)], 4, 16, 16, "C = 3"),
    ([((P, 1, 10, 2), 0, 0, 1)], 3, 16, 16, "h, w >= 2"),
    ([((P, 20, 20, 0), 0, 0, 16)], 3, 0, 16, "bad batch size"),
]


@pytest.mark.parametrize("tiles,C,Hp,Wp,msg", BAD_GATHER)
def test_abi_gather_refuses_bad_tiles(pkg, tiles, C, Hp, Wp, msg):
    rc, err = gather(tiles, C, Hp, Wp)
    assert rc == -1 and msg in err, err


def test_abi_gather_null_list_and_good_windows(pkg):
    from grl_image_restoration_b200 import capi

    assert gather([], 3, 16, 16)[0] == 0  # an empty list launches nothing
    assert capi.lib().grl_tile_gather(None, 2, 3, 16, 16, FAKE, None) == -1
    assert "null tile list" in capi.lib().grl_last_error().decode()
    assert capi.lib().grl_tile_gather(None, 0, 3, 16, 16, None, None) == 0


def blend(images, n=4, C=3, Hy=32, Wy=32, scale=1, finish=False):
    from grl_image_restoration_b200 import capi

    arr = (capi.GrlTileImage * max(1, len(images)))(*[capi.GrlTileImage(*im) for im in images])
    lib = capi.lib()
    if finish:
        rc = lib.grl_tile_finish(arr, len(images), C, scale, None)
    else:
        rc = lib.grl_tile_accumulate(FAKE, n, C, Hy, Wy, scale, arr, len(images), None)
    return rc, lib.grl_last_error().decode()


# (E, out_u8, H, W, t, overlap, k0, k1, slot); a 40 x 40 image at t 16 / overlap 4 has 3 x 3 tiles
GOOD = (P, None, 40, 40, 16, 4, 0, 9, 0)
BAD_BLEND = [
    (dict(images=[GOOD], n=8), "past the batch"),
    (dict(images=[(P, None, 40, 40, 16, 4, 2, 9, 0)], n=6), "past the batch"),
    (dict(images=[(P, None, 40, 40, 16, 4, 0, 10, 0)], n=16), "outside its 9 tiles"),
    (dict(images=[(P, None, 40, 40, 16, 4, 3, 3, 0)], n=16), "outside its 9 tiles"),
    (dict(images=[(P, None, 40, 40, 16, 4, 0, 2, -1)], n=16), "past the batch"),
    (dict(images=[(None, None, 40, 40, 16, 4, 0, 9, 0)], n=16), "null accumulator"),
    (dict(images=[(P, None, 40, 10, 16, 4, 0, 1, 0)], n=16), "tile 16, overlap 4"),
    (dict(images=[(P, None, 40, 40, 16, 16, 0, 1, 0)], n=16), "tile 16, overlap 16"),
    (dict(images=[(P, None, 0, 40, 1, 0, 0, 1, 0)], n=16), "bad size"),
    (dict(images=[GOOD], n=16, Hy=15), "bigger than the batch"),
    (dict(images=[GOOD], n=16, scale=3), "bigger than the batch"),
    (dict(images=[GOOD], n=16, C=9), "outside 1..8"),
    (dict(images=[GOOD], n=16, scale=0), "scale 0"),
    (dict(images=[GOOD, (P, P, 40, 40, 16, 4, 0, 9, 0)], C=3, finish=True), "one output kind per call"),
    (dict(images=[(P, None, 40, 40, 41, 4, 0, 9, 0)], finish=True), "tile 41"),
    (dict(images=[GOOD], C=0, finish=True), "outside 1..8"),
    (dict(images=[GOOD], scale=0, finish=True), "bad scale"),
]


@pytest.mark.parametrize("kw,msg", BAD_BLEND)
def test_abi_blend_refuses_bad_images(pkg, kw, msg):
    rc, err = blend(**kw)
    assert rc == -1 and msg in err, err


def test_abi_blend_null_list(pkg):
    from grl_image_restoration_b200 import capi

    lib = capi.lib()
    assert lib.grl_tile_accumulate(None, 0, 3, 8, 8, 1, None, 0, None) == 0
    assert lib.grl_tile_finish(None, 0, 3, 1, None) == 0
    assert lib.grl_tile_accumulate(FAKE, 4, 3, 8, 8, 1, None, 2, None) == -1
    assert "null image list" in lib.grl_last_error().decode()
    assert lib.grl_tile_finish(None, 1, 3, 1, None) == -1
    assert "null image list" in lib.grl_last_error().decode()
