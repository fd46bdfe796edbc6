"""Closed-form index arithmetic (csrc/grl_geometry.h, expanded by the C ABI's *_host functions) must be BIT-EXACT
against the reference's tensors (golden digests) and the oracle.  CPU only."""
import pytest
import torch

from support import sha


NAMES = ["sr_small_128", "dn_small_128", "deblur_96x192", "jpeg_144", "dm_64", "yaml_default_64", "groups_g1_32",
         "micro_16x32", "micro_32_df1", "sr_base_256", "dn_base_128x256"]


@pytest.mark.parametrize("name", NAMES)
def test_closed_forms_match_reference_digests(pkg, geometry_golden, name):
    """GRL.set_table_index_mask(materialize=True) == the reference's 13 buffers, by sha256."""
    g = geometry_golden["geometries"][name]
    m = object.__new__(pkg.GRL)  # geometry only: no network needed
    m.stripe_size, m.stripe_groups = g["stripe"], g["groups"]
    m.anchor_window_down_factor = g["df"]
    m.window_size = pkg.geometry.to_2tuple(g["window"])
    m.shift_size = [w // 2 for w in m.window_size]
    out = pkg.GRL.set_table_index_mask(m, tuple(g["x_size"]), materialize=True)
    assert set(out) == set(g["sha256"])
    for k, digest in g["sha256"].items():
        assert list(out[k].shape) == g["shape"][k], k
        assert sha(out[k]) == digest, f"{name}:{k} differs from the reference"


@pytest.mark.parametrize("ws,df", [((32, 32), 1), ((64, 64), 2), ((64, 128), 4), ((4, 86), 2), ((6, 12), 3), ((7, 5), 1)])
def test_index_and_table_vs_oracle(pkg, oracle, ws, df):
    G = pkg.geometry
    assert torch.equal(G.coords_table(ws, df), oracle.coords_table(list(ws), df))
    for w2a in (True, False):
        assert torch.equal(G.position_index(ws, df, w2a), oracle.position_index(list(ws), df, w2a))


@pytest.mark.parametrize("res,ws,sh,df", [
    ((64, 64), (32, 32), (16, 16), 1), ((64, 128), (64, 64), (32, 32), 4), ((32, 32), (32, 8), (0, 4), 2),
    ((32, 32), (8, 32), (4, 0), 2), ((24, 36), (12, 12), (6, 6), 1), ((48, 96), (48, 96), (24, 48), 4),
    ((16, 16), (8, 8), (0, 0), 2), ((30, 20), (6, 10), (3, 5), 1),
])
def test_masks_vs_oracle_including_degenerate_shifts(pkg, oracle, res, ws, sh, df):
    for w2a in (True, False):
        a = pkg.geometry.shift_mask(res, ws, sh, df, w2a)
        b = oracle.shift_mask(list(res), list(ws), list(sh), df, w2a)
        assert torch.equal(a, b)


def test_stripe_info(pkg, oracle):
    for args in (([64, 64], [None, None], True, (256, 256)), ([8, None], [None, 4], True, (64, 96)),
                 ([None, 8], [1, None], True, (32, 32)), ([48, 96], [None, None], False, (96, 192))):
        assert pkg.geometry.stripe_info(*args) == oracle.stripe_info(*args)


def test_bad_geometry_is_an_error(pkg):
    with pytest.raises(RuntimeError):
        pkg.geometry.shift_mask((30, 30), (8, 8), (4, 4))


# ---------------------------------------------------------------------------------------------------------------
# property tests: random geometries (beyond the released configurations) against the oracle's tensor constructions
# ---------------------------------------------------------------------------------------------------------------
from hypothesis import given, settings  # noqa: E402
from hypothesis import strategies as st  # noqa: E402


@st.composite
def _geometry(draw):
    df = draw(st.sampled_from([1, 2, 3, 4]))
    wh, ww = draw(st.integers(1, 6)) * df, draw(st.integers(1, 6)) * df  # window sides: multiples of df
    wh, ww = max(wh, 2 * df if df == 1 else df), max(ww, 2 * df if df == 1 else df)  # a side of 1 divides by zero in the reference too
    nh, nw = draw(st.integers(1, 3)), draw(st.integers(1, 3))            # windows per axis
    sh = draw(st.integers(0, wh // df)) * df if wh > df else 0          # shifts: multiples of df (anchors shift by s // df)
    sw = draw(st.integers(0, ww // df)) * df if ww > df else 0
    return (nh * wh, nw * ww), (wh, ww), (min(sh, wh - 1) // df * df, min(sw, ww - 1) // df * df), df


@settings(max_examples=60, deadline=None)
@given(_geometry())
def test_random_geometries_bit_exact(pkg, oracle, geo):
    res, ws, sh, df = geo
    G = pkg.geometry
    assert torch.equal(G.coords_table(ws, df), oracle.coords_table(list(ws), df))
    for w2a in (True, False):
        assert torch.equal(G.position_index(ws, df, w2a), oracle.position_index(list(ws), df, w2a))
        assert torch.equal(G.shift_mask(res, ws, sh, df, w2a), oracle.shift_mask(list(res), list(ws), list(sh), df, w2a))


@settings(max_examples=200, deadline=None)
@given(st.integers(8, 2000), st.integers(8, 600), st.integers(0, 64))
def test_tile_origins_match_engine_loop(pkg, size, tile, overlap):
    """engines/base.py:95-99: stride = tile - overlap; range(0, size - tile, stride) + [size - tile]."""
    from grl_image_restoration_b200 import tiling

    tile = min(tile, size)
    if overlap >= tile:
        return
    got = tiling.tile_origins(size, tile, overlap)
    assert got[-1] == size - tile and got[0] == 0 or size == tile
    assert all(0 <= o <= size - tile for o in got)
    covered = set()
    for o in got:
        covered.update(range(o, o + tile))
    assert covered == set(range(size)), "every pixel is restored by at least one tile"
    assert got[:-1] == list(range(0, size - tile, tile - overlap))
