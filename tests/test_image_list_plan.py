"""Lists of differently sized images on the CPU: the batch planner of GRL.forward_list (image_list.plan), the network
sizes it plans with, the list checks that need no device, and the argument checks of grl_list_gather / grl_list_crop,
which refuse a bad call on the host before anything launches."""
import ctypes

import pytest
import torch


def L():
    from grl_image_restoration_b200 import image_list

    return image_list


def test_groups_by_padded_size_in_input_order(pkg):
    sizes = [(30, 40), (64, 64), (17, 33), (33, 64), (32, 48), (1, 1), (64, 49)]
    chunks = L().plan(sizes, 32, 10 ** 9)
    # groups in order of their first image, images in input order within a group
    assert [(c.hp, c.wp, c.index) for c in chunks] == [(32, 64, [0, 2, 4]), (64, 64, [1, 3, 6]), (32, 32, [5])]


def test_splits_at_the_budget_exactly(pkg):
    sizes = [(64, 64)] * 7
    assert [c.index for c in L().plan(sizes, 64, 3 * 64 * 64)] == [[0, 1, 2], [3, 4, 5], [6]]
    assert [c.index for c in L().plan(sizes, 64, 3 * 64 * 64 - 1)] == [[0, 1], [2, 3], [4, 5], [6]]
    assert [c.index for c in L().plan(sizes, 64, 7 * 64 * 64)] == [list(range(7))]
    # groups are split independently; a group's chunks stay consecutive and in input order
    mixed = [(64, 64), (128, 64), (64, 64), (128, 64), (64, 64)]
    assert [(c.hp, c.index) for c in L().plan(mixed, 64, 2 * 64 * 64)] == [(64, [0, 2]), (64, [4]), (128, [1]), (128, [3])]


def test_oversize_image_runs_alone_and_empty_list_plans_nothing(pkg):
    chunks = L().plan([(300, 300), (10, 10), (290, 290)], 16, 100 * 100)
    assert [(c.hp, c.wp, c.index) for c in chunks] == [(304, 304, [0]), (304, 304, [2]), (16, 16, [1])]
    assert L().plan([], 16, 100) == []


def test_b100_orientations_share_one_bucket(pkg):
    """B100 at x4: the LR images are 120 x 80 or 80 x 120, and at GRL-Base's pad_size 64 both pad to 128 x 128."""
    cfg = pkg.configs.grl_config("base", "sr", 4, 64)
    m = pkg.GRL(**cfg)
    assert m.pad_size == 64 and m.max_batch_tokens == 16 * 256 * 256
    sizes = [(120, 80), (80, 120)] * 50
    chunks = L().plan(sizes, m.pad_size, m.max_batch_tokens)
    assert [(c.hp, c.wp, len(c.index)) for c in chunks] == [(128, 128, 64), (128, 128, 36)]
    assert [i for c in chunks for i in c.index] == list(range(100))


def test_network_sizes(pkg):
    assert L().network_sizes([(3, 17, 33), (1, 5, 6)]) == [(17, 33), (5, 6)]
    assert L().network_sizes([(17, 33, 3)], u8=True) == [(17, 33)]
    # packed Bayer planes (4, h, w) are planned at the demosaiced (2h, 2w)
    sizes = L().network_sizes([(4, 20, 28), (4, 9, 13), (4, 16, 16)], "rggb")
    assert sizes == [(40, 56), (18, 26), (32, 32)]
    assert [(c.hp, c.wp, c.index) for c in L().plan(sizes, 32, 10 ** 9)] == [(64, 64, [0]), (32, 32, [1, 2])]


def test_list_checks_without_a_device(pkg):
    m = pkg.GRL(**pkg.configs.micro_config())
    assert m.forward_list([]) == [] and m.forward_list_u8([]) == []
    with pytest.raises(ValueError, match="not a tensor"):
        m.forward_list([[1.0]])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.forward_list([torch.rand(3, 8, 8)])
    bayer = pkg.GRL(input_format="rggb", **pkg.configs.micro_config(upsampler="", upscale=1))
    with pytest.raises(ValueError, match="input_format='rggb'"):
        bayer.forward_list_u8([])


# ------------------------------------------------------------------------------------------ C ABI argument checks
def call(fn_name, refs, n, C, H, W):
    from grl_image_restoration_b200 import capi

    arr = (capi.GrlImageRef * max(1, len(refs)))(*[capi.GrlImageRef(d, h, w, k) for d, h, w, k in refs])
    lib = capi.lib()
    fake = ctypes.c_void_p(0x1000)  # never dereferenced: every refusal happens on the host
    if fn_name == "gather":
        rc = lib.grl_list_gather(arr, n, C, H, W, fake, None)
    else:
        rc = lib.grl_list_crop(fake, n, C, H, W, arr, None)
    return rc, lib.grl_last_error().decode()


P = 0x2000  # a non-NULL data pointer
BAD = [
    ("gather", [(None, 4, 4, 0)], 3, 8, 8, "null data"),
    ("gather", [(P, 0, 4, 0)], 3, 8, 8, "bad size"),
    ("gather", [(P, 4, 0, 1)], 3, 8, 8, "bad size"),
    ("gather", [(P, 1, 4, 2)], 3, 8, 8, "h, w >= 2"),
    ("gather", [(P, 9, 4, 0)], 3, 8, 8, "bigger than"),
    ("gather", [(P, 4, 5, 2)], 3, 8, 8, "bigger than"),  # RGGB 4 x 5 demosaics to 8 x 10
    ("gather", [(P, 4, 4, 0)], 0, 8, 8, "outside 1..8"),
    ("gather", [(P, 4, 4, 0)], 9, 8, 8, "outside 1..8"),
    ("gather", [(P, 4, 4, 3)], 3, 8, 8, "unknown kind"),
    ("gather", [(P, 4, 4, 0), (P, 4, 4, 1)], 3, 8, 8, "one kind per call"),
    ("gather", [(P, 2, 2, 2)], 4, 8, 8, "C = 3"),
    ("gather", [(P, 4, 4, 0)], 3, 0, 8, "bad batch size"),
    ("crop", [(P, 4, 4, 2)], 3, 8, 8, "unknown kind"),
    ("crop", [(P, 9, 8, 1)], 3, 8, 8, "bigger than"),
    ("crop", [(None, 4, 4, 1)], 3, 8, 8, "null data"),
    ("crop", [(P, 4, 4, 0)], 9, 8, 8, "outside 1..8"),
]


@pytest.mark.parametrize("fn,refs,C,H,W,msg", BAD)
def test_abi_refuses_bad_lists(pkg, fn, refs, C, H, W, msg):
    rc, err = call(fn, refs, len(refs), C, H, W)
    assert rc == -1 and msg in err, err


def test_abi_null_list(pkg):
    rc, err = call("gather", [], 0, 3, 8, 8)
    assert rc == 0  # an empty list launches nothing
    from grl_image_restoration_b200 import capi

    assert capi.lib().grl_list_gather(None, 2, 3, 8, 8, ctypes.c_void_p(P), None) == -1
    assert "null image list" in capi.lib().grl_last_error().decode()
