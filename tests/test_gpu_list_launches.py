"""Launches of every list entry point: a list of N + 1 images takes one more launch of each kernel than a list of N, where N
is the number of records one launch carries in its kernel parameters (csrc/grl_param_list.cuh), and a call with nothing to
do launches nothing.  Counted with grl_launch_count, on tiny images."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _calls(device):
    """name -> (records per launch, kernels per launch, call(n) running the entry point on a list of n images)"""
    from grl_image_restoration_b200 import capi, functional as F

    def f32(n, *shape):
        return [torch.zeros(*shape, device=device) for _ in range(n)]

    def u8(n, *shape):
        return [torch.zeros(*shape, device=device, dtype=torch.uint8) for _ in range(n)]

    def blends(n):
        return [(E, 4, 0, 0, 1, i) for i, E in enumerate(f32(n, 3, 4, 4))]

    return {
        "list_gather": (128, 1, lambda n: F.list_gather(f32(n, 3, 4, 4), capi.IMAGE_F32, 3, 4, 4)),
        "list_gather_u8": (128, 1, lambda n: F.list_gather(u8(n, 4, 4, 3), capi.IMAGE_U8, 3, 4, 4)),
        "list_crop": (128, 1, lambda n: F.list_crop(torch.zeros(n, 3, 4, 4, device=device), [(4, 4)] * n)),
        "tile_gather": (96, 1, lambda n: F.tile_gather([(x, 0, 0, 4) for x in f32(n, 3, 4, 4)], capi.IMAGE_F32, 3, 4, 4)),
        "tile_accumulate": (80, 1, lambda n: F.tile_accumulate(torch.zeros(n, 3, 4, 4, device=device), blends(n), 1)),
        "tile_finish": (80, 1, lambda n: F.tile_finish([b[:3] for b in blends(n)], 1)),
        "mosaic_list": (128, 1, lambda n: F.mosaic_list(u8(n, 4, 4, 3))),
        "mosaic": (128, 1, lambda n: F.mosaic(torch.zeros(n, 4, 4, 3, device=device, dtype=torch.uint8))),
        "luma_list": (128, 1, lambda n: F.luma_list(u8(n, 4, 4, 3))),
        "awgn_list": (64, 1, lambda n: F.awgn_list(u8(n, 4, 4, 3), 15, [[i] + [0] * 7 for i in range(n)])),
        "jpeg_gray": (80, 1, lambda n: F.jpeg_roundtrip_list(u8(n, 8, 8, 1), 10)),
        "jpeg_colour": (80, 2, lambda n: F.jpeg_roundtrip_list(u8(n, 8, 8, 3), 10)),
        "jpeg_batch": (80, 2, lambda n: F.jpeg_roundtrip(torch.zeros(n, 8, 8, 3, device=device, dtype=torch.uint8), 10)),
        "imresize_list": (64, 1, lambda n: F.imresize_list(u8(n, 8, 8, 3), 1 / 2)),
        "imresize": (64, 1, lambda n: F.imresize(torch.zeros(n, 3, 8, 8, device=device), 1 / 2)),
    }


def _launches(fn):
    from grl_image_restoration_b200 import capi

    before = capi.lib().grl_launch_count()
    fn()
    return capi.lib().grl_launch_count() - before


NAMES = ["list_gather", "list_gather_u8", "list_crop", "tile_gather", "tile_accumulate", "tile_finish", "mosaic_list",
         "mosaic", "luma_list", "awgn_list", "jpeg_gray", "jpeg_colour", "jpeg_batch", "imresize_list", "imresize"]


@pytest.mark.parametrize("name", NAMES)
def test_records_per_launch(pkg, device, name):
    per_launch, kernels, call = _calls(device)[name]
    assert _launches(lambda: call(1)) == kernels
    assert _launches(lambda: call(per_launch)) == kernels
    assert _launches(lambda: call(per_launch + 1)) == 2 * kernels
    assert _launches(lambda: call(0)) == 0  # an empty list launches nothing
    torch.cuda.synchronize()


def test_launches_without_work_are_skipped(pkg, device):
    from grl_image_restoration_b200 import functional as F

    # a mosaic of images one row high has empty destinations: a launch of only such images is skipped, chunk by chunk
    row = torch.zeros(1, 6, 3, device=device, dtype=torch.uint8)
    full = torch.zeros(4, 6, 3, device=device, dtype=torch.uint8)
    assert _launches(lambda: F.mosaic_list([row] * 3)) == 0
    assert _launches(lambda: F.mosaic_list([row] * 128 + [full])) == 1
    assert _launches(lambda: F.mosaic_list([full] + [row] * 128)) == 1
    assert _launches(lambda: F.mosaic(torch.zeros(0, 4, 4, 3, device=device, dtype=torch.uint8))) == 0
    assert _launches(lambda: F.luma(torch.zeros(0, 4, 4, 3, device=device, dtype=torch.uint8))) == 0
    assert _launches(lambda: F.awgn(torch.zeros(0, 4, 4, 3, device=device, dtype=torch.uint8), 15, [])) == 0
    assert _launches(lambda: F.imresize(torch.zeros(0, 3, 8, 8, device=device), 1 / 2)) == 0
    assert _launches(lambda: F.tile_gather([], 0, 3, 4, 4)) == 0
    torch.cuda.synchronize()
