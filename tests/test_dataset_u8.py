"""The host copies of the dataset-side inputs (csrc/grl_dataset_u8.h): the Bayer mosaic and the MATLAB luma against the
reference's fixtures, the luma against numpy's rgb2ycbcr_np expression over every RGB triple, the blind-SR reader against
to_tensor's k / 255, and the recipe table of evaluation.py against the reference's commands and yamls."""
import json
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(GOLD, "eval_cases.json")) as f:
    CASES = json.load(f)
_NPZ = np.load(os.path.join(GOLD, "eval_inputs.npz"))
MOSAIC = [k for k in CASES if k != "luma"]


@pytest.mark.parametrize("name", MOSAIC)
def test_mosaic_host_matches_reference(name, pkg):
    from grl_image_restoration_b200 import functional as F

    got = F.mosaic_host(torch.from_numpy(_NPZ[f"{name}/img"]))
    want = torch.from_numpy(_NPZ[f"{name}/mosaic"])
    assert got.shape == want.shape and torch.equal(got, want), name


def test_mosaic_host_plane_order(pkg):
    """R, G of the even rows, G of the odd rows, B, each k / 255; the odd last row and column dropped."""
    from grl_image_restoration_b200 import functional as F

    img = torch.randint(0, 256, (7, 9, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    got = F.mosaic_host(img)
    u = img.float() / 255
    want = torch.stack([u[0:6:2, 0:8:2, 0], u[0:6:2, 1:8:2, 1], u[1:6:2, 0:8:2, 1], u[1:6:2, 1:8:2, 2]])
    assert torch.equal(got, want)


def test_luma_host_matches_reference(pkg):
    from grl_image_restoration_b200 import functional as F

    got = F.luma_host(torch.from_numpy(_NPZ["luma/rgb"]))[:, 0]
    assert torch.equal(got, torch.from_numpy(_NPZ["luma/y"]))
    assert CASES["luma"]["ties"] == []


def _numpy_luma(img):
    """rgb2ycbcr_np(img, y_only=True) of an (H, W, 3) uint8 image, restated (utils/utils_image.py:143-190)."""
    x = img.astype(np.float32)
    x /= 255.0
    return (np.dot(x, [65.481, 128.553, 24.966]) + 16.0).round().astype(np.uint8)


def test_luma_host_every_rgb_triple(pkg):
    """All 2^24 triples, one 256 x 256 image per red value (numpy's dot runs per pixel on (H, W, 3) images, as the
    dataset calls it).  Any difference would be a rounding tie decided by the evaluation order; there is none."""
    from grl_image_restoration_b200 import functional as F

    g, b = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    cube = np.empty((256, 256, 256, 3), dtype=np.uint8)
    cube[..., 1], cube[..., 2] = g, b
    for r in range(256):
        cube[r, ..., 0] = r
    got = F.luma_host(torch.from_numpy(cube))[..., 0].numpy()
    bad = 0
    for r in range(256):
        bad += int((got[r] != _numpy_luma(cube[r])).sum())
    assert bad == 0, f"{bad} of 2^24 triples differ from numpy"


def test_uint2single_is_to_tensor(pkg):
    """The blind-SR dataset reads with uint2single, np.float32(img / 255.0) (two roundings, float64 then float32); for
    every byte that equals to_tensor's k / 255 in float32, so u8_to_f32 is its reader."""
    from grl_image_restoration_b200 import functional as F

    k = np.arange(256, dtype=np.uint8)
    ref = np.float32(k / 255.0)
    assert ref.dtype == np.float32
    assert np.array_equal(ref.view(np.uint32), _NPZ["uint2single"].view(np.uint32))
    host = F.u8_to_f32_host(torch.from_numpy(k).reshape(1, 1, 256, 1))[0, 0, 0]
    assert np.array_equal(host.numpy().view(np.uint32), ref.view(np.uint32))


# What the reference's test commands and yamls say, per task (cited lines in evaluation.py's docstring):
# (crop, input, level, collection, border = the SR scale?)
EXPECTED = {
    "sr": ("modcrop", "lq", None, "restorer", True),          # base_image.py:404-405; sr/grl/grl_p256.yaml:23
    "dn": ("mod8", "awgn", 15, None, False),                  # base_image.py:419-423; grl_test.md:23-29 SIGMA=15
    "jpeg": ("none", "jpeg", 10, None, False),                # restoration_jpeg.py:38-42; grl_test.md:89-91 QUALITY=10
    "dm": ("mod8", "mosaic", None, "restorer", False),        # restoration_dm.py:30-35; dm/grl.yaml:21
    "bsr": ("none", "self", None, "restorer_niqe", False),    # restoration_bsr.py:111-118; bsr/grl.yaml:26, :49
    "defocus": ("none", "lq", None, "restorer", False),       # db_defocus/grl_p480.yaml:24
    "defocus_dual": ("none", "lq_dual", None, "restorer", False),
    "deblur": ("none", "lq", None, "restorer", False),        # db_motion/grl_p480.yaml:25
}
GRAY = {"dn": ("restorer_gray", "restorer"), "jpeg": ("restorer_jpeg_gray", "restorer_jpeg")}  # METRIC=(c1 c3)
TILES = {  # grl_test.md:49 (dn base), :96 (jpeg), :62-78 and :128 (tile=0), db_defocus/grl_p480.yaml:9-10
    "dn_grl_base_c1s15.ckpt": (256, 32), "dn_grl_base_c3s15.ckpt": (256, 32), "jpeg_grl_small_c1q10.ckpt": (288, 36),
    "jpeg_grl_small_c3q10.ckpt": (288, 36), "db_defocus_single_pixel_grl_base.ckpt": (480, 48),
    "db_defocus_dual_pixel_grl_base.ckpt": (480, 48),
}


def test_every_released_checkpoint_has_its_recipe(pkg):
    from grl_image_restoration_b200 import configs, evaluation

    assert set(evaluation.RECIPES) == set(configs.RELEASED)
    for name, r in evaluation.RECIPES.items():
        _, task, scale, cin, _, _ = configs.RELEASED[name]
        crop, inp, level, coll, shave = EXPECTED[task]
        assert (r.task, r.crop, r.input, r.level) == (task, crop, inp, level), name
        assert r.collection == (GRAY[task][cin == 3] if task in GRAY else coll), name
        assert r.border == (scale if shave else 0), name
        assert r.channels == (cin if task in GRAY else 3), name
        assert (r.tile, r.tile_overlap) == TILES.get(name, (0, 0)), name
        assert set(evaluation.COLLECTIONS[r.collection]) <= {"val_psnr", "val_psnr_y", "val_ssim", "val_ssim_y",
                                                             "val_psnrb", "val_psnrb_y", "val_niqe"}


def test_collections_match_the_metric_yamls(pkg):
    from grl_image_restoration_b200 import evaluation

    assert evaluation.COLLECTIONS == {  # config/metric/<name>.yaml, val_* entries in order
        "restorer": ("val_psnr", "val_psnr_y", "val_ssim", "val_ssim_y"),
        "restorer_gray": ("val_psnr", "val_ssim"),
        "restorer_jpeg": ("val_psnr", "val_psnr_y", "val_ssim", "val_ssim_y", "val_psnrb", "val_psnrb_y"),
        "restorer_jpeg_gray": ("val_psnr", "val_ssim", "val_psnrb"),
        "restorer_niqe": ("val_niqe",),
    }
    assert evaluation.LUMA_SETS == ("live1", "bsds500", "urban100")  # base_image.py:233-237


def test_mean_is_average_metrics(pkg):
    """sum(list of 0-d tensors) / len, in the values' dtype (utils/metrics/psnr.py:37-41)."""
    from grl_image_restoration_b200 import evaluation

    v = torch.tensor([30.123456, 28.5, 31.25, 29.0078125], dtype=torch.float32)
    want = (((v[0] + v[1]) + v[2]) + v[3]) / 4
    got = evaluation.mean(list(v.unbind(0)))
    assert got.dtype == torch.float32 and torch.equal(got, want)


def test_refusals_without_a_device(pkg):
    from grl_image_restoration_b200 import evaluation

    with pytest.raises(ValueError, match="unknown checkpoint"):
        evaluation.evaluate(None, "nope.ckpt", [])
    with pytest.raises(ValueError, match="no images"):
        evaluation.evaluate(None, "dm_grl_small.ckpt", [])
    with pytest.raises(ValueError, match="CUDA"):
        evaluation.clean_images("dm_grl_small.ckpt", [torch.zeros(8, 8, 3, dtype=torch.uint8)])


def test_seed_keys_use_the_reference_set_names(pkg):
    """img_info[index][0] starts with the set's directory name (restoration_dn.py:72-88), whatever case the caller uses."""
    from grl_image_restoration_b200 import evaluation

    assert evaluation.seed_keys("cbsd68", ["0001.png"]) == ["CBSD68/0001.png"]
    assert evaluation.seed_keys("CBSD68", ["0001.png"]) == ["CBSD68/0001.png"]
    assert evaluation.seed_keys("urban100", ["img_004.png"]) == ["Urban100/img_004.png"]
    assert evaluation.seed_keys("Set12", ["01.png", "02.png"]) == ["Set12/01.png", "Set12/02.png"]
    with pytest.raises(ValueError, match="unknown denoising test set"):
        evaluation.seed_keys("cbsd-68", ["0001.png"])
