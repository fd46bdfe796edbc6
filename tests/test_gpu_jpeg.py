"""The JPEG round trip on the GPU (csrc/jpeg.cu): every stored codec case byte for byte, through jpeg_roundtrip and
jpeg_roundtrip_list; batches and mixed-size lists equal to their images run alone; the JPEG test command's metric on the
device round trip equal to the metric on the codec's own output; and the refusals of the contract."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

with open(os.path.join(GOLD, "jpeg_cases.json")) as f:
    CASES = json.load(f)
_NPZ = {C: np.load(os.path.join(GOLD, f"jpeg_{'gray' if C == 1 else 'color'}.npz")) for C in (1, 3)}


def golden(name):
    """(quality, input, codec output) of a stored case; the images on the GPU."""
    c = CASES[name]
    z = _NPZ[c["channels"]]
    return c["quality"], torch.from_numpy(z[f"{name}/input"]).cuda(), torch.from_numpy(z[f"{name}/output"]).cuda()


@pytest.fixture(scope="module")
def K(pkg):
    assert torch.cuda.is_available()
    return pkg


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_case_batch_and_list(name, K):
    q, img, want = golden(name)
    got = K.jpeg_roundtrip(img[None], q)
    assert got.shape == (1,) + want.shape and got.dtype == torch.uint8
    assert torch.equal(got[0], want), (name, int((got[0] != want).sum()))
    (got_l,) = K.jpeg_roundtrip_list([img], q)
    assert torch.equal(got_l, want)


@pytest.mark.parametrize("C", [1, 3])
def test_golden_cases_as_one_list_per_quality(C, K):
    """All stored cases of one C and quality in one call, next to each other in the flat block and pixel indices."""
    by_q = {}
    for name, c in CASES.items():
        if c["channels"] == C:
            by_q.setdefault(c["quality"], []).append(name)
    for q, names in by_q.items():
        imgs, wants = zip(*[golden(n)[1:] for n in names])
        outs = K.jpeg_roundtrip_list(list(imgs), q)
        for n, o, w in zip(names, outs, wants):
            assert torch.equal(o, w), n


@pytest.mark.parametrize("C", [1, 3])
def test_batch_equals_images_alone(C, K):
    g = torch.Generator(device="cuda").manual_seed(7 + C)
    x = torch.randint(0, 256, (5, 37, 53, C), generator=g, device="cuda", dtype=torch.uint8)
    x[1] = x[1] // 64 * 64  # flat regions
    x[2, :, :20] = 255
    y = K.jpeg_roundtrip(x, 10)
    for b in range(5):
        assert torch.equal(y[b], K.jpeg_roundtrip(x[b:b + 1].clone(), 10)[0]), b
    assert torch.equal(y[3], K.jpeg_roundtrip_host(x[3].cpu(), 10).cuda())


@pytest.mark.parametrize("C", [1, 3])
def test_mixed_size_list_equals_images_alone(C, K):
    """A list that spans several launches (more images than one launch's descriptors) and sizes of every kind."""
    g = torch.Generator(device="cuda").manual_seed(11 + C)
    sizes = [(1, 1), (2, 3), (8, 8), (16, 16), (17, 33), (481, 321), (321, 481), (64, 200)] * 12
    imgs = [torch.randint(0, 256, (h, w, C), generator=g, device="cuda", dtype=torch.uint8) for h, w in sizes]
    outs = K.jpeg_roundtrip_list(imgs, 30)
    assert len(outs) == len(imgs)
    for i, (img, out) in enumerate(zip(imgs, outs)):
        assert out.shape == img.shape and torch.equal(out, K.jpeg_roundtrip(img[None], 30)[0]), (i, sizes[i])
    for i in (5, 6, 90):
        assert torch.equal(outs[i].cpu(), K.jpeg_roundtrip_host(imgs[i].cpu(), 30)), i


def test_input_untouched_and_outputs_new(K):
    q, img, _ = golden(sorted(n for n in CASES if n.startswith("c3_100x72_q10"))[0])
    before = img.clone()
    out = K.jpeg_roundtrip_list([img], q)[0]
    assert torch.equal(img, before) and out.data_ptr() != img.data_ptr()


def test_psnrb_of_device_roundtrip_equals_codec_output(K):
    """The JPEG test command's PSNR-B, of the degraded input against the clean image: the device round trip gives the
    codec's score exactly."""
    from grl_image_restoration_b200 import metrics

    names = [n for n, c in CASES.items() if c["H"] >= 16 and c["W"] >= 16]
    assert len(names) > 30
    for n in names:
        q, img, want = golden(n)
        lq = K.jpeg_roundtrip_list([img], q)[0]
        a = metrics.psnrb_fused(lq[None], img[None])
        b = metrics.psnrb_fused(want[None], img[None])
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), n


def test_refusals(K):
    img = torch.zeros(1, 16, 16, 3, dtype=torch.uint8, device="cuda")
    for q in (0, 101, 10.5, "10", None, True):
        with pytest.raises(ValueError):
            K.jpeg_roundtrip(img, q)
        with pytest.raises(ValueError):
            K.jpeg_roundtrip_list([img[0]], q)
    with pytest.raises(RuntimeError):
        K.jpeg_roundtrip(img.cpu(), 10)
    with pytest.raises(RuntimeError):
        K.jpeg_roundtrip_list([img[0], img[0].cpu()], 10)
    for bad in (img.float(), img[..., :2], torch.zeros(1, 16, 16, 4, dtype=torch.uint8, device="cuda"), img[0],
                torch.zeros(1, 0, 16, 3, dtype=torch.uint8, device="cuda")):
        with pytest.raises(ValueError):
            K.jpeg_roundtrip(bad, 10)
    with pytest.raises(ValueError):
        K.jpeg_roundtrip_list([img[0], img[0, ..., :1]], 10)  # mixed C
    with pytest.raises(ValueError):
        K.jpeg_roundtrip_list([img[0], img[0].float()], 10)
    with pytest.raises(ValueError):
        K.jpeg_roundtrip_list([img[0], np.zeros((16, 16, 3), np.uint8)], 10)
    assert K.jpeg_roundtrip_list([], 10) == []
