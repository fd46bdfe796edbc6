"""The seeded AWGN on the GPU (csrc/awgn.cu): the reference's goldens, and mixed lists against the dataset's recipe
computed here with numpy (to_tensor + torch.from_numpy(RandomState(key).normal(0, sigma / 255, (C, H, W))).float()),
every float32 compared with torch.equal; batches against lists; streams; the refusals; and a micro denoiser fed from
the device noise against the same model fed the recipe's inputs."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from engine_oracle import to_tensor
from support import micro

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

with open(os.path.join(GOLD, "awgn_cases.json")) as f:
    CASES = json.load(f)
_NPZ = np.load(os.path.join(GOLD, "awgn.npz"))


@pytest.fixture(scope="module")
def K(pkg):
    assert torch.cuda.is_available()
    return pkg


def recipe(img, sigma, seed):
    """The dataset's img_lq of one (H, W, C) uint8 image on the CPU: to_tensor, then the float32 RandomState noise."""
    from grl_image_restoration_b200 import functional as F

    gt = to_tensor(img).contiguous()
    key = F._awgn_keys([seed], 1, "recipe")[0]
    return gt + torch.from_numpy(np.random.RandomState(key).normal(0, sigma / 255, gt.shape)).float()


def rand_u8(h, w, C, g):
    return torch.randint(0, 256, (h, w, C), generator=g, dtype=torch.uint8).cuda()


def assert_equal(got, want, what):
    assert got.shape == want.shape and got.dtype == torch.float32, (what, got.shape, want.shape)
    g = got.cpu()
    assert torch.equal(g, want), (what, int((g != want).sum()), (g - want).abs().max().item())


@pytest.mark.parametrize("C", [1, 3])
def test_goldens_as_one_list_per_sigma(C, K):
    """The reference's img_lq of every non-empty golden crop, all of one C and sigma in one call."""
    by_sigma = {}
    for name, c in CASES.items():
        lq = _NPZ[f"{name}/lq"]
        if c["channels"] == C and lq.size:
            by_sigma.setdefault(c["sigma"], []).append(name)
    assert by_sigma
    for sigma, names in by_sigma.items():
        imgs = []
        for n in names:
            x = _NPZ[f"{n}/input"]
            imgs.append(torch.from_numpy(x).cuda()[: x.shape[0] // 8 * 8, : x.shape[1] // 8 * 8].contiguous())
        outs = K.awgn_list(imgs, sigma, [CASES[n]["key"] for n in names])
        for n, o in zip(names, outs):
            assert_equal(o, torch.from_numpy(_NPZ[f"{n}/lq"]), n)


def test_mixed_rgb_list_against_recipe(K):
    """CBSD68-sized images, more small images than one launch takes, two Urban100-sized images sharing their key, a
    1 x 1 image and an odd sample count, in one list."""
    g = torch.Generator().manual_seed(3)
    imgs, seeds = [], []
    for i in range(68):
        imgs.append(rand_u8(*((480, 320) if i % 2 else (320, 480)), 3, g))
        seeds.append(f"CBSD68/{i:04d}.png")
    for i in range(70):
        imgs.append(rand_u8(1 + i % 29, 1 + (7 * i) % 31, 3, g))
        seeds.append([int(v) for v in torch.randint(0, 2 ** 32, (8,), generator=g, dtype=torch.int64)])
    imgs += [rand_u8(1024, 768, 3, g), rand_u8(1024, 1024, 3, g), rand_u8(1, 1, 3, g), rand_u8(37, 53, 3, g)]
    seeds += ["Urban100/img_004.png", "Urban100/img_092.png", "Set5/baby.png", "Kodak24/kodim07.png"]
    assert (37 * 53 * 3) % 2 == 1 and len(imgs) > 128
    outs = K.awgn_list(imgs, 15, seeds)
    torch.cuda.synchronize()
    assert len(outs) == len(imgs)
    for i, (img, s, o) in enumerate(zip(imgs, seeds, outs)):
        assert_equal(o, recipe(img, 15, s), (i, tuple(img.shape)))


@pytest.mark.parametrize("sigma", [15, 25, 50])
def test_gray_list_against_recipe(sigma, K):
    g = torch.Generator().manual_seed(sigma)
    sizes = [(256, 256), (481, 321), (1, 1), (7, 9), (64, 200), (200, 64)] + [(1 + i, 2 + 3 * i) for i in range(66)]
    imgs = [rand_u8(h, w, 1, g) for h, w in sizes]
    seeds = [f"Set12/{i:02d}.png" for i in range(len(imgs))]
    outs = K.awgn_list(imgs, sigma, seeds)
    for i, (img, s, o) in enumerate(zip(imgs, seeds, outs)):
        assert_equal(o, recipe(img, sigma, s), (i, sizes[i]))


@pytest.mark.parametrize("C", [1, 3])
def test_batch_equals_list(C, K):
    g = torch.Generator().manual_seed(10 + C)
    x = torch.randint(0, 256, (5, 37, 41, C), generator=g, dtype=torch.uint8).cuda()
    seeds = ["CBSD68/0001.png", "Urban100/img_001.png", list(range(8)), "Urban100/img_002.png", K.dn_seed("x")]
    y = K.awgn(x, 25, seeds)
    assert y.shape == (5, C, 37, 41) and y.dtype == torch.float32
    for b, o in enumerate(K.awgn_list(list(x.unbind(0)), 25, seeds)):
        assert torch.equal(y[b], o), b
    assert_equal(y[2], recipe(x[2], 25, seeds[2]), "words")
    assert K.awgn(x[:0], 25, []).shape == (0, C, 37, 41)


def test_empty_list_and_zero_sigma(K):
    assert K.awgn_list([], 15, []) == []
    img = torch.randint(0, 256, (9, 11, 3), dtype=torch.uint8).cuda()
    (o,) = K.awgn_list([img], 0, ["CBSD68/0001.png"])
    assert torch.equal(o, K.functional.u8_to_f32(img[None])[0])


def test_input_untouched_and_outputs_new(K):
    img = torch.randint(0, 256, (17, 19, 3), dtype=torch.uint8).cuda()
    before = img.clone()
    (o,) = K.awgn_list([img], 15, ["CBSD68/0001.png"])
    assert torch.equal(img, before) and o.data_ptr() != img.data_ptr()


def _delayed_copy(srcs, stream, cycles):
    """Copies of srcs made on `stream` behind a bounded sleep: zero until the sleep ends."""
    with torch.cuda.stream(stream):
        bufs = [torch.zeros_like(t) for t in srcs]
        torch.cuda._sleep(cycles)
        for b, t in zip(bufs, srcs):
            b.copy_(t)
    return bufs


def test_off_the_default_stream_and_across_streams(K):
    """On a side stream behind a sleep, and produced on one stream and consumed on another after wait_stream: the same
    bits as on the default stream.  The control launches on the wrong stream and must see the zeros."""
    from grl_image_restoration_b200 import capi, functional as F

    g = torch.Generator().manual_seed(5)
    srcs = [rand_u8(64, 48, 3, g), rand_u8(31, 17, 3, g), rand_u8(200, 120, 3, g)]
    seeds = ["CBSD68/0001.png", "Urban100/img_001.png", "Kodak24/kodim01.png"]
    want = [o.cpu() for o in K.awgn_list(srcs, 15, seeds)]
    torch.cuda.synchronize()
    cycles = 50_000_000  # tens of milliseconds: far longer than the launches queued behind it take to enqueue
    S, A, B = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    for s in (S, A, B):
        s.wait_stream(torch.cuda.current_stream())

    bufs = _delayed_copy(srcs, S, cycles)
    with torch.cuda.stream(S):
        outs = K.awgn_list(bufs, 15, seeds)
        batch = K.awgn(bufs[0][None], 15, seeds[:1])
    torch.cuda.current_stream().wait_stream(S)
    for o, w in zip(outs, want):
        assert torch.equal(o.cpu(), w)
    assert torch.equal(batch[0].cpu(), want[0])

    bufs = _delayed_copy(srcs, A, cycles)
    B.wait_stream(A)
    with torch.cuda.stream(B):
        outs = K.awgn_list(bufs, 15, seeds)
    torch.cuda.current_stream().wait_stream(B)
    for o, w in zip(outs, want):
        assert torch.equal(o.cpu(), w)

    # control: the same call launched on another stream than the one the inputs are ordered on
    bufs = _delayed_copy(srcs, S, cycles)
    with torch.cuda.stream(S):
        outs = [torch.empty(3, t.shape[0], t.shape[1], device="cuda") for t in bufs]
    keys = F._awgn_keys(seeds, 3, "control")
    other = torch.cuda.Stream()
    capi.check(capi.lib().grl_awgn_u8(F._image_refs(bufs, capi.IMAGE_U8), F._image_refs(outs, capi.IMAGE_F32),
                                      keys.ctypes.data_as(ctypes.c_void_p), 3, 3, 15 / 255, ctypes.c_void_p(other.cuda_stream)))
    other.synchronize()
    assert not torch.equal(outs[0].cpu(), want[0]), "a launch on the wrong stream went unnoticed"
    torch.cuda.synchronize()


def test_refusals(K):
    img = torch.zeros(2, 16, 16, 3, dtype=torch.uint8, device="cuda")
    seeds = ["a.png", "b.png"]
    for sigma in (-1, float("nan"), float("inf"), True, "15", None):
        with pytest.raises(ValueError):
            K.awgn(img, sigma, seeds)
        with pytest.raises(ValueError):
            K.awgn_list(list(img), sigma, seeds)
    with pytest.raises(RuntimeError):
        K.awgn(img.cpu(), 15, seeds)
    with pytest.raises(RuntimeError):
        K.awgn_list([img[0], img[1].cpu()], 15, seeds)
    for bad in (img.float(), img[..., :2], torch.zeros(2, 16, 16, 4, dtype=torch.uint8, device="cuda"), img[0],
                torch.zeros(2, 0, 16, 3, dtype=torch.uint8, device="cuda")):
        with pytest.raises(ValueError):
            K.awgn(bad, 15, seeds)
    with pytest.raises(ValueError):
        K.awgn_list([img[0], img[1, ..., :1]], 15, seeds)  # mixed C
    with pytest.raises(ValueError):
        K.awgn_list([img[0], img[1].float()], 15, seeds)
    for bad_seeds in (seeds[:1], seeds * 2, ["a.png", [1] * 7], ["a.png", [2 ** 32] + [0] * 7], ["a.png", None]):
        with pytest.raises(ValueError):
            K.awgn(img, 15, bad_seeds)
        with pytest.raises(ValueError):
            K.awgn_list(list(img), 15, bad_seeds)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_micro_denoiser_on_device_noise(precision, K, oracle):
    """Wiring: dn_seed -> crop -> awgn_list -> forward_list equals forward_list of the recipe's inputs moved to the
    device, bit for bit."""
    m = micro(K, oracle, "micro_pad_dn", torch.device("cuda:0"), precision)
    g = torch.Generator().manual_seed(21)
    gts = [rand_u8(h, w, 3, g) for h, w in [(45, 61), (33, 50), (24, 40), (70, 41)]]
    names = ["CBSD68/0001.png", "Kodak24/kodim01.png", "Urban100/img_004.png", "Urban100/img_092.png"]
    crops = [t[: t.shape[0] // 8 * 8, : t.shape[1] // 8 * 8].contiguous() for t in gts]
    lq = K.awgn_list(crops, 15, names)
    want = m.forward_list([recipe(c, 15, n).cuda() for c, n in zip(crops, names)])
    got = m.forward_list(lq)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), i
