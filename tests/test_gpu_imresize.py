"""The bicubic downscale on the GPU (csrc/resize.cu): the kernel equal to the library's host copy with torch.equal on
float batches and every fixture input, within the derived bound (tests/test_imresize.py) of the float64 oracle on every
fixture; the 8-bit list equal to the batch of u8_to_f32 images over mixed lists, an Urban100-sized and a DIV2K-sized
image; inputs untouched; streams; refusals; evaluate(synthesize_lr=True) equal to the calls by hand on micro SR models of
upscale 2, 3 and 4; and tools/evaluate.py --bicubic-lr scoring a checkpoint from HR image files alone."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import imresize_oracle as oracle
from support import build, same_bits

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLD, "imresize_cases.json")) as f:
    CASES = json.load(f)["cases"]
_NPZ = np.load(os.path.join(GOLD, "imresize.npz"))
MIN = {2: 4, 3: 6, 4: 7}


@pytest.fixture(scope="module")
def K(pkg):
    assert torch.cuda.is_available()
    return pkg


def rand_u8(h, w, C, g):
    return torch.randint(0, 256, (h, w, C), generator=g, dtype=torch.uint8).cuda()


def host(x, s):
    from grl_image_restoration_b200 import functional as F

    return F.imresize_host(x.cpu(), 1 / s)


@pytest.mark.parametrize("s", oracle.SCALES)
@pytest.mark.parametrize("C", [1, 3, 8])
def test_float_batches_equal_the_host_copy(s, C, K):
    g = torch.Generator().manual_seed(10 * s + C)
    m = MIN[s]
    for B, H, W in ((2, 37, 53), (1, 64, 64), (3, m, m), (1, m, 70), (2, 1, 1), (1, 1, 40), (1, 100, 33), (1, 181, 301)):
        x = (torch.rand(B, C, H, W, generator=g) * 1.5 - 0.25).cuda()
        y = K.imresize(x, 1 / s)
        assert y.shape == (B, C, -(-H // s), -(-W // s)) and y.dtype == torch.float32
        assert torch.equal(y.cpu(), host(x, s)), (s, C, B, H, W)


@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_equal_the_host_copy_and_sit_within_the_bound(name, K):
    from grl_image_restoration_b200 import functional as F

    c = CASES[name]
    s, img = c["s"], torch.from_numpy(_NPZ[f"{name}/input"])
    x = F.u8_to_f32(img[None].cuda()) if c["kind"] == "u8" else img[None].cuda()
    y = K.imresize(x, 1 / s)
    assert torch.equal(y.cpu(), host(x, s)), name
    v = x[0].double().cpu().numpy()
    assert (np.abs(y[0].double().cpu().numpy() - oracle.resize(v, s)) <= oracle.host_bound(v, s)).all(), name
    if c["kind"] == "u8":
        (o,) = K.imresize_list([img.cuda()], 1 / s)
        assert torch.equal(o, y[0]), name


def _assert_list_equals_batch(K, imgs, s):
    from grl_image_restoration_b200 import functional as F

    outs = K.imresize_list(imgs, 1 / s)
    assert len(outs) == len(imgs)
    for i, (img, o) in enumerate(zip(imgs, outs)):
        want = K.imresize(F.u8_to_f32(img[None]), 1 / s)[0]
        assert o.shape == want.shape and torch.equal(o, want), (i, tuple(img.shape))


@pytest.mark.parametrize("s", oracle.SCALES)
@pytest.mark.parametrize("C", [1, 3])
def test_mixed_list_equals_the_batch(s, C, K):
    """More images than one launch takes (64), of sides from 1 and the minimum up, in one call."""
    g = torch.Generator().manual_seed(100 * s + C)
    sizes = [(MIN[s] + (7 * i) % 53, MIN[s] + (11 * i) % 61) for i in range(140)] + [(1, 1), (1, 19), (23, 1)]
    _assert_list_equals_batch(K, [rand_u8(h, w, C, g) for h, w in sizes], s)


@pytest.mark.parametrize("s", oracle.SCALES)
def test_urban100_and_div2k_sized_images(s, K):
    g = torch.Generator().manual_seed(s)
    imgs = [rand_u8(1024, 768, 3, g), rand_u8(1356, 2040, 3, g), rand_u8(2040, 1356, 3, g)]
    _assert_list_equals_batch(K, imgs, s)
    x = K.functional.u8_to_f32(imgs[1][None])
    assert torch.equal(K.imresize(x, 1 / s).cpu(), host(x, s))


def test_inputs_untouched_and_outputs_new(K):
    g = torch.Generator().manual_seed(1)
    imgs = [rand_u8(37, 41, 3, g), rand_u8(64, 48, 3, g)]
    before = [t.clone() for t in imgs]
    outs = K.imresize_list(imgs, 1 / 2)
    x = torch.rand(2, 3, 40, 50, generator=g).cuda()
    xb = x.clone()
    y = K.imresize(x, 1 / 3)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(imgs, before)) and torch.equal(x, xb)
    assert len({o.data_ptr() for o in outs} | {t.data_ptr() for t in imgs} | {y.data_ptr(), x.data_ptr()}) == 6
    assert K.imresize_list([], 1 / 4) == [] and K.imresize(x[:0], 1 / 4).shape == (0, 3, 10, 13)


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
    want = [o.cpu() for o in K.imresize_list(srcs, 1 / 3)]
    want_b = K.imresize(F.u8_to_f32(srcs[0][None]), 1 / 3).cpu()
    torch.cuda.synchronize()
    cycles = 50_000_000  # tens of milliseconds: far longer than the launches queued behind it take to enqueue
    S, A, B = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    for st in (S, A, B):
        st.wait_stream(torch.cuda.current_stream())

    bufs = _delayed_copy(srcs, S, cycles)
    with torch.cuda.stream(S):
        outs = K.imresize_list(bufs, 1 / 3)
        batch = K.imresize(F.u8_to_f32(bufs[0][None]), 1 / 3)
    torch.cuda.current_stream().wait_stream(S)
    for o, w in zip(outs, want):
        assert torch.equal(o.cpu(), w)
    assert torch.equal(batch.cpu(), want_b)

    bufs = _delayed_copy(srcs, A, cycles)
    B.wait_stream(A)
    with torch.cuda.stream(B):
        outs = K.imresize_list(bufs, 1 / 3)
    torch.cuda.current_stream().wait_stream(B)
    for o, w in zip(outs, want):
        assert torch.equal(o.cpu(), w)

    # control: the same call launched on another stream than the one the inputs are ordered on
    bufs = _delayed_copy(srcs, S, cycles)
    with torch.cuda.stream(S):
        outs = [torch.empty(3, -(-t.shape[0] // 3), -(-t.shape[1] // 3), device="cuda") for t in bufs]
    other = torch.cuda.Stream()
    capi.check(capi.lib().grl_imresize_u8_list(F._image_refs(bufs, capi.IMAGE_U8), F._image_refs(outs, capi.IMAGE_F32),
                                               3, 3, 3, ctypes.c_void_p(other.cuda_stream)))
    other.synchronize()
    assert not torch.equal(outs[0].cpu(), want[0]), "a launch on the wrong stream went unnoticed"
    torch.cuda.synchronize()


def test_refusals(K):
    img = torch.zeros(16, 16, 3, dtype=torch.uint8, device="cuda")
    x = torch.zeros(1, 3, 16, 16, device="cuda")
    for bad in (2, 0.3, 1 / 5, True, None):
        with pytest.raises(ValueError, match="1/2, 1/3 and 1/4"):
            K.imresize(x, bad)
        with pytest.raises(ValueError, match="1/2, 1/3 and 1/4"):
            K.imresize_list([img], bad)
    with pytest.raises(RuntimeError):
        K.imresize(x.cpu(), 1 / 2)
    with pytest.raises(RuntimeError):
        K.imresize(x.double(), 1 / 2)
    with pytest.raises(RuntimeError):
        K.imresize(torch.zeros(1, 9, 16, 16, device="cuda"), 1 / 2)
    with pytest.raises(RuntimeError, match="too small"):
        K.imresize(torch.zeros(1, 3, 5, 16, device="cuda"), 1 / 4)
    with pytest.raises(RuntimeError, match="too small"):
        K.imresize_list([img, img[:3]], 1 / 2)
    with pytest.raises(ValueError):
        K.imresize_list([img, img[..., :1]], 1 / 2)  # mixed C
    with pytest.raises(ValueError):
        K.imresize_list([img.float()], 1 / 2)
    with pytest.raises(RuntimeError):
        K.imresize_list([img.cpu()], 1 / 2)


def sr_model(K, oracle_mod, s, precision):
    cfg = K.configs.micro_config(upscale=s)
    return build(K, oracle_mod, cfg, torch.device("cuda:0"), precision, style="init")


@pytest.mark.parametrize("s", oracle.SCALES)
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_evaluate_synthesize_lr_equals_the_calls_by_hand(s, precision, K, oracle):
    """crop -> imresize_list -> forward_list -> f32_to_u8 -> psnr_fused / ssim_fused, bit for bit."""
    from grl_image_restoration_b200 import functional as F, metrics

    m = sr_model(K, oracle, s, precision)
    g = torch.Generator().manual_seed(40 + s)
    gts = [rand_u8(h, w, 3, g) for h, w in [(61, 75), (72, 56), (65, 90), (MIN[s] * s + 1, 50)]]
    name = f"sr_grl_tiny_c3x{s}.ckpt"
    got = K.evaluate(m, name, gts, synthesize_lr=True)
    clean = [t[: t.shape[0] // s * s, : t.shape[1] // s * s] for t in gts]
    lq = K.imresize_list([c.contiguous() for c in clean], 1 / s)
    outs = [F.f32_to_u8(o[None])[0] for o in m.forward_list(lq)]
    want = {}
    for o, c in zip(outs, clean):
        p, py = metrics.psnr_fused(o[None], c[None], s)
        ss, sy = metrics.ssim_fused(o[None], c[None], s)
        for k, v in (("val_psnr", p), ("val_psnr_y", py), ("val_ssim", ss), ("val_ssim_y", sy)):
            want.setdefault(k, []).append(v[0])
    assert list(got["scores"]) == list(want)
    for k, vs in want.items():
        w = torch.stack(vs).cpu()
        assert not w.isnan().any(), (k, w)
        same_bits(got["scores"][k], w)
    with pytest.raises(ValueError, match="low-quality"):
        K.evaluate(m, name, gts)  # the file-based path is unchanged: it still needs lqs


def test_cli_scores_an_sr_checkpoint_from_hr_files(K, oracle, tmp_path):
    """tools/evaluate.py NAME --gt DIR --bicubic-lr prints a table from HR files alone; without --bicubic-lr or --lq it
    still exits with 'needs --lq'."""
    cv2 = pytest.importorskip("cv2")
    name = "sr_grl_tiny_c3x2.ckpt"
    cfg = K.configs.released_config(name, img_size=256)
    sd = oracle.synth_state_dict(cfg, seed=3, style="init")
    ckpt = tmp_path / "sr.ckpt"
    torch.save({"state_dict": {"model." + k: v for k, v in sd.items()}}, ckpt)
    gt = tmp_path / "Set5"
    gt.mkdir()
    rng = np.random.default_rng(0)
    for i, (h, w) in enumerate([(41, 57), (64, 48)]):
        cv2.imwrite(str(gt / f"{i}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    cmd = [sys.executable, os.path.join(ROOT, "tools", "evaluate.py"), str(ckpt), name, "--gt", str(gt),
           "--precision", "fp32"]
    r = subprocess.run(cmd + ["--bicubic-lr"], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "val_psnr " in r.stdout and "(2 images)" in r.stdout, r.stdout
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode != 0 and "needs --lq" in r.stderr, r.stderr[-2000:]
