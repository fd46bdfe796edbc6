"""Lists of differently sized images on the GPU: the pad-gather and crop-scatter kernels (csrc/image_list.cu) bit-exact
against check_image_size / to_tensor / demosaic and slices / tensor_round, and GRL.forward_list / forward_list_u8 equal,
bit for bit, to the loop of B = 1 forwards they replace, on every precision, input format, CUDA-graph and self-ensemble
setting.  A forward of a batch gives each image what its own forward gives, so any difference here is a kernel whose
result depends on the rest of the batch."""
import pytest
import torch

from engine_oracle import check_image_size, to_tensor
from support import MICRO, assert_equal_lists, build, count_calls, dm_model, micro, random_images, round8_ref

pytestmark = pytest.mark.gpu


# sizes against a (48, 40) batch: 1 x 1, a pad >= size on one axis only (zeros on both), the exact batch size, odd sizes,
# one that reflects by exactly size - 1 rows
SPECIAL = [(1, 1), (40, 5), (5, 40), (48, 40), (17, 33), (25, 21), (47, 39), (24, 20), (33, 3)]


def sizes_for(n, Hp, Wp, seed):
    g = torch.Generator().manual_seed(seed)
    rest = [(int(torch.randint(1, Hp + 1, (1,), generator=g)), int(torch.randint(1, Wp + 1, (1,), generator=g)))
            for _ in range(n - len(SPECIAL))]
    return SPECIAL + rest


@pytest.mark.parametrize("C", [1, 3, 6])
@pytest.mark.parametrize("u8", [False, True])
def test_gather_bit_exact(pkg, device, C, u8):
    """130 images: more than one launch's worth of descriptors."""
    from grl_image_restoration_b200 import capi, functional as K

    Hp, Wp = 48, 40
    sizes = sizes_for(130, Hp, Wp, C + 10 * u8)
    g = torch.Generator().manual_seed(C)
    if u8:
        imgs = [torch.randint(0, 256, (h, w, C), dtype=torch.uint8, generator=g).to(device) for h, w in sizes]
        refs = [check_image_size(to_tensor(x)[None], Hp, Wp)[0] for x in imgs]
    else:
        imgs = [(torch.randn(C, h, w, generator=g) * 2).to(device) for h, w in sizes]
        refs = [check_image_size(x[None].cpu(), Hp, Wp)[0] for x in imgs]
    out = K.list_gather(imgs, capi.IMAGE_U8 if u8 else capi.IMAGE_F32, C, Hp, Wp)
    assert out.shape == (130, C, Hp, Wp) and out.dtype == torch.float32
    out = out.cpu()
    for i, (r, s) in enumerate(zip(refs, sizes)):
        assert torch.equal(out[i], r), (i, s)


def test_gather_equals_check_image_size(pkg, device):
    """Images that pad to the batch's size: each slice is exactly the model's check_image_size of the image."""
    from grl_image_restoration_b200 import capi, functional as K

    m = pkg.GRL(**pkg.configs.micro_config())
    assert m.pad_size == 16
    g = torch.Generator().manual_seed(3)
    # one list per padded size; the 16 x 32 images are smaller than a pad on one axis: zeros on both
    for (Hp, Wp), sizes in {(32, 32): [(20, 30), (32, 32), (17, 17), (31, 20)],
                            (16, 32): [(5, 24), (1, 30), (16, 17)]}.items():
        imgs = [torch.rand(3, h, w, generator=g).to(device) for h, w in sizes]
        out = K.list_gather(imgs, capi.IMAGE_F32, 3, Hp, Wp)
        assert torch.equal(out, torch.cat([m.check_image_size(x[None]) for x in imgs]))


def test_gather_rggb_equals_padded_demosaic(pkg, device):
    from grl_image_restoration_b200 import capi, functional as K

    Hp, Wp = 64, 48
    packed = [(2, 2), (9, 13), (32, 24), (20, 3), (5, 24), (17, 11)] + [(2 + i % 30, 2 + (7 * i) % 22) for i in range(124)]
    g = torch.Generator().manual_seed(5)
    cfa = [torch.rand(4, h, w, generator=g).to(device) for h, w in packed]
    out = K.list_gather(cfa, capi.IMAGE_RGGB, 3, Hp, Wp)
    for i, x in enumerate(cfa):
        assert torch.equal(out[i:i + 1], check_image_size(K.demosaic(x[None]), Hp, Wp)), (i, packed[i])


@pytest.mark.parametrize("C", [1, 3, 6])
@pytest.mark.parametrize("u8", [False, True])
def test_crop_bit_exact(pkg, device, C, u8):
    from grl_image_restoration_b200 import functional as K

    Hy, Wy = 96, 80
    sizes = [(96, 80), (1, 1), (33, 7), (95, 79), (8, 80)] + [(1 + i % 13, 1 + (3 * i) % 17) for i in range(126)]
    y = torch.rand(len(sizes), C, Hy, Wy, generator=torch.Generator().manual_seed(C)) * 1.4 - 0.2
    special = torch.tensor([0.0, -0.0, 1.0, 0.5 / 255, 1.5 / 255, 254.5 / 255, float("nan"), float("inf"), float("-inf"),
                            -1e-8, 1.0000001])
    y[:, :, 0, : special.numel()] = special
    outs = K.list_crop(y.to(device), sizes, u8=u8)
    assert len(outs) == len(sizes)
    for i, (o, (h, w)) in enumerate(zip(outs, sizes)):
        want = y[i, :, :h, :w]
        want = round8_ref(want) if u8 else want.contiguous().view(torch.int32)  # fp32: the bits, NaN included
        o = o.cpu() if u8 else o.cpu().view(torch.int32)
        assert o.shape == want.shape and torch.equal(o, want), (i, h, w)


# ------------------------------------------------------------------------------------------ end to end
# several buckets, repeats of one bucket, both orientations, zero padding on one axis, a 1-pixel-wide image
SIZES = [(24, 40), (40, 24), (17, 30), (24, 40), (9, 9), (30, 5), (33, 20), (20, 33), (1, 12), (16, 16)]


@pytest.mark.parametrize("name", list(MICRO))
@pytest.mark.parametrize("precision,ensemble,graph", [("fp32", False, False), ("fp16", False, False),
                                                      ("bf16", False, False), ("fp16", False, True),
                                                      ("fp32", True, False), ("fp16", True, False)])
def test_forward_list_equals_loop(pkg, oracle, device, name, precision, ensemble, graph):
    from grl_image_restoration_b200 import image_list

    m = micro(pkg, oracle, name, device, precision, self_ensemble=ensemble)
    m.use_cuda_graph = graph
    xs = random_images(lambda h, w: (m.in_channels, h, w), SIZES, list(MICRO).index(name), device)
    kept = [x.clone() for x in xs]
    want = [m(x[None])[0] for x in xs]
    calls = count_calls(m, "_forward_once")
    got = m.forward_list(xs)
    assert_equal_lists(got, want)
    assert all(torch.equal(a, b) for a, b in zip(xs, kept)), "forward_list changed its inputs"
    sizes = image_list.network_sizes([tuple(x.shape) for x in xs])
    if not ensemble:
        chunks = image_list.plan(sizes, m.pad_size, m.max_batch_tokens)
        assert len(chunks) < len(xs) and calls == [(len(c.index), m.in_channels, c.hp, c.wp) for c in chunks]
    if graph:
        assert any(k[0][0] > 1 for k in m._graphs), "the batched forward must have replayed a captured graph"
        assert_equal_lists(m.forward_list(xs), want)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_forward_list_splits_a_bucket_at_the_budget(pkg, oracle, device, precision):
    m = micro(pkg, oracle, "micro_cab_x2", device, precision)
    sizes = [(24, 40), (20, 33), (32, 48), (24, 40), (30, 35), (17, 40), (32, 33)]  # all pad to 32 x 48
    xs = random_images(lambda h, w: (3, h, w), sizes, 11, device)
    want = [m(x[None])[0] for x in xs]
    m.max_batch_tokens = 3 * 32 * 48
    calls = count_calls(m, "_forward_once")
    assert_equal_lists(m.forward_list(xs), want)
    assert [c[0] for c in calls] == [3, 3, 1]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_forward_list_other_float_dtypes(pkg, oracle, device, precision, dtype):
    """Half-precision inputs give the dtype and the bits of the image's own forward."""
    m = micro(pkg, oracle, "micro_pad_dn", device, precision)
    xs = random_images(lambda h, w: (3, h, w), SIZES[:6], 2, device, dtype)
    assert_equal_lists(m.forward_list(xs), [m(x[None])[0] for x in xs])


@pytest.mark.parametrize("precision,ensemble,graph", [("fp32", False, False), ("fp16", False, False),
                                                      ("bf16", False, False), ("fp16", False, True),
                                                      ("fp16", True, False)])
def test_forward_list_rggb(pkg, oracle, device, precision, ensemble, graph):
    m = dm_model(pkg, oracle, device, precision, self_ensemble=ensemble)
    m.use_cuda_graph = graph
    packed = [(10, 14), (9, 13), (2, 2), (10, 14), (14, 10), (20, 28), (16, 3)]
    xs = random_images(lambda h, w: (4, h, w), packed, 4, device)
    want = [m(x[None])[0] for x in xs]
    calls = count_calls(m, "_forward_once")
    got = m.forward_list(xs)
    assert_equal_lists(got, want)
    assert got[0].shape == (3, 20, 28)
    if not ensemble:
        assert len(calls) < len(xs)
    half = [x.half() for x in xs]
    assert_equal_lists(m.forward_list(half), [m(x[None])[0] for x in half])


@pytest.mark.parametrize("name", ["micro_cab_x2", "micro_gray", "micro_dual"])
@pytest.mark.parametrize("precision,ensemble,graph", [("fp32", False, False), ("fp16", False, False),
                                                      ("fp16", False, True), ("fp16", True, False)])
def test_forward_list_u8_equals_loop(pkg, oracle, device, name, precision, ensemble, graph):
    m = micro(pkg, oracle, name, device, precision, self_ensemble=ensemble)
    m.use_cuda_graph = graph
    g = torch.Generator().manual_seed(8)
    xs = [torch.randint(0, 256, (h, w, m.in_channels), dtype=torch.uint8, generator=g).to(device) for h, w in SIZES]
    kept = [x.clone() for x in xs]
    want = [m.forward_u8(x[None])[0] for x in xs]
    got = m.forward_list_u8(xs)
    assert_equal_lists(got, want)
    assert all(torch.equal(a, b) for a, b in zip(xs, kept))


def test_cuda_graphs_of_several_resolutions_replay_exactly(pkg, oracle, device):
    """Each block caches its attention constants for the last resolution it ran; a captured graph reads them at their
    address, so it must keep them alive when a forward at another resolution replaces the cache."""
    m = micro(pkg, oracle, "micro_cab_x2", device, "fp16")
    xs = random_images(lambda h, w: (3, 1, h, w), [(32, 48), (48, 32), (16, 16), (32, 32)], 12, device)
    eager = [m(x) for x in xs]
    m.use_cuda_graph = True
    for _ in range(2):
        for x, want in zip(xs, eager):
            assert torch.equal(m(x), want)
            # fill whatever small blocks a forward has released with NaN
            junk = [torch.full((n,), float("nan"), device=device) for n in range(64, 16384, 64)]
            del junk


def test_forward_list_base_x4_b100_sizes(pkg, oracle, device):
    """The released GRL-Base x4 SR architecture on whole B100-sized images: both orientations share one forward."""
    cfg = pkg.configs.grl_config("base", "sr", 4, 64)
    m = build(pkg, oracle, cfg, device, "fp16", style="init")
    xs = random_images(lambda h, w: (3, h, w), [(120, 80), (80, 120), (120, 80)], 21, device)
    want = [m(x[None])[0] for x in xs]
    calls = count_calls(m, "_forward_once")
    got = m.forward_list(xs)
    assert calls == [(3, 3, 128, 128)]
    assert_equal_lists(got, want)
    assert got[1].shape == (3, 320, 480)


def test_forward_list_rejects_bad_input_before_launching(pkg, oracle, device):
    from grl_image_restoration_b200 import capi

    m = micro(pkg, oracle, "micro_cab_x2", device, "fp16")
    good = torch.rand(3, 20, 20, device=device)
    bad = {
        "wrong rank": (ValueError, "shape", torch.rand(1, 3, 20, 20, device=device)),
        "wrong channel count": (ValueError, "shape", torch.rand(4, 20, 20, device=device)),
        "empty axis": (ValueError, "shape", torch.rand(3, 0, 20, device=device)),
        "wrong dtype": (ValueError, "dtype", torch.rand(3, 20, 20, device=device, dtype=torch.float64)),
        "integer dtype": (ValueError, "dtype", torch.zeros(3, 20, 20, device=device, dtype=torch.uint8)),
        "cpu tensor": (RuntimeError, "CUDA device", torch.rand(3, 20, 20)),
        "mixed dtypes": (ValueError, "different dtypes", good.half()),
    }
    for what, (exc, msg, x) in bad.items():
        before = capi.lib().grl_launch_count()
        with pytest.raises(exc, match=msg):
            m.forward_list([good, x])
        assert capi.lib().grl_launch_count() == before, what
    if torch.cuda.device_count() > 1:
        with pytest.raises(RuntimeError, match="current device"):
            m.forward_list([good, torch.rand(3, 20, 20, device="cuda:1")])
    with pytest.raises(ValueError, match="shape"):
        m.forward_list_u8([torch.zeros(20, 20, 4, dtype=torch.uint8, device=device)])
    with pytest.raises(ValueError, match="dtype"):
        m.forward_list_u8([good])
    bayer = dm_model(pkg, oracle, device, "fp16")
    with pytest.raises(ValueError, match="h, w >= 2"):
        bayer.forward_list([torch.rand(4, 1, 8, device=device)])
    with pytest.raises(ValueError, match="input_format='rggb'"):
        bayer.forward_list_u8([torch.zeros(8, 8, 3, dtype=torch.uint8, device=device)])
    assert m.forward_list([]) == [] and m.forward_list_u8([]) == []
