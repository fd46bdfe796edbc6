"""The dataset-side input kernels (csrc/dataset_u8.cu) against the reference's fixtures and their host copies, as batches
and as lists, and evaluation.evaluate on micro models: for every task row the scores equal, bit for bit, those of the
same public calls composed by hand, so the recipe wiring is pinned; one run off the default stream; and a two-rank split
whose gathered means equal the single-process means."""
import os

import numpy as np
import pytest
import torch

from support import micro, same_bits

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_NPZ = np.load(os.path.join(GOLD, "eval_inputs.npz"))
MOSAIC = sorted({k.split("/")[0] for k in _NPZ.files if k.endswith("/mosaic")})
NIQE = os.path.join(GOLD, "niqe_pris_params.npz")


@pytest.fixture(scope="module")
def K(pkg):
    assert torch.cuda.is_available()
    return pkg


def rand_u8(h, w, C, g):
    return torch.randint(0, 256, (h, w, C), generator=g, dtype=torch.uint8).cuda()


def test_mosaic_goldens_as_list_and_batches(K):
    imgs = [torch.from_numpy(_NPZ[f"{n}/img"]).cuda() for n in MOSAIC]
    outs = K.mosaic_list(imgs)
    for n, o in zip(MOSAIC, outs):
        want = torch.from_numpy(_NPZ[f"{n}/mosaic"])
        assert o.dtype == torch.float32 and o.shape == want.shape and torch.equal(o.cpu(), want), n
        b = K.mosaic(torch.from_numpy(_NPZ[f"{n}/img"]).cuda()[None].expand(3, -1, -1, -1))
        assert b.shape == (3, *want.shape) and all(torch.equal(b[i].cpu(), want) for i in range(3)), n


def test_mosaic_long_list_against_host(K):
    """More images than one launch takes (128), odd and even sizes, one 1-row image."""
    from grl_image_restoration_b200 import functional as F

    g = torch.Generator().manual_seed(1)
    sizes = [(1 + (7 * i) % 61, 1 + (11 * i) % 67) for i in range(300)] + [(1, 9), (481, 321), (2, 2)]
    imgs = [rand_u8(h, w, 3, g) for h, w in sizes]
    outs = K.mosaic_list(imgs)
    torch.cuda.synchronize()
    for i, (img, o) in enumerate(zip(imgs, outs)):
        assert torch.equal(o.cpu(), F.mosaic_host(img.cpu())), (i, sizes[i])


def test_luma_goldens_and_every_triple(K):
    from grl_image_restoration_b200 import functional as F

    rgb = torch.from_numpy(_NPZ["luma/rgb"]).cuda()
    (y,) = K.luma_list([rgb[None]])
    assert y.shape == (1, rgb.shape[0], 1) and torch.equal(y[0, :, 0].cpu(), torch.from_numpy(_NPZ["luma/y"]))
    cube = torch.arange(1 << 24, dtype=torch.int64)
    cube = torch.stack([cube >> 16, (cube >> 8) & 255, cube & 255], 1).to(torch.uint8).reshape(4096, 4096, 3)
    got = K.luma(cube.cuda()[None])[0]
    assert torch.equal(got.cpu(), F.luma_host(cube))


def test_luma_long_list_and_batch(K):
    from grl_image_restoration_b200 import functional as F

    g = torch.Generator().manual_seed(2)
    imgs = [rand_u8(1 + i % 37, 1 + (5 * i) % 41, 3, g) for i in range(260)]
    outs = K.luma_list(imgs)
    for i, (img, o) in enumerate(zip(imgs, outs)):
        assert o.shape == (*img.shape[:2], 1) and torch.equal(o.cpu(), F.luma_host(img.cpu())), i
    x = torch.randint(0, 256, (4, 33, 47, 3), generator=g, dtype=torch.uint8).cuda()
    y = K.luma(x)
    for b, o in enumerate(K.luma_list(list(x.unbind(0)))):
        assert torch.equal(y[b], o), b


def test_refusals(K):
    img = torch.zeros(2, 16, 16, 3, dtype=torch.uint8, device="cuda")
    for fn in (K.mosaic, K.luma):
        with pytest.raises(RuntimeError):
            fn(img.cpu())
        for bad in (img.float(), img[..., :1], img[0], torch.zeros(2, 0, 16, 3, dtype=torch.uint8, device="cuda")):
            with pytest.raises(ValueError):
                fn(bad)
    for fn in (K.mosaic_list, K.luma_list):
        assert fn([]) == []
        with pytest.raises(ValueError):
            fn([img[0], img[1, ..., :1]])


# ---- evaluate ------------------------------------------------------------------------------------------------------------
# task row -> (checkpoint name, micro architecture, extra GRL kwargs)
ROWS = {
    "sr": ("sr_grl_tiny_c3x2.ckpt", "micro_cab_x2", {}),
    "dn_c3": ("dn_grl_base_c3s15.ckpt", "micro_pad_dn", {}),
    "dn_c1": ("dn_grl_small_c1s15.ckpt", "micro_gray", {}),
    "jpeg_c3": ("jpeg_grl_small_c3q10.ckpt", "micro_pad_dn", {}),
    "jpeg_c1": ("jpeg_grl_small_c1q10.ckpt", "micro_gray", {}),
    "dm": ("dm_grl_small.ckpt", "micro_pad_dn", {"input_format": "rggb"}),
    "bsr": ("bsr_grl_base.ckpt", "micro_pad_dn", {}),
    "defocus": ("db_defocus_single_pixel_grl_base.ckpt", "micro_pad_dn", {}),
    "defocus_dual": ("db_defocus_dual_pixel_grl_base.ckpt", "micro_dual", {}),
    "motion": ("db_motion_grl_base_gopro.ckpt", "micro_pad_dn", {}),
}


def row_data(row, seed=0):
    """(gts, lqs, keys, dataset) of a small test set for a row."""
    g = torch.Generator().manual_seed(100 + seed)
    sizes = [(200, 104), (104, 197), (196, 196)] if row == "bsr" else [(61, 75), (72, 56), (65, 90)]
    C = 1 if row == "dn_c1" else 3
    gts = [rand_u8(h, w, C, g) for h, w in sizes]
    lqs = keys = dataset = None
    if row == "sr":
        lqs = [rand_u8(h // 2, w // 2, 3, g) for h, w in sizes]
    elif row in ("defocus", "motion"):
        lqs = [rand_u8(h, w, 3, g) for h, w in sizes]
    elif row == "defocus_dual":
        lqs = [(rand_u8(h, w, 3, g), rand_u8(h, w, 3, g)) for h, w in sizes]
    elif row.startswith("dn"):
        dataset = "CBSD68" if C == 3 else "Set12"
        keys = [f"{dataset}/{i:04d}.png" for i in range(len(gts))]
    elif row == "jpeg_c1":
        dataset = "live1"  # the luma of the RGB images
    return gts, lqs, keys, dataset


def by_hand(K, m, row, gts, lqs, keys):
    """The row's test command composed from the public calls."""
    from grl_image_restoration_b200 import functional as F, metrics, tiling

    def u8(ys):
        return [F.f32_to_u8(y[None])[0] for y in ys]

    if row == "sr":
        clean = [g[: g.shape[0] // 2 * 2, : g.shape[1] // 2 * 2] for g in gts]
        outs, border = m.forward_list_u8(lqs), 2
    elif row.startswith("dn"):
        clean = [g[: g.shape[0] // 8 * 8, : g.shape[1] // 8 * 8].contiguous() for g in gts]
        lq = K.awgn_list(clean, 15, keys)
        outs = u8(tiling.forward_tile_list(m, lq, 256, 32) if row == "dn_c3" else m.forward_list(lq))
        border = 0
    elif row.startswith("jpeg"):
        clean = K.luma_list(gts) if row == "jpeg_c1" else gts
        outs, border = tiling.forward_tile_list_u8(m, K.jpeg_roundtrip_list(clean, 10), 288, 36), 0
    elif row == "dm":
        clean = [g[: g.shape[0] // 8 * 8, : g.shape[1] // 8 * 8] for g in gts]
        outs, border = u8(m.forward_list(K.mosaic_list(clean))), 0
    elif row == "bsr":
        outs = m.forward_list_u8(gts)
        return {"val_niqe": [metrics.niqe(o[None], NIQE)[0] for o in outs]}
    elif row == "defocus_dual":
        clean = gts
        outs, border = tiling.forward_tile_list_u8(m, [torch.cat(p, 2) for p in lqs], 480, 48), 0
    elif row == "defocus":
        clean, outs, border = gts, tiling.forward_tile_list_u8(m, lqs, 480, 48), 0
    else:
        clean, outs, border = gts, m.forward_list_u8(lqs), 0
    res = {}
    for o, c in zip(outs, clean):
        p, py = metrics.psnr_fused(o[None], c[None], border)
        s, sy = metrics.ssim_fused(o[None], c[None], border)
        vals = {"val_psnr": p, "val_psnr_y": py, "val_ssim": s, "val_ssim_y": sy}
        if row.startswith("jpeg"):
            pb, pby = metrics.psnrb_fused(o[None], c[None])
            vals.update(val_psnrb=pb, val_psnrb_y=pby)
        if C1(row):
            vals = {k: v for k, v in vals.items() if not k.endswith("_y")}
        for k, v in vals.items():
            res.setdefault(k, []).append(v[0])
    return res


def C1(row):
    return row in ("dn_c1", "jpeg_c1")


def model_for(K, oracle, row, precision="fp32"):
    name, arch, kw = ROWS[row]
    return name, micro(K, oracle, arch, torch.device("cuda:0"), precision, **kw)


@pytest.mark.parametrize("row", list(ROWS))
def test_evaluate_equals_the_calls_by_hand(row, K, oracle):
    name, m = model_for(K, oracle, row)
    gts, lqs, keys, dataset = row_data(row)
    got = K.evaluate(m, name, gts, lqs, keys, dataset, niqe_params=NIQE)
    want = by_hand(K, m, row, gts, lqs, keys)
    assert list(got["scores"]) == list(want), (list(got["scores"]), list(want))
    for k, vs in want.items():
        w = torch.stack(vs).cpu()
        assert not w.isnan().any(), (k, w)
        same_bits(got["scores"][k], w)
        acc = 0
        for v in w.unbind(0):
            acc = acc + v
        assert got["means"][k] == float(acc / len(vs)), k


def test_evaluate_off_the_default_stream(K, oracle):
    name, m = model_for(K, oracle, "dn_c3", "fp16")
    gts, lqs, keys, dataset = row_data("dn_c3", seed=1)
    want = K.evaluate(m, name, gts, lqs, keys, dataset)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = K.evaluate(m, name, gts, lqs, keys, dataset)
    torch.cuda.current_stream().wait_stream(side)
    for k in want["scores"]:
        assert torch.equal(got["scores"][k], want["scores"][k]), k
    assert got["means"] == want["means"]


def test_evaluate_two_ranks_gather_to_the_single_process_means(K, oracle, monkeypatch):
    """Each rank of a two-process group restores its shard_range slice; the gathered per-image scores, put back in image
    order, give the single-process scores and means.  The group is simulated: each rank's local scores are recorded, and
    the gather returns both ranks' in rank order, as all_gather does."""
    from grl_image_restoration_b200 import evaluation, sharding

    name, m = model_for(K, oracle, "dm")
    g = torch.Generator().manual_seed(7)
    gts = [rand_u8(40 + 8 * (i % 3), 48 + 8 * (i % 2), 3, g) for i in range(5)]
    single = K.evaluate(m, name, gts)

    dist = torch.distributed
    local = {}
    monkeypatch.setattr(dist, "is_available", lambda: True)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    for rank in (0, 1):
        monkeypatch.setattr(dist, "get_rank", lambda group=None, r=rank: r)
        monkeypatch.setattr(sharding, "gather_metric", lambda v, i, group=None, r=rank: local.setdefault(r, []).append((v, i)) or (v, i))
        evaluation.evaluate(m, name, gts)
    lo, hi = sharding.shard_range(len(gts), 1, 2)
    assert local[1][0][1].tolist() == list(range(lo, hi))
    calls = iter(zip(local[0], local[1]))

    def gathered(v, i, group=None):
        (v0, i0), (v1, i1) = next(calls)
        return torch.cat([v0, v1]), torch.cat([i0, i1])

    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    monkeypatch.setattr(sharding, "gather_metric", gathered)
    split = evaluation.evaluate(m, name, gts)
    for k in single["scores"]:
        assert torch.equal(split["scores"][k], single["scores"][k]), k
    assert split["means"] == single["means"]


# ---- against the reference pipeline (oracle/make_golden_eval.py) ----------------------------------------------------------
with open(os.path.join(GOLD, "eval_pipeline.json")) as _f:
    PIPELINE = __import__("json").load(_f)
_PIPE = np.load(os.path.join(GOLD, "eval_pipeline.npz"))
# How far the package's metric kernels may sit from the reference's metric functions on the SAME bytes: the kernels sum
# the squared errors of the 8-bit integers exactly (float64 windows for SSIM), the reference in float32 tensor ops.
# float32 sums over n <= 2^16 terms carry a relative error below n * 2^-24 <= 2^-8 in the worst case, but torch's
# reductions are pairwise (relative error ~ log2(n) * 2^-24 < 2^-19), so the PSNR and PSNR-B error is below
# 10 / ln(10) * 2^-19 < 1e-5 dB; SSIM's float32 convolutions leave ~1e-6 on a value in [-1, 1].  IMPL allows 10x that.
IMPL = {"val_psnr": 1e-4, "val_psnr_y": 1e-4, "val_psnrb": 1e-4, "val_psnrb_y": 1e-4, "val_ssim": 1e-5,
        "val_ssim_y": 1e-5, "val_niqe": 1e-3}
TOL = {"val_psnr": 0.01, "val_psnr_y": 0.01, "val_psnrb": 0.01, "val_psnrb_y": 0.01, "val_ssim": 1e-4,
       "val_ssim_y": 1e-4, "val_niqe": 0.01}


@pytest.mark.parametrize("row", list(PIPELINE))
def test_fp32_scores_against_the_reference_pipeline(row, K, oracle):
    """evaluate on the fp32 path against the reference pipeline's per-image scores.

    The model inputs must equal the reference dataset's bit for bit (AWGN, JPEG, mosaic), so a recipe that crops,
    degrades or takes the luma at another step fails here.  The scores then differ from the reference's by
        score(ours) - ref(ref bytes) = [score(ours) - score(ref bytes)] + [score(ref bytes) - ref(ref bytes)],
    the first term from output bytes that the fp32 forward (max-abs ~1e-6 against the float64-free oracle) rounds to the
    other side of a half level, computed here exactly with the same metric kernel; the second the metric implementation
    difference, bounded by IMPL.  The test derives bound = |first| + IMPL, checks it is within the tolerance (0.01 dB
    for PSNR / PSNR-B, 1e-4 for SSIM) and that the scores are within the bound."""
    from grl_image_restoration_b200 import evaluation

    c = PIPELINE[row]
    name = c["name"]
    n = len(c["sizes"])
    arch_kw = {"input_format": "rggb"} if row == "dm" else {}
    m = micro(K, oracle, c["arch"], torch.device("cuda:0"), "fp32", **arch_kw)
    dev = lambda a: torch.from_numpy(a).cuda()  # noqa: E731
    gts = [dev(_PIPE[f"{row}/gt{i}"]) for i in range(n)]
    lqs = None
    if f"{row}/lqr0" in _PIPE.files:
        lqs = [(dev(_PIPE[f"{row}/lq{i}"]), dev(_PIPE[f"{row}/lqr{i}"])) for i in range(n)]
    elif f"{row}/lq0" in _PIPE.files:
        lqs = [dev(_PIPE[f"{row}/lq{i}"]) for i in range(n)]
    got = K.evaluate(m, name, gts, lqs, c["keys"], c["dataset"], niqe_params=NIQE)

    clean = evaluation.clean_images(name, gts, c["dataset"])
    inputs = evaluation.model_inputs(name, clean, lqs, c["keys"])
    for i in range(n):
        key = f"{row}/input{i}"
        if key in _PIPE.files:
            want = torch.from_numpy(_PIPE[key])
            x = inputs[i].cpu()
            if want.dtype == torch.uint8 and x.dtype == torch.float32:
                x = (x * 255).round().to(torch.uint8)
            elif x.dtype == torch.uint8:
                x = x.permute(2, 0, 1)
            assert torch.equal(x, want), (row, i, "model input differs from the reference dataset's")
    outs = evaluation.restore(m, name, inputs)
    for i in range(n):
        ref_bytes = dev(_PIPE[f"{row}/out{i}"])
        assert ref_bytes.shape == outs[i].shape, (row, i)
        d = (outs[i].int() - ref_bytes.int()).abs()
        assert int(d.max()) <= 1, (row, i, "an output byte is more than one level from the reference's")
        on_ref = evaluation.score(name, ref_bytes, clean[i], NIQE)
        for k in c["metrics"]:
            ours, ref = float(got["scores"][k][i]), float(_PIPE[f"{row}/{k}"][i])
            flips = abs(ours - float(on_ref[k]))
            impl = abs(float(on_ref[k]) - ref)
            bound = flips + IMPL[k]
            assert impl <= IMPL[k], (row, i, k, "metric kernel vs reference function", impl)
            assert bound <= TOL[k], (row, i, k, "derived bound above the tolerance", bound, int((d > 0).sum()))
            assert abs(ours - ref) <= bound, (row, i, k, ours, ref, bound)
