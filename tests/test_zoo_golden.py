"""The configs of the released checkpoints configs.grl_config gained last (blind x4 SR, single- and dual-pixel defocus
deblurring, grayscale denoising / JPEG) and the oracle against the UNMODIFIED reference's outputs for them
(tests/golden/zoo_*.npz, written by oracle/make_golden_zoo.py).  CPU only."""
import hashlib
import json
import math
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(GOLD, "zoo_cases.json")) as _f:
    ZOO = json.load(_f)["cases"]


def zoo_input(oracle, c):
    return oracle.synth_input((c["batch"], c["kwargs"]["in_channels"], *c["hw"]), seed=c["input_seed"],
                              noise_sigma=c["noise_sigma"])


@pytest.mark.parametrize("name", sorted(ZOO))
def test_oracle_reproduces_zoo_golden(oracle, name):
    """Bit for bit: the stored input, the sub-sampled output and the digest of the whole output."""
    c = ZOO[name]
    gold = np.load(os.path.join(GOLD, f"zoo_{name}.npz"))
    cfg = c["kwargs"]
    x = zoo_input(oracle, c)
    assert torch.equal(x, torch.from_numpy(gold["x"]))
    with torch.no_grad():
        y = oracle.grl_forward(oracle.synth_state_dict(cfg, seed=c["weight_seed"], style=c["style"]), cfg, x).contiguous()
    s = int(gold["stride"])
    assert list(y.shape) == gold["shape"].tolist() == c["out_shape"]
    err = (y[..., ::s, ::s] - torch.from_numpy(gold["sub"])).abs().max().item()
    print(f"{name}: out {tuple(y.shape)}, |oracle - reference| max {err}")
    assert err == 0.0
    assert hashlib.sha256(y.numpy().tobytes()).hexdigest() == str(np.asarray(gold["sha256"]))


@pytest.mark.parametrize("name", sorted(ZOO))
def test_zoo_config_builds_the_reference_parameters(pkg, name):
    """grl_config's kwargs give the module the reference's parameter names and shapes (the json records the reference
    network's own state_dict through param_summary: every name and shape via its digest), and the golden's kwargs are
    what grl_config returns today."""
    from make_golden_zoo import param_summary

    c = ZOO[name]
    a = dict(c["grl_config"])
    assert pkg.configs.grl_config(a.pop("variant"), a.pop("task"), a.pop("upscale"), a.pop("img_size"), **a) == c["kwargs"]
    m = pkg.GRL(**c["kwargs"])
    mine = {k: list(v.shape) for k, v in m.state_dict().items() if not k.startswith("table_")}
    assert param_summary(mine) == c["params"]


def test_released_table(pkg):
    """Every RELEASED entry builds with its own channel counts; the tile settings are the evaluation's."""
    C = pkg.configs
    assert len(C.RELEASED) == 24
    for name, (variant, task, upscale, cin, tile, overlap) in C.RELEASED.items():
        cfg = C.released_config(name)
        m = pkg.GRL(**dict(cfg, img_size=math.lcm(cfg["window_size"], *cfg["stripe_size"])))
        assert m.in_channels == cin and m.conv_first.weight.shape[1] == cin, name
        assert m.out_channels == (3 if task == "defocus_dual" else cin), name
        assert m.upscale == upscale and (tile, overlap) in ((0, 0), (256, 32), (288, 36), (480, 48)), name
    assert C.RELEASED["db_defocus_dual_pixel_grl_base.ckpt"] == ("base", "defocus_dual", 1, 6, 480, 48)
    assert C.RELEASED["bsr_grl_base.ckpt"] == ("base", "bsr", 4, 3, 0, 0)
    assert C.RELEASED["dn_grl_base_c1s15.ckpt"][4:] == (256, 32)
    assert C.RELEASED["jpeg_grl_small_c1q10.ckpt"] == ("small", "jpeg", 1, 1, 288, 36)


def test_new_tasks(pkg):
    g = pkg.configs.grl_config
    bsr = g("base", "bsr", 4, 128)
    assert (bsr["upsampler"], bsr["window_size"], bsr["stripe_size"], bsr["anchor_window_down_factor"],
            bsr["local_connection"]) == ("nearest+conv", 16, [32, 64], 4, True)
    d, dd = g("base", "defocus", 1, 480), g("base", "defocus_dual", 1, 480)
    assert (d["window_size"], d["stripe_size"], d["anchor_window_down_factor"], d["upsampler"]) == (16, [48, 96], 4, "")
    assert dd == dict(d, in_channels=6, out_channels=3)
    assert g("small", "dn", 1, in_channels=1) == dict(g("small", "dn", 1), in_channels=1)
    assert g("small", "jpeg", 1, in_channels=1)["in_channels"] == 1
    with pytest.raises(ValueError):
        g("small", "bsr")
    with pytest.raises(ValueError):
        g("base", "sr", 4, in_channels=1)
