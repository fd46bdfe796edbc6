"""The model-switch cases (anchor_proj_type / anchor_one_stage / conv_type) shared by test_switches.py and
test_gpu_switches.py, and the launch listing of the released configs that the switches must leave unchanged."""
import hashlib
import json
import os

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LISTING_SHAPE = (1, 64, 64)  # (batch, H, W) of the meta input the released listings are taken on


def switch_cases():
    with open(os.path.join(GOLD, "switches_cases.json")) as f:
        return json.load(f)


def released_listings(pkg):
    """{released checkpoint: sha256 of its fp32 launch list and of its fp16 tensor-core GEMM launch list} on a meta
    (1, Cin, 64, 64) input: every launch's name and arguments."""
    from grl_image_restoration_b200 import modules, tc

    out = {}
    for name in sorted(pkg.configs.RELEASED):
        cfg = pkg.configs.released_config(name, img_size=1152)
        m = pkg.GRL(**cfg)
        shape = (LISTING_SHAPE[0], cfg["in_channels"], *LISTING_SHAPE[1:])
        f32 = repr(modules.f32_launches(m, shape))
        m.set_precision("fp16")
        g = repr(tc.gemm_launches(m, shape))
        out[name] = {"f32": hashlib.sha256(f32.encode()).hexdigest(), "tc": hashlib.sha256(g.encode()).hexdigest()}
    return out


# ----------------------------------------------------------------------------------------------------------------------
# The restatement of a switched GRL forward: grl_oracle's attention, CAB, MLP and LayerNorm, composed with the anchor
# projection and stage conv of mixed_attn_block.py:679-785 and swin_v1_block.py:457-485.  oracle/make_golden_switches.py
# checks it against the reference.
# ----------------------------------------------------------------------------------------------------------------------
def anchor_projection(sd, pre, x, x_size, c):
    """AnchorProjection.forward (mixed_attn_block.py:772-785) for anchor_proj_type / anchor_one_stage of config c."""
    import torch
    import torch.nn.functional as F

    proj, df = c["anchor_proj_type"], c["anchor_window_down_factor"]
    B, L, C = x.shape
    t = x.transpose(1, 2).reshape(B, C, *x_size)
    if proj in ("avgpool", "maxpool"):
        t = (F.avg_pool2d if proj == "avgpool" else F.max_pool2d)(t, df, df).flatten(2).transpose(1, 2)
        t = F.linear(t, sd[pre + "body.0.reduction.weight"], sd[pre + "body.0.reduction.bias"])
        return t.reshape(B, x_size[0] // df, x_size[1] // df, -1)
    n = 1 if c["anchor_one_stage"] else int(torch.log2(torch.tensor(float(df))).item())
    for i in range(n):
        p = f"{pre}body.{i}."
        if proj == "conv2d":
            k, s, pad = (df + 1, df, (df + 1) // 2) if c["anchor_one_stage"] else (3, 2, 1)
            t = F.conv2d(t, sd[p + "weight"], sd[p + "bias"], stride=s, padding=pad)
        else:  # PatchMerging (mixed_attn_block.py:691-711)
            u = t.permute(0, 2, 3, 1)
            u = torch.cat([u[:, 0::2, 0::2], u[:, 1::2, 0::2], u[:, 0::2, 1::2], u[:, 1::2, 1::2]], -1)
            t = F.linear(u, sd[p + "reduction.weight"]).permute(0, 3, 1, 2)
    return t.permute(0, 2, 3, 1)


def last_conv(sd, pre, t, c):
    """build_last_conv's block (swin_v1_block.py:469-485) on (B, C, H, W)."""
    import torch.nn.functional as F

    ct = c["conv_type"]
    if ct == "1conv":
        return F.conv2d(t, sd[pre + "weight"], sd[pre + "bias"], padding=1)
    if ct == "1conv1x1":
        return F.conv2d(t, sd[pre + "weight"], sd[pre + "bias"])
    if ct == "linear":
        B, C, H, W = t.shape
        return F.linear(t.flatten(2).transpose(1, 2), sd[pre + "weight"], sd[pre + "bias"]).transpose(1, 2).reshape(B, -1, H, W)
    t = F.leaky_relu(F.conv2d(t, sd[pre + "0.weight"], sd[pre + "0.bias"], padding=1), 0.2)
    t = F.leaky_relu(F.conv2d(t, sd[pre + "2.weight"], sd[pre + "2.bias"]), 0.2)
    return F.conv2d(t, sd[pre + "4.weight"], sd[pre + "4.bias"], padding=1)


def mixed_attention(O, sd, pre, x, x_size, bc, t, c):
    """grl_oracle.mixed_attention with the switched anchor projection."""
    import torch
    import torch.nn.functional as F

    B, L, C = x.shape
    qkv = F.linear(x, sd[pre + "qkv.body.weight"], sd[pre + "qkv.body.bias"])
    qkv_w, qkv_s = torch.split(qkv, C * 3 // 2, dim=-1)
    anchor = anchor_projection(sd, pre + "anchor.", x, x_size, c)
    xw = O.window_attention(sd, pre + "window_attn.", qkv_w, x_size, bc["ws"], bc["heads_w"], bc["win_shift"],
                            t["table_w"], t["index_w"], t["mask_w"])
    xs = O.stripe_attention(sd, pre + "stripe_attn.", qkv_s, anchor, x_size, bc["stripe_size"], bc["stripe_groups"],
                            bc["stripe_shift"], bc["df"], bc["heads_s"], t["table_s"], t["index_a2w"], t["index_w2a"],
                            t["mask_a2w"], t["mask_w2a"])
    return F.linear(torch.cat([xw, xs], dim=-1), sd[pre + "proj.weight"], sd[pre + "proj.bias"])


def transformer_block(O, sd, pre, x, x_size, bc, tim, c):
    """grl_oracle.transformer_block with the switched anchor projection."""
    t = O.block_tables(tim, bc["stripe_type"], bc["win_shift"], bc["stripe_shift"])
    a = O.layer_norm(sd, pre + "norm1.", mixed_attention(O, sd, pre + "attn.", x, x_size, bc, t, c))
    if bc["local_connection"]:
        x = x + bc["res_scale"] * a + O.cab(sd, pre + "conv.", x, x_size)
    else:
        x = x + bc["res_scale"] * a
    return x + bc["res_scale"] * O.layer_norm(sd, pre + "norm2.", O.mlp(sd, pre + "mlp.", x))


def forward_features(O, sd, cfg, x):
    """grl_oracle.forward_features with the switched anchor projection and stage conv."""
    c = O.full_config(cfg)
    x_size = (x.shape[2], x.shape[3])
    t = O.layer_norm(sd, "norm_start.", x.flatten(2).transpose(1, 2))
    tim = O.table_index_mask(cfg, x_size)
    for s in range(len(c["depths"])):
        r = t
        for i in range(c["depths"][s]):
            r = transformer_block(O, sd, f"layers.{s}.blocks.{i}.", r, x_size, O.block_settings(cfg, s, i), tim, c)
        B, L, C = r.shape
        t = last_conv(sd, f"layers.{s}.conv.", r.transpose(1, 2).reshape(B, C, *x_size), c).flatten(2).transpose(1, 2) + t
    t = O.layer_norm(sd, "norm_end.", t)
    return t.transpose(1, 2).reshape(x.shape[0], -1, *x_size)


def grl_forward(O, sd, cfg, x):
    """grl_oracle.grl_forward with the switches of cfg, for a pixelshuffle x2 network (the micro configs the goldens
    run)."""
    import torch
    import torch.nn.functional as F

    c = O.full_config(cfg)
    assert c["upsampler"] == "pixelshuffle" and c["upscale"] == 2 and c["in_channels"] == 3
    conv = lambda n, t: F.conv2d(t, sd[n + ".weight"], sd[n + ".bias"], padding=1)
    H, W = x.shape[2:]
    p = O.pad_size(cfg)
    x = F.pad(x, (0, (p - W % p) % p, 0, (p - H % p) % p), "reflect")
    mean = torch.tensor((0.4488, 0.4371, 0.4040), dtype=x.dtype).view(1, 3, 1, 1)
    x = (x - mean) * c["img_range"]
    x = conv("conv_first", x)
    x = last_conv(sd, "conv_after_body.", forward_features(O, sd, cfg, x), c) + x
    x = F.leaky_relu(conv("conv_before_upsample.0", x), 0.01)
    x = conv("conv_last", F.pixel_shuffle(conv("upsample.up.0", x), 2))
    x = x / c["img_range"] + mean
    return x[:, :, : H * 2, : W * 2]


def synth_state_dict(O, cfg, shapes, seed=0):
    """grl_oracle.synth_state_dict's "routed" weights for the parameters it knows, and the same rules for the switched
    anchor and stage-conv parameters, whose names and shapes come from the reference (`shapes`): one generator per name;
    Conv2d weight and bias uniform in +-1/sqrt(fan_in) (PyTorch's default); Linear weight trunc_normal(0.02) and
    Linear bias 0.02 N(0, 1) from a second per-name generator, so a dropped or misplaced bias changes the output."""
    import zlib
    from math import prod

    import torch

    base = O.synth_state_dict(cfg, seed=seed, style="routed")
    sd = {}
    for name, shape in sorted(shapes.items()):
        shape = tuple(shape)
        if name in base and tuple(base[name].shape) == shape:
            sd[name] = base[name]
            continue
        g = torch.Generator().manual_seed((zlib.crc32(name.encode()) + 7919 * seed) % (2 ** 31))
        wname = name.rsplit(".", 1)[0] + ".weight"
        if len(shapes[wname]) == 4:
            fan_in = prod(shapes[wname][1:])
            sd[name] = ((torch.rand(shape, generator=g) * 2 - 1) / fan_in ** 0.5).float()
        elif name.endswith("bias"):
            r = torch.Generator().manual_seed((zlib.crc32(name.encode()) + 7919 * seed + 104729) % (2 ** 31))
            sd[name] = 0.02 * torch.randn(shape, generator=r)
        else:
            sd[name] = torch.nn.init.trunc_normal_(torch.empty(shape), std=0.02, generator=g).float()
    return sd
