"""The reference's nn.Module surface for the GRL forward path, re-implemented on the sm_90a kernels.

Class names, constructor signatures, parameter names/shapes (SURVEY.md Appendix C) and forward signatures
follow the reference so that `hydra.utils.instantiate(_target_=...GRL)`, `load_state_dict(strict=True)`,
`convert_checkpoint` and `self.model(x)` in the LightningIR engine keep working (engines/base.py:44,:106,:177;
tools/trainer.py:93-115).  Differences, all deliberate:
  * inference only (the engine's validation path runs under torch.no_grad()); no autograd support;
  * every forward runs hand-written CUDA through libgrl_b200.so - CPU tensors raise, there is no fallback;
  * relative-position indices and shift masks are closed forms inside the kernels, so the `index*` / `mask*`
    arguments are accepted but only their None-ness is used (mask None = unshifted block).
Reference files: models/networks/grl.py, models/common/mixed_attn_block_efficient.py,
models/common/mixed_attn_block.py, models/common/swin_v1_block.py, models/common/upsample.py.
"""
import inspect
import math
import os
from types import SimpleNamespace
from typing import NamedTuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import functional as K
from . import geometry as G
from . import image_list
from . import tc
from .geometry import to_2tuple, _get_stripe_info
from .streams import Produced, upload

_LN_MAX = math.log(1.0 / 0.01)


def _closed_form_marker(device=None):
    """Placeholder standing for an index / mask tensor that the kernels evaluate in closed form."""
    return torch.empty(0, device=device)


# The fp32 forward is written once, in the module forwards below, and issues every kernel through a launcher (tc.Device
# runs them, tc.Listing records the GEMMs and attention calls without a device: f32_launches).  Callers allocate every
# output, so a listing run on a meta input allocates meta tensors and launches nothing.  Modules that issue one listed
# launch take its full name ("stage0.block1.qkv"); the others take the prefix of their launches' names.
def linear(launch, name, x, lin, act=K.ACT_NONE):
    """nn.Linear `lin` on x (..., K) -> (..., N), launched as `name`."""
    y = torch.empty(*x.shape[:-1], lin.weight.shape[0], device=x.device, dtype=torch.float32)
    launch.listed(name, K.linear, x, lin.weight, lin.bias, act, out=y)
    return y


def conv3x3(launch, name, owner, key, x, act=K.ACT_NONE, slope=0.0, res=None):
    """nn.Conv2d(3x3, stride 1, pad 1) `owner.<key>` on channels-last x (B, H, W, Cin), launched as `name`.  Its
    (Cout, 9*Cin) im2col-ordered weight is cached on the owner under `key` (a streams.Produced) and re-packed when the
    weight changes."""
    conv = owner.get_submodule(key)
    w = conv.weight
    version = (w.data_ptr(), w._version, w.device)
    cache = owner.__dict__.setdefault("_f32_convs", {})
    if cache.get(key, (None,))[0] != version:
        cache[key] = (version, Produced(K.pack_conv_weight(w)))
    y = torch.empty(*x.shape[:-1], w.shape[0], device=x.device, dtype=torch.float32)
    launch.listed(name, K.conv3x3, x, cache[key][1].use(), conv.bias, act, slope, res, out=y)
    return y


def ln_residual(launch, norm, u, x=None, res_scale=1.0, cab_y=None, cab_gate=None):
    """(x or 0) + res_scale * norm(u) (+ cab_y * cab_gate[b]) for u (B, L, C)."""
    out = torch.empty(u.shape, device=u.device, dtype=torch.float32)
    launch.run(K.ln_residual, x, u, norm.weight, norm.bias, norm.eps, res_scale, cab_y, cab_gate, out=out)
    return out


def pixel_shuffle_cl(x, r):
    """nn.PixelShuffle(r) on channels-last data: (B, H, W, C*r*r) -> (B, H*r, W*r, C)."""
    B, H, W, Crr = x.shape
    C = Crr // (r * r)
    return x.view(B, H, W, C, r, r).permute(0, 1, 4, 2, 5, 3).reshape(B, H * r, W * r, C)


# ----------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------
class CPB_MLP(nn.Sequential):
    """mixed_attn_block.py:24-31."""

    def __init__(self, in_channels, out_channels, channels=512):
        super().__init__(nn.Linear(in_channels, channels, bias=True), nn.ReLU(inplace=True),
                         nn.Linear(channels, out_channels, bias=False))


class AffineTransform(nn.Module):
    """mixed_attn_block_efficient.py:23-58: learned per-head logit scale + continuous position bias (+ mask)."""

    def __init__(self, num_heads):
        super().__init__()
        self.logit_scale = nn.Parameter(torch.log(10 * torch.ones((num_heads, 1, 1))), requires_grad=True)
        self.cpb_mlp = CPB_MLP(2, num_heads)

    def bias_table(self, relative_coords_table, launch=tc.DEVICE):
        """(heads, rows) = 16*sigmoid(cpb_mlp(table)) -- what the fused attention kernels consume."""
        out = torch.empty(self.cpb_mlp[2].weight.shape[0], relative_coords_table.numel() // 2,
                          device=relative_coords_table.device, dtype=torch.float32)
        launch.run(K.bias_table, relative_coords_table, self.cpb_mlp[0].weight, self.cpb_mlp[0].bias,
                   self.cpb_mlp[2].weight, out=out)
        return out

    @torch.no_grad()
    def forward(self, attn, relative_coords_table, relative_position_index, mask):
        bias = self.bias_table(relative_coords_table)
        return K.affine_(attn.clone(), self.logit_scale, bias, relative_position_index, mask)


class WindowAttention(nn.Module):
    """mixed_attn_block_efficient.py:97-171.  qkv is the input of forward."""

    def __init__(self, input_resolution, window_size, num_heads, window_shift=False, attn_drop=0.0,
                 pretrained_window_size=[0, 0], args=None):
        super().__init__()
        self.input_resolution = input_resolution
        self.window_size = to_2tuple(window_size)
        self.pretrained_window_size = pretrained_window_size
        self.num_heads = num_heads
        self.shift_size = self.window_size[0] // 2 if window_shift else 0
        self.euclidean_dist = bool(getattr(args, "euclidean_dist", False))
        if self.euclidean_dist:
            raise NotImplementedError("euclidean_dist is an ablation outside the hot path")
        self.attn_transform = AffineTransform(num_heads)
        self.attn_drop = nn.Dropout(attn_drop)
        self.softmax = nn.Softmax(dim=-1)

    @torch.no_grad()
    def forward(self, qkv, x_size, table, index, mask, out=None, launch=tc.DEVICE, name="window_attn"):
        """qkv (B, L, 3c) -> (B, L, c).  `index` is unused (closed form); `mask is not None` enables the shift mask."""
        B, L, C = qkv.shape
        s = self.shift_size
        grid = G.token_grid(x_size, self.window_size, (s, s))
        bias = self.attn_transform.bias_table(table, launch)
        out = torch.empty(B, L, C // 3, device=qkv.device, dtype=torch.float32) if out is None else out
        launch.listed(name, K.window_attention, qkv, B, grid, self.num_heads, self.attn_transform.logit_scale, bias,
                      mask is not None, out)
        return out

    def extra_repr(self):
        return (f"window_size={self.window_size}, shift_size={self.shift_size}, "
                f"pretrained_window_size={self.pretrained_window_size}, num_heads={self.num_heads}")


class AnchorStripeAttention(nn.Module):
    """mixed_attn_block_efficient.py:177-276."""

    def __init__(self, input_resolution, stripe_size, stripe_groups, stripe_shift, num_heads, attn_drop=0.0,
                 pretrained_stripe_size=[0, 0], anchor_window_down_factor=1, args=None):
        super().__init__()
        self.input_resolution = input_resolution
        self.stripe_size = stripe_size
        self.stripe_groups = stripe_groups
        self.stripe_shift = stripe_shift
        self.num_heads = num_heads
        self.pretrained_stripe_size = pretrained_stripe_size
        self.anchor_window_down_factor = anchor_window_down_factor
        self.euclidean_dist = bool(getattr(args, "euclidean_dist", False))
        if self.euclidean_dist:
            raise NotImplementedError("euclidean_dist is an ablation outside the hot path")
        self.attn_transform1 = AffineTransform(num_heads)
        self.attn_transform2 = AffineTransform(num_heads)
        self.attn_drop = nn.Dropout(attn_drop)
        self.softmax = nn.Softmax(dim=-1)

    def grids(self, x_size):
        ss, sh = _get_stripe_info(self.stripe_size, self.stripe_groups, self.stripe_shift, x_size)
        if not self.stripe_shift:  # with stripe_groups the info carries a shift even for unshifted blocks, but
            sh = [0, 0]            # the roll itself is guarded by stripe_shift (efficient.py:235)
        df = self.anchor_window_down_factor
        return G.token_grid(x_size, ss, sh), G.anchor_grid(x_size, ss, sh, df)

    @torch.no_grad()
    def forward(self, qkv, anchor, x_size, table, index_a2w, index_w2a, mask_a2w, mask_w2a, out=None, launch=tc.DEVICE,
                name="stripe_attn"):
        B, L, C = qkv.shape
        tok, anc = self.grids(x_size)
        b1 = self.attn_transform1.bias_table(table, launch)
        b2 = self.attn_transform2.bias_table(table, launch)
        out = torch.empty(B, L, C // 3, device=qkv.device, dtype=torch.float32) if out is None else out
        launch.listed(name, K.stripe_attention, qkv, anchor, B, tok, anc, self.num_heads,
                      self.attn_transform1.logit_scale, b1, self.attn_transform2.logit_scale, b2, mask_a2w is not None,
                      out)
        return out

    def extra_repr(self):
        return (f"stripe_size={self.stripe_size}, stripe_groups={self.stripe_groups}, stripe_shift={self.stripe_shift}, "
                f"pretrained_stripe_size={self.pretrained_stripe_size}, num_heads={self.num_heads}, "
                f"anchor_window_down_factor={self.anchor_window_down_factor}")


class QKVProjection(nn.Module):
    """mixed_attn_block.py:661-676 (proj_type 'linear' -- the only one any released config uses)."""

    def __init__(self, dim, qkv_bias, proj_type, args):
        super().__init__()
        if proj_type != "linear":
            raise NotImplementedError(f"qkv_proj_type={proj_type!r}: only 'linear' is on the hot path")
        self.proj_type = proj_type
        self.body = nn.Linear(dim, dim * 3, bias=qkv_bias)

    @torch.no_grad()
    def forward(self, x, x_size, launch=tc.DEVICE, name="qkv"):
        return linear(launch, name, x, self.body)


class AnchorLinear(nn.Module):
    """mixed_attn_block.py:714-736: AvgPool2d(df) then Linear(C -> C/2); returns (B, H/df, W/df, C/2)."""

    def __init__(self, in_channels, out_channels, down_factor, pooling_mode, bias):
        super().__init__()
        if pooling_mode != "avgpool":
            raise NotImplementedError(f"anchor pooling {pooling_mode!r}: only 'avgpool' is on the hot path")
        self.down_factor = down_factor
        self.pooling = nn.AvgPool2d(down_factor, down_factor)
        self.reduction = nn.Linear(in_channels, out_channels, bias=bias)

    @torch.no_grad()
    def forward(self, x, x_size, launch=tc.DEVICE, name="anchor"):
        B, L, C = x.shape
        df = self.down_factor
        pooled = torch.empty(B, x_size[0] // df, x_size[1] // df, C, device=x.device, dtype=torch.float32)
        launch.run(K.avgpool, x.view(B, x_size[0], x_size[1], C), df, out=pooled)
        return linear(launch, name, pooled, self.reduction)


class AnchorProjection(nn.Module):
    """mixed_attn_block.py:739-785 (one-stage avgpool variant)."""

    def __init__(self, dim, proj_type, one_stage, anchor_window_down_factor, args):
        super().__init__()
        if not one_stage or proj_type.find("pool") < 0:
            raise NotImplementedError("only the one-stage avgpool anchor projection is on the hot path")
        self.proj_type = proj_type
        self.body = nn.ModuleList([AnchorLinear(dim, dim // 2, anchor_window_down_factor, proj_type, True)])

    def forward(self, x, x_size, launch=tc.DEVICE, name="anchor"):
        for m in self.body:
            x = m(x, x_size, launch, name)
        return x


class MixedAttention(nn.Module):
    """mixed_attn_block_efficient.py:282-403: shared QKV / anchor projections, window + stripe attention, proj."""

    def __init__(self, dim, input_resolution, num_heads_w, num_heads_s, window_size, window_shift, stripe_size,
                 stripe_groups, stripe_shift, qkv_bias=True, qkv_proj_type="linear", anchor_proj_type="separable_conv",
                 anchor_one_stage=True, anchor_window_down_factor=1, attn_drop=0.0, proj_drop=0.0,
                 pretrained_window_size=[0, 0], pretrained_stripe_size=[0, 0], args=None):
        super().__init__()
        self.dim = dim
        self.input_resolution = input_resolution
        self.args = args
        self.qkv = QKVProjection(dim, qkv_bias, qkv_proj_type, args)
        self.anchor = AnchorProjection(dim, anchor_proj_type, anchor_one_stage, anchor_window_down_factor, args)
        self.window_attn = WindowAttention(input_resolution, window_size, num_heads_w, window_shift, attn_drop,
                                           pretrained_window_size, args)
        self.stripe_attn = AnchorStripeAttention(input_resolution, stripe_size, stripe_groups, stripe_shift,
                                                 num_heads_s, attn_drop, pretrained_stripe_size,
                                                 anchor_window_down_factor, args)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)

    @torch.no_grad()
    def forward(self, x, x_size, table_index_mask, launch=tc.DEVICE, name=""):
        B, L, C = x.shape
        qkv = self.qkv(x, x_size, launch, f"{name}.qkv")
        qkv_window, qkv_stripe = torch.split(qkv, C * 3 // 2, dim=-1)
        anchor = self.anchor(x, x_size, launch, f"{name}.anchor")
        merged = torch.empty(B, L, C, device=x.device, dtype=torch.float32)  # cat([window, stripe]) without the copy
        t = table_index_mask
        self.window_attn(qkv_window, x_size, t["table_w"], t["index_w"], t["mask_w"], merged[..., : C // 2], launch,
                         f"{name}.window_attn")
        self.stripe_attn(qkv_stripe, anchor, x_size, t["table_s"], t["index_a2w"], t["index_w2a"], t["mask_a2w"],
                         t["mask_w2a"], merged[..., C // 2:], launch, f"{name}.stripe_attn")
        return linear(launch, f"{name}.proj", merged, self.proj)

    def extra_repr(self):
        return f"dim={self.dim}, input_resolution={self.input_resolution}"


# ----------------------------------------------------------------------------------------------
# conv / channel-attention block, MLP
# ----------------------------------------------------------------------------------------------
class ChannelAttention(nn.Module):
    """mixed_attn_block.py:948-967."""

    def __init__(self, num_feat, reduction=16):
        super().__init__()
        self.attention = nn.Sequential(nn.AdaptiveAvgPool2d(1), nn.Conv2d(num_feat, num_feat // reduction, 1, padding=0),
                                       nn.ReLU(inplace=True), nn.Conv2d(num_feat // reduction, num_feat, 1, padding=0),
                                       nn.Sigmoid())

    @torch.no_grad()
    def gate(self, y, launch=tc.DEVICE):
        """y (B, L, C) channels-last -> (B, C) sigmoid gate."""
        a1, a3 = self.attention[1], self.attention[3]
        gate = torch.empty(y.shape[0], y.shape[2], device=y.device, dtype=torch.float32)
        launch.run(K.channel_gate, y, a1.weight.view(a1.weight.shape[0], -1), a1.bias,
                   a3.weight.view(a3.weight.shape[0], -1), a3.bias, out=gate)
        return gate

    @torch.no_grad()
    def forward(self, x):
        """x (B, C, H, W) like the reference."""
        B, C, H, W = x.shape
        y = x.permute(0, 2, 3, 1).reshape(B, H * W, C).contiguous()
        return x * self.gate(y).view(B, C, 1, 1)


class CAB(nn.Module):
    """mixed_attn_block.py:970-983: conv3x3(C->C/4) GELU conv3x3(C/4->C) ChannelAttention, on (B, L, C)."""

    def __init__(self, num_feat, compress_ratio=4, reduction=18):
        super().__init__()
        self.cab = nn.Sequential(nn.Conv2d(num_feat, num_feat // compress_ratio, 3, 1, 1), nn.GELU(),
                                 nn.Conv2d(num_feat // compress_ratio, num_feat, 3, 1, 1),
                                 ChannelAttention(num_feat, reduction))

    @torch.no_grad()
    def features_and_gate(self, x, x_size, launch=tc.DEVICE, name=""):
        """Returns (y, gate): y (B, L, C) = conv2(gelu(conv1(x))), gate (B, C); CAB(x) = y * gate."""
        B, L, C = x.shape
        t = conv3x3(launch, f"{name}.cab1", self, "cab.0", x.view(B, x_size[0], x_size[1], C), K.ACT_GELU)
        y = conv3x3(launch, f"{name}.cab2", self, "cab.2", t).view(B, L, C)
        return y, self.cab[3].gate(y, launch)

    @torch.no_grad()
    def forward(self, x, x_size):
        y, g = self.features_and_gate(x, x_size)
        return y * g.unsqueeze(1)


class Mlp(nn.Module):
    """swin_v1_block.py:15-43 (GELU is the exact erf form)."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        if act_layer is not nn.GELU:
            raise NotImplementedError("only nn.GELU is on the hot path")
        drop_probs = to_2tuple(drop)
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.drop1 = nn.Dropout(drop_probs[0])
        self.fc2 = nn.Linear(hidden_features, out_features)
        self.drop2 = nn.Dropout(drop_probs[1])

    @torch.no_grad()
    def forward(self, x, launch=tc.DEVICE, name=""):
        return linear(launch, f"{name}.fc2", linear(launch, f"{name}.fc1", x, self.fc1, K.ACT_GELU), self.fc2)


class EfficientMixAttnTransformerBlock(nn.Module):
    """mixed_attn_block_efficient.py:406-564: post-norm residual block
    x = x + rs*LN1(attn(x)) [+ CAB(x)];  x = x + rs*LN2(mlp(x))."""

    def __init__(self, dim, input_resolution, num_heads_w, num_heads_s, window_size=7, window_shift=False,
                 stripe_size=[8, 8], stripe_groups=[None, None], stripe_shift=False, stripe_type="H", mlp_ratio=4.0,
                 qkv_bias=True, qkv_proj_type="linear", anchor_proj_type="separable_conv", anchor_one_stage=True,
                 anchor_window_down_factor=1, drop=0.0, attn_drop=0.0, drop_path=0.0, act_layer=nn.GELU,
                 norm_layer=nn.LayerNorm, pretrained_window_size=[0, 0], pretrained_stripe_size=[0, 0], res_scale=1.0,
                 args=None):
        super().__init__()
        self.dim = dim
        self.input_resolution = input_resolution
        self.num_heads_w = num_heads_w
        self.num_heads_s = num_heads_s
        self.window_size = window_size
        self.window_shift = window_shift
        self.stripe_shift = stripe_shift
        self.stripe_type = stripe_type
        self.args = args
        if self.stripe_type == "W":
            self.stripe_size = stripe_size[::-1]
            self.stripe_groups = stripe_groups[::-1]
        else:
            self.stripe_size = stripe_size
            self.stripe_groups = stripe_groups
        self.mlp_ratio = mlp_ratio
        self.res_scale = res_scale
        if norm_layer is not nn.LayerNorm:
            raise NotImplementedError("only nn.LayerNorm is on the hot path")
        self.attn = MixedAttention(dim, input_resolution, num_heads_w, num_heads_s, window_size, window_shift,
                                   self.stripe_size, self.stripe_groups, stripe_shift, qkv_bias, qkv_proj_type,
                                   anchor_proj_type, anchor_one_stage, anchor_window_down_factor, attn_drop, drop,
                                   pretrained_window_size, pretrained_stripe_size, args)
        self.norm1 = norm_layer(dim)
        if self.args.local_connection:
            self.conv = CAB(dim)
        self.drop_path = nn.Identity()  # stochastic depth is the identity at inference (timm DropPath in eval)
        self.mlp = Mlp(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer, drop=drop)
        self.norm2 = norm_layer(dim)

    def _get_table_index_mask(self, all_table_index_mask):
        """mixed_attn_block_efficient.py:510-537."""
        a = all_table_index_mask
        d = "sv" if self.stripe_type == "W" else "sh"
        return {
            "table_w": a["table_w"], "index_w": a["index_w"],
            "table_s": a["table_" + d], "index_a2w": a[f"index_{d}_a2w"], "index_w2a": a[f"index_{d}_w2a"],
            "mask_w": a["mask_w"] if self.window_shift else None,
            "mask_a2w": a[f"mask_{d}_a2w"] if self.stripe_shift else None,
            "mask_w2a": a[f"mask_{d}_w2a"] if self.stripe_shift else None,
        }

    precision = "fp32"  # "fp32": exact-parity SIMT kernels; "fp16" / "bf16": fused wgmma path (tc.py)

    @torch.no_grad()
    def forward_tc(self, x32, x16, x_size, all_table_index_mask):
        """Tensor-core path with the residual stream as an explicit PAIR: x32 fp32 (B, L, C) and its 16-bit operand copy
        x16 (B, L, Cpad) (None: packed here).  Returns the pair of the block's output, so a stage / network chains
        blocks without re-packing and without hiding state on tensors."""
        K.capi.require_device(x32)
        return tc.block_plan(self, tc.FMT[self.precision]).run(self, x32, x16, x_size, all_table_index_mask)

    @torch.no_grad()
    def forward(self, x, x_size, all_table_index_mask, launch=tc.DEVICE, name=""):
        if self.precision != "fp32":
            return self.forward_tc(x, None, x_size, all_table_index_mask)[0]
        t = self._get_table_index_mask(all_table_index_mask)
        u = self.attn(x, x_size, t, launch, name)
        y = gate = None
        if self.args.local_connection:
            y, gate = self.conv.features_and_gate(x, x_size, launch, name)
        x = ln_residual(launch, self.norm1, u, x, self.res_scale, y, gate)
        return ln_residual(launch, self.norm2, self.mlp(x, launch, name), x, self.res_scale)

    def extra_repr(self):
        return (f"dim={self.dim}, input_resolution={self.input_resolution}, num_heads=({self.num_heads_w}, "
                f"{self.num_heads_s}), window_size={self.window_size}, window_shift={self.window_shift}, "
                f"stripe_size={self.stripe_size}, stripe_groups={self.stripe_groups}, stripe_shift={self.stripe_shift}, "
                f"self.stripe_type={self.stripe_type}, mlp_ratio={self.mlp_ratio}, res_scale={self.res_scale}")


def build_last_conv(conv_type, dim):
    """swin_v1_block.py:469-485 ('1conv' is what every GRL config uses)."""
    if conv_type != "1conv":
        raise NotImplementedError(f"conv_type={conv_type!r}: only '1conv' is on the hot path")
    return nn.Conv2d(dim, dim, 3, 1, 1)


class Upsample(nn.Module):
    """upsample.py:6-30."""

    def __init__(self, scale, num_feat):
        super().__init__()
        m = []
        if (scale & (scale - 1)) == 0:
            for _ in range(int(math.log(scale, 2))):
                m += [nn.Conv2d(num_feat, 4 * num_feat, 3, 1, 1), nn.PixelShuffle(2)]
        elif scale == 3:
            m += [nn.Conv2d(num_feat, 9 * num_feat, 3, 1, 1), nn.PixelShuffle(3)]
        else:
            raise ValueError(f"scale {scale} is not supported. Supported scales: 2^n and 3.")
        self.up = nn.Sequential(*m)

    @torch.no_grad()
    def forward_cl(self, x, launch=tc.DEVICE, name="upsample"):
        """Channels-last (B, H, W, C) in and out."""
        for i, m in enumerate(self.up):
            if isinstance(m, nn.Conv2d):
                x = conv3x3(launch, f"{name}.up.{i}", self, f"up.{i}", x)
            else:
                x = pixel_shuffle_cl(x, m.upscale_factor)
        return x

    def forward(self, x):
        return self.forward_cl(x.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2)


class UpsampleOneStep(nn.Module):
    """upsample.py:33-50."""

    def __init__(self, scale, num_feat, num_out_ch):
        super().__init__()
        self.num_feat = num_feat
        self.up = nn.Sequential(nn.Conv2d(num_feat, (scale ** 2) * num_out_ch, 3, 1, 1), nn.PixelShuffle(scale))

    @torch.no_grad()
    def forward_cl(self, x, launch=tc.DEVICE, name="upsample"):
        """Channels-last (B, H, W, C) in and out."""
        return pixel_shuffle_cl(conv3x3(launch, f"{name}.up.0", self, "up.0", x), self.up[1].upscale_factor)

    def forward(self, x):
        return self.forward_cl(x.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2)


# ----------------------------------------------------------------------------------------------
# stage / network
# ----------------------------------------------------------------------------------------------
class TransformerStage(nn.Module):
    """models/networks/grl.py:31-173: `depth` blocks, then conv3x3 + residual."""

    def __init__(self, dim, input_resolution, depth, num_heads_window, num_heads_stripe, window_size, stripe_size,
                 stripe_groups, stripe_shift, mlp_ratio=4.0, qkv_bias=True, qkv_proj_type="linear",
                 anchor_proj_type="avgpool", anchor_one_stage=True, anchor_window_down_factor=1, drop=0.0,
                 attn_drop=0.0, drop_path=0.0, norm_layer=nn.LayerNorm, pretrained_window_size=[0, 0],
                 pretrained_stripe_size=[0, 0], conv_type="1conv", init_method="", fairscale_checkpoint=False,
                 offload_to_cpu=False, args=None):
        super().__init__()
        self.dim = dim
        self.input_resolution = input_resolution
        self.init_method = init_method
        self.blocks = nn.ModuleList()
        for i in range(depth):
            self.blocks.append(EfficientMixAttnTransformerBlock(
                dim=dim, input_resolution=input_resolution, num_heads_w=num_heads_window, num_heads_s=num_heads_stripe,
                window_size=window_size, window_shift=i % 2 == 0, stripe_size=stripe_size, stripe_groups=stripe_groups,
                stripe_type="H" if i % 2 == 0 else "W", stripe_shift=i % 4 in [2, 3] if stripe_shift else False,
                mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, qkv_proj_type=qkv_proj_type, anchor_proj_type=anchor_proj_type,
                anchor_one_stage=anchor_one_stage, anchor_window_down_factor=anchor_window_down_factor, drop=drop,
                attn_drop=attn_drop, drop_path=drop_path[i] if isinstance(drop_path, list) else drop_path,
                norm_layer=norm_layer, pretrained_window_size=pretrained_window_size,
                pretrained_stripe_size=pretrained_stripe_size, res_scale=0.1 if init_method == "r" else 1.0, args=args))
            # fairscale_checkpoint / offload_to_cpu: activation checkpointing is a no-op for inference (grl.py:133)
        self.conv = build_last_conv(conv_type, dim)

    def _init_weights(self):
        """grl.py:138-162."""
        for n, m in self.named_modules():
            if self.init_method == "w":
                if isinstance(m, (nn.Linear, nn.Conv2d)) and n.find("cpb_mlp") < 0:
                    m.weight.data *= 0.1
            elif self.init_method == "l":
                if isinstance(m, nn.LayerNorm):
                    nn.init.constant_(m.bias, 0)
                    nn.init.constant_(m.weight, 0)
            elif self.init_method.find("t") >= 0:
                scale = 0.1 ** (len(self.init_method) - 1) * int(self.init_method[-1])
                if isinstance(m, nn.Linear) and n.find("cpb_mlp") < 0:
                    nn.init.trunc_normal_(m.weight, std=scale)
                elif isinstance(m, nn.Conv2d):
                    m.weight.data *= 0.1
            else:
                raise NotImplementedError(f"Parameter initialization method {self.init_method} not implemented in TransformerStage.")

    @torch.no_grad()
    def forward_tc(self, x32, x16, x_size, table_index_mask):
        """Tensor-core path of the stage on the explicit (fp32 stream, 16-bit operand copy) pair; returns the pair."""
        K.capi.require_device(x32)
        return tc.stage_forward(self, x32, x16, x_size, table_index_mask)

    @torch.no_grad()
    def forward(self, x, x_size, table_index_mask, launch=tc.DEVICE, name=""):
        if len(self.blocks) and self.blocks[0].precision != "fp32":
            return self.forward_tc(x, None, x_size, table_index_mask)[0]
        res = x
        for bi, blk in enumerate(self.blocks):
            res = blk(res, x_size, table_index_mask, launch, f"{name}.block{bi}")
        B, L, C = x.shape
        H, W = x_size
        return conv3x3(launch, f"{name}.conv", self, "conv", res.view(B, H, W, C), res=x.view(B, H, W, C)).view(B, L, C)


class GRL(nn.Module):
    """models/networks/grl.py:176-569.  Same constructor kwargs (plus **kwargs swallowing the extra yaml keys),
    parameter names and call contract as the reference network."""

    def __init__(self, img_size=64, in_channels=3, out_channels=None, embed_dim=96, upscale=2, img_range=1.0,
                 upsampler="", depths=[6, 6, 6, 6, 6, 6], num_heads_window=[3, 3, 3, 3, 3, 3],
                 num_heads_stripe=[3, 3, 3, 3, 3, 3], window_size=8, stripe_size=[8, 8], stripe_groups=[None, None],
                 stripe_shift=False, mlp_ratio=4.0, qkv_bias=True, qkv_proj_type="linear", anchor_proj_type="avgpool",
                 anchor_one_stage=True, anchor_window_down_factor=1, out_proj_type="linear", local_connection=False,
                 drop_rate=0.0, attn_drop_rate=0.0, drop_path_rate=0.1, norm_layer=nn.LayerNorm,
                 pretrained_window_size=[0, 0], pretrained_stripe_size=[0, 0], conv_type="1conv", init_method="n",
                 fairscale_checkpoint=False, offload_to_cpu=False, euclidean_dist=False, self_ensemble=False,
                 input_format="rgb", **kwargs):
        super().__init__()
        # x8 geometric self-ensemble in forward (off: the reference's forward).  Views are forwarded in chunks of at most
        # ensemble_max_batch images, which bounds the activation memory of the 8x larger batch.
        self.self_ensemble = bool(self_ensemble)
        self.ensemble_max_batch = 16
        # forward_list runs the images of one padded size in forwards of at most max_batch_tokens padded pixels each
        # (default: bench.py's per-GPU batch, 16 images of 256 x 256), which bounds the activation memory of a list
        self.max_batch_tokens = 16 * 256 * 256
        # "rggb": forward takes the dm task's packed RGGB Bayer planes (B, 4, h, w) and demosaics them on the device with
        # the reference engine's dm_matlab (engines/base.py:127-128) before the network; "rgb" (default): the reference's
        # forward.  Feed "rggb" only data that the caller has not demosaiced already.
        if input_format not in ("rgb", "rggb"):
            raise ValueError(f"input_format must be 'rgb' or 'rggb', got {input_format!r}")
        if input_format == "rggb" and in_channels != 3:
            raise ValueError(f"input_format='rggb' demosaics to 3 channels, but in_channels={in_channels}")
        self.input_format = input_format
        self._requested_precision = kwargs.pop("precision", None) or os.environ.get("GRL_B200_PRECISION", "fp32")
        out_channels = out_channels or in_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        num_out_feats = 64
        self.embed_dim, self.upscale, self.upsampler, self.img_range = embed_dim, upscale, upsampler, img_range
        if in_channels == 3:
            self.mean = torch.Tensor((0.4488, 0.4371, 0.4040)).view(1, 3, 1, 1)
        else:
            self.mean = torch.zeros(1, 1, 1, 1)
        stripe_size, stripe_groups = list(stripe_size), list(stripe_groups)
        max_stripe_size = max([0 if s is None else s for s in stripe_size])
        max_stripe_groups = max([0 if s is None else s for s in stripe_groups]) * anchor_window_down_factor
        self.pad_size = max(window_size, max_stripe_size, max_stripe_groups)
        self.input_resolution = to_2tuple(img_size)
        self.window_size = to_2tuple(window_size)
        self.shift_size = [w // 2 for w in self.window_size]
        self.stripe_size, self.stripe_groups = stripe_size, stripe_groups
        self.pretrained_window_size, self.pretrained_stripe_size = pretrained_window_size, pretrained_stripe_size
        self.anchor_window_down_factor = anchor_window_down_factor
        if out_proj_type != "linear":
            raise NotImplementedError("only out_proj_type='linear' is on the hot path")
        if any(int(v) != 0 for v in list(pretrained_window_size) + list(pretrained_stripe_size)):
            # ops.get_relative_coords_table_all divides by the pretrained size when it is > 0 (ops.py:225-271); no released
            # config sets it, and the closed-form tables here always normalise by the current size
            raise NotImplementedError("pretrained_window_size / pretrained_stripe_size != 0 are not on the hot path")

        self.conv_first = nn.Conv2d(in_channels, embed_dim, 3, 1, 1)
        self.norm_start = norm_layer(embed_dim)
        self.pos_drop = nn.Dropout(p=drop_rate)
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, sum(depths))]
        args = SimpleNamespace(out_proj_type=out_proj_type, local_connection=local_connection,
                               euclidean_dist=euclidean_dist)
        # Only the three coordinate tables are buffers (a few KB).  The reference also registers ~1.5 GB of int64
        # indices and fp32 masks (grl.py:309-310); here those are closed forms inside the kernels.  The constructor
        # still validates img_size like the reference does (ops.py:46 view error, SURVEY.md D.1).
        ss, _ = _get_stripe_info(self.stripe_size, self.stripe_groups, True, self.input_resolution)
        for s, d in zip(list(ss) + list(self.window_size), list(self.input_resolution) * 2):
            if s <= 0 or d % s != 0:
                raise RuntimeError(f"img_size {self.input_resolution} is not a multiple of the window/stripe size {s}")
        for k, v in self._tables(self.input_resolution).items():
            self.register_buffer(k, v)

        self.layers = nn.ModuleList()
        for i in range(len(depths)):
            self.layers.append(TransformerStage(
                dim=embed_dim, input_resolution=self.input_resolution, depth=depths[i],
                num_heads_window=num_heads_window[i], num_heads_stripe=num_heads_stripe[i],
                window_size=self.window_size, stripe_size=stripe_size, stripe_groups=stripe_groups,
                stripe_shift=stripe_shift, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, qkv_proj_type=qkv_proj_type,
                anchor_proj_type=anchor_proj_type, anchor_one_stage=anchor_one_stage,
                anchor_window_down_factor=anchor_window_down_factor, drop=drop_rate, attn_drop=attn_drop_rate,
                drop_path=dpr[sum(depths[:i]): sum(depths[: i + 1])], norm_layer=norm_layer,
                pretrained_window_size=pretrained_window_size, pretrained_stripe_size=pretrained_stripe_size,
                conv_type=conv_type, init_method=init_method, fairscale_checkpoint=fairscale_checkpoint,
                offload_to_cpu=offload_to_cpu, args=args))
        self.norm_end = norm_layer(embed_dim)
        self.conv_after_body = build_last_conv(conv_type, embed_dim)

        if self.upsampler == "pixelshuffle":
            self.conv_before_upsample = nn.Sequential(nn.Conv2d(embed_dim, num_out_feats, 3, 1, 1),
                                                      nn.LeakyReLU(inplace=True))
            self.upsample = Upsample(upscale, num_out_feats)
            self.conv_last = nn.Conv2d(num_out_feats, out_channels, 3, 1, 1)
        elif self.upsampler == "pixelshuffledirect":
            self.upsample = UpsampleOneStep(upscale, embed_dim, out_channels)
        elif self.upsampler == "nearest+conv":
            assert self.upscale == 4, "only support x4 now."
            self.conv_before_upsample = nn.Sequential(nn.Conv2d(embed_dim, num_out_feats, 3, 1, 1),
                                                      nn.LeakyReLU(inplace=True))
            self.conv_up1 = nn.Conv2d(num_out_feats, num_out_feats, 3, 1, 1)
            self.conv_up2 = nn.Conv2d(num_out_feats, num_out_feats, 3, 1, 1)
            self.conv_hr = nn.Conv2d(num_out_feats, num_out_feats, 3, 1, 1)
            self.conv_last = nn.Conv2d(num_out_feats, out_channels, 3, 1, 1)
            self.lrelu = nn.LeakyReLU(negative_slope=0.2, inplace=True)
        else:
            self.conv_last = nn.Conv2d(embed_dim, out_channels, 3, 1, 1)
        self._mean_list = [float(v) for v in self.mean.flatten().tolist()]  # host copy (no device sync in forward)
        self._graphs = {}
        # opt-in CUDA-graph replay of the tensor-core forward (one captured graph per input shape): a forward is ~540
        # launches, which bounds small batches (one 256x256 Base tile) by launch latency, not by the kernels
        self.use_cuda_graph = os.environ.get("GRL_B200_CUDA_GRAPH", "0") == "1"

        self.apply(self._init_weights)
        if init_method in ["l", "w"] or init_method.find("t") >= 0:
            for layer in self.layers:
                layer._init_weights()
        self.precision = "fp32"
        self.set_precision(self._requested_precision)
        # a full reference state_dict also carries index_*/mask_* buffers: drop them instead of failing strict loads
        self._register_load_state_dict_pre_hook(self._drop_reference_buffers)

    # ---- precision ----------------------------------------------------------------------------
    def set_precision(self, precision):
        """"fp32": exact-parity kernels (<= 1e-3 vs the reference).  "fp16" / "bf16": wgmma tensor-core path with
        that MMA operand format (fp32 accumulation, residual stream, LayerNorm and softmax statistics); fp16 operands
        (11-bit mantissa) are what meets the 0.01 dB PSNR gate, bf16 is provided for range-critical checkpoints.
        "auto": fp16 when the architecture fits the tensor-core kernels (head_dim <= 32, C % 4 == 0), else fp32."""
        if precision not in ("fp32", "fp16", "bf16", "auto"):
            raise ValueError(f"precision must be fp32 / fp16 / bf16 / auto, got {precision!r}")
        ok = all(tc.supported(self.embed_dim, b.num_heads_w, b.num_heads_s) for l in self.layers for b in l.blocks)
        if precision in ("fp16", "bf16") and not ok:
            raise RuntimeError(f"this architecture is outside the tensor-core path (needs head_dim <= 32, <= 8 heads, C % 4 == 0 "
                               f"and C <= {tc.LN_MAX_C}); use precision='fp32' or 'auto'")
        self.precision = ("fp16" if precision == "auto" else precision) if (precision != "fp32" and ok) else "fp32"
        for l in self.layers:
            for b in l.blocks:
                b.precision = self.precision
        return self.precision

    # ---- tables / indices / masks ------------------------------------------------------------
    def _tables(self, x_size):
        """The coordinate tables of the stripes the blocks run at x_size.  A vertical-stripe block splits the image with
        stripe_size[::-1] and stripe_groups[::-1] (efficient.py:466-468), which differs from the horizontal stripe
        transposed when stripe_groups split a non-square image; the reference's table_sv is the transposed one (see
        set_table_index_mask), so its own forward cannot run there."""
        ss, _ = _get_stripe_info(self.stripe_size, self.stripe_groups, True, x_size)
        sv, _ = _get_stripe_info(list(self.stripe_size)[::-1], list(self.stripe_groups)[::-1], True, x_size)
        df = self.anchor_window_down_factor
        return {"table_w": G.coords_table(self.window_size), "table_sh": G.coords_table(ss, df),
                "table_sv": G.coords_table(sv, df)}

    def set_table_index_mask(self, x_size, materialize=False):
        """grl.py:386-429.  With materialize=True returns the reference's 13 CPU tensors (bit-exact); the default
        returns the three tables plus zero-size markers for the indices / masks the kernels compute on the fly."""
        out = self._tables(x_size)
        names_i = ("index_w", "index_sh_a2w", "index_sh_w2a", "index_sv_a2w", "index_sv_w2a")
        names_m = ("mask_w", "mask_sh_a2w", "mask_sh_w2a", "mask_sv_a2w", "mask_sv_w2a")
        if not materialize:
            for n in names_i + names_m:
                out[n] = _closed_form_marker()
            return out
        ss, sss = _get_stripe_info(self.stripe_size, self.stripe_groups, True, x_size)
        df = self.anchor_window_down_factor
        out["table_sv"] = G.coords_table(ss[::-1], df)
        out["index_w"] = G.position_index(self.window_size)
        out["mask_w"] = G.shift_mask(x_size, self.window_size, self.shift_size)
        for d, s, sh in (("sh", ss, sss), ("sv", ss[::-1], sss[::-1])):
            for tag, w2a in (("a2w", False), ("w2a", True)):
                out[f"index_{d}_{tag}"] = G.position_index(s, df, w2a)
                out[f"mask_{d}_{tag}"] = G.shift_mask(x_size, s, sh, df, w2a)
        return out

    def get_table_index_mask(self, device=None, input_resolution=None):
        """grl.py:431-453 -- but a resolution change costs three small table uploads instead of a 1.3 GB rebuild."""
        if tuple(input_resolution) == tuple(self.input_resolution):
            t = {"table_w": self.table_w, "table_sh": self.table_sh, "table_sv": self.table_sv}
        else:
            # the coordinate tables depend only on the resolution: uploaded once per (resolution, device), which also
            # keeps host->device copies out of a CUDA-graph capture
            key = (tuple(input_resolution), str(device))
            cache = self.__dict__.setdefault("_table_cache", {})
            if key not in cache:
                if len(cache) >= 16:
                    cache.clear()
                cache[key] = Produced({k: upload(v, device) for k, v in self._tables(input_resolution).items()})
            t = dict(cache[key].use())
        for n in ("index_w", "index_sh_a2w", "index_sh_w2a", "index_sv_a2w", "index_sv_w2a", "mask_w", "mask_sh_a2w",
                  "mask_sh_w2a", "mask_sv_a2w", "mask_sv_w2a"):
            t[n] = _closed_form_marker()
        return t

    @staticmethod
    def _drop_reference_buffers(state_dict, prefix, *args):
        for k in list(state_dict.keys()):
            n = k[len(prefix):] if k.startswith(prefix) else None
            if n is not None and "." not in n and (n.startswith("index_") or n.startswith("mask_")):
                state_dict.pop(k)

    def _init_weights(self, m):
        """grl.py:455-462."""
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"absolute_pos_embed"}

    @torch.jit.ignore
    def no_weight_decay_keywords(self):
        return {"relative_position_bias_table"}

    # ---- forward --------------------------------------------------------------------------------
    def check_image_size(self, x):
        """grl.py:479-489."""
        _, _, h, w = x.size()
        mod_pad_h = (self.pad_size - h % self.pad_size) % self.pad_size
        mod_pad_w = (self.pad_size - w % self.pad_size) % self.pad_size
        try:
            x = F.pad(x, (0, mod_pad_w, 0, mod_pad_h), "reflect")
        except BaseException:
            x = F.pad(x, (0, mod_pad_w, 0, mod_pad_h), "constant")
        return x

    # ---- CUDA graphs ----------------------------------------------------------------------------
    def reset_cuda_graphs(self):
        """Drops every captured graph (they bake in the addresses of the packed weights and of their static buffers).
        A graph is also dropped and recaptured by itself when a packed-weight plan it reads is no longer current: after
        set_precision, or after an in-place edit of a parameter (which bumps its version).  An edit through
        `param.data` bypasses the version counter, so nothing can detect it, neither here nor in the eager path's
        packed weights: edit parameters in place under torch.no_grad(), or load_state_dict."""
        self._graphs = {}

    def _graph_plans(self):
        """The packed-weight plans a tensor-core forward reads: every block's tc.BlockPlan and every tc.ConvPlan."""
        return ([b._tc_plan for layer in self.layers for b in layer.blocks] +
                [p for m in self.modules() for p in m.__dict__.get("_tc_convs", {}).values()])

    def _graph_current(self, ent):
        """Whether a captured graph reads the current weights: no parameter changed version since the capture, and
        every plan is still the one captured (set_precision / an edit rebuild them and free the captured ones)."""
        plans, vkey = ent[3], ent[4]
        now = self._graph_plans()
        return tc._version_key(self) == vkey and len(now) == len(plans) and all(a is b for a, b in zip(now, plans))

    def _apply(self, fn, *args, **kwargs):  # .to() / .cuda() / .half() move parameters: captured graphs are stale
        self._graphs = {}
        return super()._apply(fn, *args, **kwargs)

    def load_state_dict(self, *args, **kwargs):
        self._graphs = {}
        return super().load_state_dict(*args, **kwargs)

    @torch.no_grad()
    def _forward_graphed(self, x, rggb=False):
        """Replays a captured graph of tc.forward for this input shape and format (captures it on first use, after two
        eager warm-up forwards that build the packed weights / bias tables / kernel attributes).  The result is a fresh
        tensor (the caller may mutate it in place, engines/base.py:113).  Replays of one graph share its static buffers,
        so they are serialised across streams: the entry's `done` (a streams.Produced of every tensor the graph reads or
        writes) is recorded after the output's clone, and the next replay's stream waits on it."""
        key = (tuple(x.shape), x.device.index, self.precision, "rggb" if rggb else "rgb")
        ent = self._graphs.get(key)
        if ent is not None and not self._graph_current(ent):
            del self._graphs[key]
            ent = None
        if ent is None:
            static_in = x.clone()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    tc.forward(self, static_in, rggb)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_out = tc.forward(self, static_in, rggb)
            # the graph reads every block's cached attention constants (tc.BlockPlan) at their addresses at capture; a
            # forward at another resolution replaces that cache, so the graph holds its own references to them
            consts = [b._tc_plan._consts for layer in self.layers for b in layer.blocks]
            # ... and the packed weights of the plans it was captured with: it replays only while they are current
            plans = self._graph_plans()
            held = (static_in, static_out, [c.value for c in consts], [p.ready.value for p in plans])
            ent = [graph, Produced(held), consts, plans, tc._version_key(self)]
            self._graphs[key] = ent
        graph, done = ent[:2]
        static_in, static_out = done.use()[:2]
        static_in.copy_(x)
        graph.replay()
        y = static_out.clone()
        ent[1] = Produced(done.value)
        return y

    @torch.no_grad()
    def forward_features(self, x, launch=tc.DEVICE):
        """(B, C, H, W) -> (B, C, H, W) like the reference (grl.py:491-504).  Channels-last in between: a permuted
        channels-last input is read and the result returned as such a view, without layout copies."""
        B, C, H, W = x.shape
        t = ln_residual(launch, self.norm_start, x.permute(0, 2, 3, 1).contiguous().view(B, H * W, C))
        tim = self.get_table_index_mask(x.device, (H, W))
        for si, layer in enumerate(self.layers):
            t = layer(t, (H, W), tim, launch, f"stage{si}")
        return ln_residual(launch, self.norm_end, t).view(B, H, W, C).permute(0, 3, 1, 2)

    @torch.no_grad()
    def forward(self, x):
        K.capi.require_device(x)
        if self.input_format == "rgb":
            return self.forward_rgb(x)
        if self.input_format != "rggb":
            raise ValueError(f"input_format must be 'rgb' or 'rggb', got {self.input_format!r}")
        if self.in_channels != 3 or x.dim() != 4 or x.shape[1] != 4 or x.shape[2] < 2 or x.shape[3] < 2:
            raise ValueError(f"input_format='rggb' takes packed RGGB Bayer planes (B, 4, h, w) with h, w >= 2 and a "
                             f"3-channel network; got input {tuple(x.shape)}, in_channels={self.in_channels}")
        cfa = x.float().contiguous()
        if self.self_ensemble:
            # demosaic once, then the RGB forward (the engine's order: the ensemble's views are views of the RGB image)
            return self.forward_rgb(K.demosaic(cfa)).to(x.dtype)
        return self._forward_once(cfa, rggb=True).to(x.dtype)

    @torch.no_grad()
    def forward_rgb(self, x):
        """The forward on a (B, in_channels, H, W) image whatever input_format says (self_ensemble applies)."""
        K.capi.require_device(x)
        return self._forward_self_ensemble(x) if self.self_ensemble else self._forward_once(x)

    @torch.no_grad()
    def forward_u8(self, img):
        """The forward on decoded 8-bit images: img (B, H, W, in_channels) uint8 on the GPU -> (B, H*s, W*s,
        out_channels) uint8.  Exactly f32_to_u8(forward_rgb(u8_to_f32(img))): the datasets' to_tensor and the validation
        step's tensor_round as one kernel each around the forward, so precision, self_ensemble and use_cuda_graph apply."""
        if self.input_format == "rggb":
            raise ValueError("forward_u8 takes (B, H, W, C) 8-bit images; packed 8-bit Bayer input (input_format='rggb') "
                             "is not supported")
        K.capi.require_device(img)
        if img.dim() != 4 or img.shape[3] != self.in_channels:
            raise ValueError(f"forward_u8 takes (B, H, W, {self.in_channels}) uint8 images, got {tuple(img.shape)}")
        return K.f32_to_u8(self.forward_rgb(K.u8_to_f32(img)))

    def forward_list(self, images):
        """The forward on a list of differently sized images, as a test set comes: images[i] is (in_channels, H_i, W_i)
        (input_format "rggb": packed Bayer planes (4, h_i, w_i)), all of one float dtype, on the GPU.  Returns the list of
        outputs in input order; element i equals self(images[i][None])[0] bit for bit, whatever precision,
        use_cuda_graph and self_ensemble say.  Images that pad to the same size run in one batched forward of at most
        max_batch_tokens padded pixels (image_list.py); with self_ensemble each image runs on its own."""
        return image_list.forward_list(self, images)

    def forward_list_u8(self, images):
        """forward_list of decoded 8-bit images (H_i, W_i, in_channels) uint8 on the GPU -> (H_i*s, W_i*s, out_channels)
        uint8; element i equals forward_u8(images[i][None])[0] bit for bit."""
        return image_list.forward_list(self, images, u8=True)

    @torch.no_grad()
    def _forward_self_ensemble(self, x):
        """y = 0.125 * (V_0 + ... + V_7), V_m = inverse_m(forward(augment_img_tensor4(x, m))) (utils/utils_bsr/
        utils_image.py:444-460): 8 independent forwards, each with its own padding, on the views gathered by one kernel
        per group.  Group A (modes 0, 2, 4, 6) keeps (H, W) and goes first, group B (the transposed modes) follows; when
        H == W both groups share one view batch.  Each forward takes at most ensemble_max_batch views."""
        xin = x.float().contiguous()
        B, C, H, W = xin.shape
        if H == W:
            views = torch.empty(8 * B, C, H, W, device=xin.device, dtype=torch.float32)
            K.ens_gather(xin, 0, out=views[: 4 * B])
            K.ens_gather(xin, 1, out=views[4 * B:])
            y = self._forward_chunks(views)
            ya, yb = y[: 4 * B], y[4 * B:]
        else:
            ya = self._forward_chunks(K.ens_gather(xin, 0))
            yb = self._forward_chunks(K.ens_gather(xin, 1))
        return K.ens_merge(ya, yb, B).to(x.dtype)

    def _forward_chunks(self, views):
        n = max(1, int(self.ensemble_max_batch))
        outs = [self._forward_once(views[i:i + n]) for i in range(0, views.shape[0], n)]
        return outs[0] if len(outs) == 1 else torch.cat(outs)

    @torch.no_grad()
    def _forward_once(self, x, rggb=False):
        """One forward on the tensor-core or fp32 kernels; rggb: x is packed Bayer planes (the tensor-core path demosaics
        inside its head kernel)."""
        if self.precision == "fp32":
            return self._forward_f32(x, rggb)
        xin = x.float().contiguous()
        y = self._forward_graphed(xin, rggb) if self.use_cuda_graph else tc.forward(self, xin, rggb)
        return y.to(x.dtype)

    @torch.no_grad()
    def _forward_f32(self, x, rggb=False, launch=tc.DEVICE):
        """The fp32 forward (grl.py:506-551), channels-last between the head and the tail, every kernel issued through
        `launch`; rggb: x is packed (B, 4, h, w) Bayer planes, demosaiced first."""
        if rggb:
            rgb = torch.empty(x.shape[0], 3, 2 * x.shape[2], 2 * x.shape[3], device=x.device, dtype=torch.float32)
            launch.run(K.demosaic, x, out=rgb)
            x = rgb
        H, W = x.shape[2:]
        x = self.check_image_size(x)
        mean = upload(self.mean, x.device).to(x.dtype)
        x = ((x - mean) * self.img_range).float()
        xc = x.permute(0, 2, 3, 1).contiguous()

        def conv(name, inp, act=K.ACT_NONE, slope=0.0, res=None, key=None):
            return conv3x3(launch, name, self, key or name, inp, act, slope, res)

        first = conv("conv_first", xc)
        body = conv("conv_after_body", self.forward_features(first.permute(0, 3, 1, 2), launch).permute(0, 2, 3, 1),
                    res=first)
        if self.upsampler == "pixelshuffle":
            t = conv("conv_before_upsample", body, K.ACT_LEAKY, 0.01, key="conv_before_upsample.0")
            y = conv("conv_last", self.upsample.forward_cl(t, launch))
        elif self.upsampler == "pixelshuffledirect":
            y = self.upsample.forward_cl(body, launch)
        elif self.upsampler == "nearest+conv":
            t = conv("conv_before_upsample", body, K.ACT_LEAKY, 0.01, key="conv_before_upsample.0")
            up = lambda v: v.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
            t = conv("conv_up1", up(t), K.ACT_LEAKY, 0.2)
            t = conv("conv_up2", up(t), K.ACT_LEAKY, 0.2)
            y = conv("conv_last", conv("conv_hr", t, K.ACT_LEAKY, 0.2))
        else:
            y = conv("conv_last", body, res=xc if self.in_channels == self.out_channels else None)
        y = y.permute(0, 3, 1, 2) / self.img_range + mean
        return y[:, :, : H * self.upscale, : W * self.upscale].contiguous()

    def flops(self):
        pass

    def convert_checkpoint(self, state_dict):
        """grl.py:556-569."""
        for k in list(state_dict.keys()):
            if (k.find("relative_coords_table") >= 0 or k.find("relative_position_index") >= 0
                    or k.find("attn_mask") >= 0 or k.find("model.table_") >= 0 or k.find("model.index_") >= 0
                    or k.find("model.mask_") >= 0):
                state_dict.pop(k)
                print(k)
        return state_dict


# ----------------------------------------------------------------------------------------------
# launch listing
# ----------------------------------------------------------------------------------------------
class GemmF32(NamedTuple):
    """One K.linear / K.conv3x3 launch of an fp32 forward (K = 9 Cin for a conv)."""
    name: str
    conv: bool
    K: int
    N: int
    act: int
    slope: float
    bias: bool
    res: bool


class AttnF32(NamedTuple):
    """One attention pass of an fp32 forward: a K.window_attention launch ("window"), or pass 1 ("stripe1": anchors
    attend to the stripe's tokens) / pass 2 ("stripe2": tokens attend to the anchors) of a K.stripe_attention launch."""
    name: str
    role: str
    gq: object
    gk: object
    heads: int
    d: int
    use_mask: bool


def f32_launches(model, x_shape):
    """GemmF32 / AttnF32 descriptors of one fp32 forward of GRL `model` on a (B, Cin, H, W) input, in launch order:
    GRL._forward_f32 run with tc.Listing on a meta input (with input_format "rggb", x_shape is the packed (B, 4, h, w)
    Bayer input of the (2h, 2w) image).  Needs no device: conv weights are packed on the model's device, nothing runs."""
    if model.precision != "fp32":
        raise ValueError(f"f32_launches lists the fp32 forward; the model runs {model.precision}")
    listing = tc.Listing()
    model._forward_f32(torch.empty(x_shape, device="meta"), model.input_format == "rggb", listing)
    out = []
    for name, fn, args, kw in listing.launches:
        a = inspect.signature(fn).bind(*args, **kw)
        a.apply_defaults()
        a = a.arguments
        if fn in (K.linear, K.conv3x3):
            w = a["weight"] if fn is K.linear else a["wpacked"]
            out.append(GemmF32(name, fn is K.conv3x3, w.shape[1], w.shape[0], a["act"], a["slope"], a["bias"] is not None,
                               a["res"] is not None))
        else:
            h, d, mask = a["heads"], a["qkv"].shape[2] // 3 // a["heads"], bool(a["use_mask"])
            if fn is K.window_attention:
                out.append(AttnF32(name, "window", a["grid"], a["grid"], h, d, mask))
            else:
                tok, anc = a["tok_grid"], a["anc_grid"]
                out += [AttnF32(name, "stripe1", anc, tok, h, d, mask), AttnF32(name, "stripe2", tok, anc, h, d, mask)]
    return out
