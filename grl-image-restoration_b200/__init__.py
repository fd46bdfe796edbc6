"""grl-image-restoration_b200: H100-native (sm_90a) implementation of GRL's forward hot path behind the
reference's nn.Module surface.  See DESIGN.md / INTEGRATION.md at the repository root."""
from . import checkpoint, configs, geometry, tiling  # noqa: F401
from .modules import (  # noqa: F401
    GRL, AffineTransform, AnchorLinear, AnchorProjection, AnchorStripeAttention, CAB, ChannelAttention, CPB_MLP,
    EfficientMixAttnTransformerBlock, MixedAttention, Mlp, QKVProjection, TransformerStage, Upsample, UpsampleOneStep,
    WindowAttention, build_last_conv,
)
from .functional import (  # noqa: F401
    awgn, awgn_list, awgn_noise_host, demosaic, dn_seed, jpeg_quant_tables, jpeg_roundtrip, jpeg_roundtrip_host,
    jpeg_roundtrip_list, luma, luma_list, mosaic, mosaic_list,
)
from .evaluation import RECIPES, evaluate  # noqa: F401

__all__ = ["GRL", "TransformerStage", "EfficientMixAttnTransformerBlock", "MixedAttention", "WindowAttention",
           "AnchorStripeAttention", "AffineTransform", "CAB", "ChannelAttention", "Mlp", "QKVProjection",
           "AnchorProjection", "AnchorLinear", "CPB_MLP", "Upsample", "UpsampleOneStep", "build_last_conv",
           "configs", "geometry", "demosaic", "jpeg_roundtrip", "jpeg_roundtrip_list", "jpeg_roundtrip_host",
           "jpeg_quant_tables", "dn_seed", "awgn", "awgn_list", "awgn_noise_host", "mosaic", "mosaic_list", "luma",
           "luma_list", "RECIPES", "evaluate"]
