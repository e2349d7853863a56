"""nn layers on the hand-written sm_90a kernels (see layers.py)."""
from .layers import (FUSED_MOE, FusedLinear, FusedMaskBlock, FusedMLP, MoEOps, dot_interaction, fm_interaction, fused_din_attention,
                     fused_encoder_layer, fused_expert_mlps, fused_gru, fused_moe_mix)

__all__ = ["FUSED_MOE", "FusedLinear", "FusedMaskBlock", "FusedMLP", "MoEOps", "dot_interaction", "fm_interaction", "fused_din_attention", "fused_encoder_layer",
           "fused_expert_mlps", "fused_gru", "fused_moe_mix"]
