"""nn layers on the hand-written sm_90a kernels (see layers.py)."""
from .layers import FusedLinear, FusedMaskBlock, FusedMLP, dot_interaction, fm_interaction, fused_encoder_layer, fused_gru

__all__ = ["FusedLinear", "FusedMaskBlock", "FusedMLP", "dot_interaction", "fm_interaction", "fused_encoder_layer", "fused_gru"]
