"""nn layers on the hand-written sm_90a kernels (see layers.py)."""
from .layers import FusedLinear, FusedMLP, dot_interaction, fm_interaction

__all__ = ["FusedLinear", "FusedMLP", "dot_interaction", "fm_interaction"]
