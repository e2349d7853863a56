"""DLRM as a plain PyTorch module on the framework API (EmbeddingVariable + feature lookups).

This is the portable path (CPU host engine or CUDA device tables through autograd) and the fp32
numerics oracle for :class:`deeprec_b200.models.dlrm_engine.DLRMEngine`.
Architecture: modelzoo/dlrm/train.py:68-243.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
from torch import nn

from ..config import EmbeddingVariableOption
from ..embedding_variable import EmbeddingVariable, get_embedding_variable


class _HostDotInteraction(torch.autograd.Function):
    """CPU fp32: the native per-sample kernel of csrc/host/host_engine.cc (no cat / bmm / index gather / index_put)."""

    @staticmethod
    def forward(ctx, dense, embs):
        from .. import _native
        dense, embs = dense.contiguous(), embs.contiguous()
        B, T, D = embs.shape
        out = torch.empty(B, D + (T + 1) * T // 2, dtype=torch.float32)
        _native.host().dr_host_dot_interaction_fwd(_native.ptr(dense), _native.ptr(embs), B, T, D, _native.ptr(out))
        ctx.save_for_backward(dense, embs)
        return out

    @staticmethod
    def backward(ctx, dz):
        from .. import _native
        dense, embs = ctx.saved_tensors
        B, T, D = embs.shape
        dz = dz.contiguous()
        dd, de = torch.empty_like(dense), torch.empty_like(embs)
        _native.host().dr_host_dot_interaction_bwd(_native.ptr(dense), _native.ptr(embs), _native.ptr(dz), B, T, D, _native.ptr(dd), _native.ptr(de))
        return dd, de


def dot_interaction(dense: torch.Tensor, embs: torch.Tensor) -> torch.Tensor:
    """dense [B, D], embs [B, T, D] -> [B, D + (T+1)T/2]; pair order (i, j<i) row-major
    (tf.boolean_mask of the strict lower triangle, modelzoo/dlrm/train.py:121-133)."""
    if dense.device.type == "cpu" and dense.shape[1] == embs.shape[2] and dense.dtype in (torch.float32, torch.bfloat16):
        # under bf16 autocast the bottom MLP hands over bf16: the interaction itself stays fp32 (it is bandwidth-, not FLOP-bound)
        return _HostDotInteraction.apply(dense.float(), embs.float())
    return dot_interaction_reference(dense, embs)


def dot_interaction_reference(dense: torch.Tensor, embs: torch.Tensor) -> torch.Tensor:
    """The composite expression (any device / dtype): the numerics oracle of every dot-interaction kernel."""
    feats = torch.cat([dense.unsqueeze(1), embs], dim=1)
    gram = torch.bmm(feats, feats.transpose(1, 2))
    F = feats.shape[1]
    li, lj = torch.tril_indices(F, F, offset=-1, device=dense.device)
    return torch.cat([dense, gram[:, li, lj]], dim=1)


class DLRM(nn.Module):
    def __init__(self, num_dense: int = 13, cardinalities: Sequence[int] = (1000,) * 26, embedding_dim: int = 16,
                 mlp_bot: Sequence[int] = (512, 256, 64, 16), mlp_top: Sequence[int] = (512, 256), interaction_op: str = "dot",
                 ev_option: Optional[EmbeddingVariableOption] = None, device=None, use_ev: bool = True,
                 bn_eps: float = 1e-3, bn_momentum: float = 0.99, name: str = "dlrm", fused_kernels: bool = False):
        super().__init__()
        self.fused_kernels = fused_kernels
        import copy
        self.interaction_op = interaction_op
        T = len(cardinalities)
        if use_ev:
            self.tables = nn.ModuleList([
                get_embedding_variable(f"{name}/C{i + 1}", embedding_dim, ev_option=copy.deepcopy(ev_option) if ev_option else None, device=device)
                for i in range(T)])
        else:
            self.tables = nn.ModuleList([nn.Embedding(int(c), embedding_dim, device=device) for c in cardinalities])
        layers: List[nn.Module] = []
        k = num_dense
        for n in mlp_bot:
            layers += [nn.Linear(k, n, device=device), nn.ReLU(), nn.BatchNorm1d(n, eps=bn_eps, momentum=1.0 - bn_momentum, device=device)]
            k = n
        self.bot = nn.Sequential(*layers)
        k = (embedding_dim + (T + 1) * T // 2) if interaction_op == "dot" else embedding_dim * (T + 1)
        layers = []
        for n in mlp_top:
            layers += [nn.Linear(k, n, device=device), nn.ReLU()]
            k = n
        self.top = nn.Sequential(*layers)
        self.logits = nn.Linear(k, 1, device=device)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight); nn.init.zeros_(m.bias)

    def embedding_variables(self) -> List[EmbeddingVariable]:
        return [t for t in self.tables if isinstance(t, EmbeddingVariable)]

    def forward(self, dense: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
        """dense [B, num_dense]; ids [T, B] (feature-major) -> logits [B]."""
        x = self.bot(dense)
        embs = None
        if x.device.type == "cpu" and isinstance(self.tables[0], EmbeddingVariable):
            from ..ops.host_group import group_lookup_dense_host
            embs = group_lookup_dense_host(list(self.tables), ids)           # one native call -> [B, T, D]
        if embs is None:
            embs = torch.stack([(t.lookup(ids[i]) if isinstance(t, EmbeddingVariable) else t(ids[i])).to(x.device) for i, t in enumerate(self.tables)], dim=1)
        if self.interaction_op == "dot":
            if self.fused_kernels:
                from ..nn import dot_interaction as fused_dot   # tensor-core kernel on CUDA (bf16), the expression above on CPU
                z = fused_dot(x, embs)
            else:
                z = dot_interaction(x, embs)                    # fp32 oracle path
        else:
            z = torch.cat([x, embs.flatten(1)], dim=1)
        return self.logits(self.top(z)).squeeze(-1)

    def loss(self, dense, ids, labels) -> torch.Tensor:
        return nn.functional.binary_cross_entropy_with_logits(self.forward(dense, ids), labels)
