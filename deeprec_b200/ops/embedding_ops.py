"""Embedding lookup API (python/ops/embedding_ops.py:365-2055 in the reference).

``SparseIds`` is the SparseTensor analogue: flat ``values`` [nnz] with ``row_ids`` [nnz]
(sorted by row) and ``batch_size``; optional per-id ``weights``.

On CUDA tensors the combiner runs in the fused sm_90a multi-table kernel
(csrc/cuda/embedding_kernels.cu -- one launch for all tables of a group); on CPU it is
index_add over the host engine's gather.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Union

import torch

from ..embedding_variable import (DynamicEmbeddingVariable, EmbeddingVariable, MultiHashVariable,
                                  PartitionedEmbeddingVariable)


@dataclass
class SparseIds:
    values: torch.Tensor                     # [nnz] int64
    row_ids: torch.Tensor                    # [nnz] int64, non-decreasing
    batch_size: int
    weights: Optional[torch.Tensor] = None   # [nnz] float

    @staticmethod
    def from_padded(ids: torch.Tensor, pad_value: int = -1, weights: Optional[torch.Tensor] = None) -> "SparseIds":
        """[B, L] matrix padded with ``pad_value`` (ids < 0 are treated as padding)."""
        mask = ids != pad_value
        rows = torch.arange(ids.shape[0], device=ids.device).unsqueeze(1).expand_as(ids)
        return SparseIds(ids[mask], rows[mask], ids.shape[0], weights[mask] if weights is not None else None)

    @staticmethod
    def from_offsets(values: torch.Tensor, offsets: torch.Tensor, weights: Optional[torch.Tensor] = None) -> "SparseIds":
        """CSR: ``offsets`` [B+1]."""
        lens = offsets[1:] - offsets[:-1]
        rows = torch.repeat_interleave(torch.arange(lens.numel(), device=values.device), lens)
        return SparseIds(values, rows, lens.numel(), weights)

    @staticmethod
    def from_dense(ids: torch.Tensor) -> "SparseIds":
        """[B] or [B, L] with every position valid."""
        if ids.dim() == 1:
            ids = ids.unsqueeze(1)
        rows = torch.arange(ids.shape[0], device=ids.device).unsqueeze(1).expand_as(ids)
        return SparseIds(ids.reshape(-1), rows.reshape(-1), ids.shape[0])

    def to(self, device) -> "SparseIds":
        return SparseIds(self.values.to(device), self.row_ids.to(device), self.batch_size,
                         self.weights.to(device) if self.weights is not None else None)


Table = Union[EmbeddingVariable, PartitionedEmbeddingVariable, MultiHashVariable, torch.nn.Embedding, torch.Tensor]


def _rows(params: Table, ids: torch.Tensor) -> torch.Tensor:
    if isinstance(params, (EmbeddingVariable, PartitionedEmbeddingVariable, MultiHashVariable)):
        return params.lookup(ids)
    if isinstance(params, torch.nn.Embedding):
        return params(ids)
    return params[ids]


def embedding_lookup(params: Table, ids: torch.Tensor, max_norm: Optional[float] = None,
                     blocknums: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``tf.nn.embedding_lookup`` (embedding_ops.py:365): ids [...] -> [..., D]."""
    if isinstance(params, DynamicEmbeddingVariable):
        e = params.lookup(ids, blocknums)
    else:
        e = _rows(params, ids)
    if max_norm is not None:
        n = e.norm(dim=-1, keepdim=True)
        e = e * torch.clamp(max_norm / (n + 1e-12), max=1.0)
    return e


def _combine(rows: torch.Tensor, sp: SparseIds, combiner: str) -> torch.Tensor:
    B, D = sp.batch_size, rows.shape[-1]
    rid = sp.row_ids.to(rows.device)
    w = sp.weights.to(rows.device, rows.dtype) if sp.weights is not None else None
    if w is not None:
        rows = rows * w.unsqueeze(-1)
    out = torch.zeros(B, D, dtype=rows.dtype, device=rows.device).index_add_(0, rid, rows)
    if combiner == "sum":
        return out
    ones = w if w is not None else torch.ones(rid.numel(), dtype=rows.dtype, device=rows.device)
    if combiner == "mean":
        den = torch.zeros(B, dtype=rows.dtype, device=rows.device).index_add_(0, rid, ones)
        return out / den.clamp_min(1e-12).unsqueeze(-1) * (den > 0).unsqueeze(-1)
    if combiner == "sqrtn":
        den = torch.zeros(B, dtype=rows.dtype, device=rows.device).index_add_(0, rid, ones * ones)
        return out / den.sqrt().clamp_min(1e-12).unsqueeze(-1) * (den > 0).unsqueeze(-1)
    raise ValueError(f"combiner must be sum|mean|sqrtn, got {combiner}")


def embedding_lookup_sparse(params: Table, sp_ids: SparseIds, sp_weights: Optional[torch.Tensor] = None,
                            combiner: str = "mean", max_norm: Optional[float] = None) -> torch.Tensor:
    """``tf.nn.embedding_lookup_sparse`` (embedding_ops.py:484): [B, D]."""
    if sp_weights is not None:
        sp_ids = SparseIds(sp_ids.values, sp_ids.row_ids, sp_ids.batch_size, sp_weights)
    rows = embedding_lookup(params, sp_ids.values, max_norm=max_norm)
    return _combine(rows, sp_ids, combiner)


def safe_embedding_lookup_sparse(params: Table, sp_ids: SparseIds, sp_weights: Optional[torch.Tensor] = None,
                                 combiner: str = "mean", default_id: Optional[int] = None,
                                 max_norm: Optional[float] = None) -> torch.Tensor:
    """``safe_embedding_lookup_sparse`` (embedding_ops.py:838): prune invalid ids (<0) and
    non-positive weights, empty rows yield the ``default_id`` row or zeros."""
    v, r, w = sp_ids.values, sp_ids.row_ids, sp_weights if sp_weights is not None else sp_ids.weights
    keep = v >= 0
    if w is not None:
        keep &= w > 0
    v, r = v[keep], r[keep]
    w = w[keep] if w is not None else None
    B = sp_ids.batch_size
    filled = None
    if default_id is not None:
        present = torch.zeros(B, dtype=torch.bool, device=v.device).index_fill_(0, r, True)
        empty = (~present).nonzero(as_tuple=True)[0]
        if empty.numel():
            v = torch.cat([v, torch.full_like(empty, default_id)])
            r = torch.cat([r, empty])
            if w is not None:
                w = torch.cat([w, torch.ones(empty.numel(), dtype=w.dtype, device=w.device)])
            order = torch.argsort(r, stable=True)
            v, r = v[order], r[order]
            w = w[order] if w is not None else None
        filled = True
    return embedding_lookup_sparse(params, SparseIds(v, r, B, w), None, combiner, max_norm)


# The reference ships "fused" variants that collapse the ~dozen graph ops of the safe lookup into
# Pre/Post kernels (core/ops/fused_embedding_ops.cc:12-276).  Here every lookup is already one
# gather + one combine, so the fused names map onto the same implementation; on CUDA they hit the
# fused multi-table kernel.
def fused_embedding_lookup_sparse(params, sp_ids, sparse_weights=None, combiner="mean", max_norm=None,
                                  default_id=None, prune_invalid_ids=False, fill_empty_row=True, blocknums=None):
    if prune_invalid_ids or fill_empty_row:
        return safe_embedding_lookup_sparse(params, sp_ids, sparse_weights, combiner,
                                            default_id if fill_empty_row else None, max_norm)
    return embedding_lookup_sparse(params, sp_ids, sparse_weights, combiner, max_norm)


def fused_safe_embedding_lookup_sparse(params, sp_ids, sparse_weights=None, combiner="mean", default_id=None,
                                       max_norm=None, prune=True):
    return safe_embedding_lookup_sparse(params, sp_ids, sparse_weights, combiner, default_id, max_norm)


def embedding_lookup_sparse_multi_dim(params: Sequence[Table], sp_ids: SparseIds, sp_weights=None,
                                      combiners: Sequence[str] = ("mean",), max_norm=None) -> List[torch.Tensor]:
    """``embedding_lookup_sparse_multi_dim`` (embedding_ops.py:1200): same ids, several tables."""
    combs = list(combiners) * (len(params) // len(combiners)) if len(combiners) != len(params) else list(combiners)
    return [embedding_lookup_sparse(p, sp_ids, sp_weights, c, max_norm) for p, c in zip(params, combs)]


def adaptive_embedding_lookup_sparse(hash_params: Table, ev_params: Table, sp_ids: SparseIds, hash_ev_ids: SparseIds,
                                     sp_weights=None, combiner: str = "mean", max_norm=None,
                                     adaptive_mask_tensor: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Adaptive embedding (embedding_ops.py:1454-1592): per id, ``adaptive_mask`` selects the EV
    (hot ids, mask==1) or the static hashed table (cold ids, looked up with ``hash_ev_ids``)."""
    if adaptive_mask_tensor is None:
        adaptive_mask_tensor = torch.ones_like(sp_ids.values, dtype=torch.bool)
    m = adaptive_mask_tensor.to(torch.bool)
    ev_rows = embedding_lookup(ev_params, sp_ids.values, max_norm=max_norm)
    hs_rows = embedding_lookup(hash_params, hash_ev_ids.values, max_norm=max_norm)
    rows = torch.where(m.unsqueeze(-1).to(ev_rows.device), ev_rows, hs_rows.to(ev_rows.device))
    if sp_weights is not None:
        sp_ids = SparseIds(sp_ids.values, sp_ids.row_ids, sp_ids.batch_size, sp_weights)
    return _combine(rows, sp_ids, combiner)


# ---------------------------------------------------------------------------------------------
# Group embedding (embedding_ops.py:1594-2055; kernels/group_embedding/*)
# ---------------------------------------------------------------------------------------------
def group_embedding_lookup_sparse(params: Sequence[Table], sp_ids: Sequence[SparseIds],
                                  combiners: Sequence[str], sp_weights: Optional[Sequence] = None,
                                  is_sequence: bool = False, params_num_per_group: int = 0) -> List[torch.Tensor]:
    """``tf.nn.group_embedding_lookup_sparse``: N tables looked up and combined together.
    Device tables of equal dim go through ONE fused gather+combine launch; with a collective
    strategy active (``parallel.CollectiveStrategy``) tables are model-parallel and the call
    routes through the fused P2P dispatch kernel."""
    from ..parallel import strategy as _strategy
    st = _strategy.current()
    if st is not None and st.in_embedding_scope and st.world_size > 1:
        return st.distributed_lookup(params, sp_ids, combiners, sp_weights)
    if sp_weights is None:
        sp_weights = [None] * len(params)
    dev_ok = all(isinstance(p, EmbeddingVariable) and p.device.type == "cuda" for p in params)
    if dev_ok and not is_sequence:
        from .device_table import group_lookup_sparse_device
        return group_lookup_sparse_device(params, sp_ids, combiners, sp_weights)
    outs = []
    for p, s, c, w in zip(params, sp_ids, combiners, sp_weights):
        if is_sequence:
            outs.append(embedding_lookup(p, s.values))
        else:
            outs.append(embedding_lookup_sparse(p, s, w, c))
    return outs


def group_embedding_lookup(params: Sequence[Table], ids: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    """``tf.nn.group_embedding_lookup`` (embedding_ops.py:1934): dense ids per table."""
    return [embedding_lookup(p, i) for p, i in zip(params, ids)]
