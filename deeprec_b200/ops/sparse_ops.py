"""Sparse utility ops of the input / embedding front-end: prune + fill-empty-rows, COO slice / reshape, sparse segment reductions.

Reference: the fused-embedding "pre" kernels (``kernels/fused_embedding/fused_embedding_pre_ops_gpus.cu.cc:23-123``), ``SparseFillEmptyRows``
(``kernels/sparse_fill_empty_rows_op_util.cu.cc``), ``SparseSlice`` (``kernels/sparse_slice_op_gpu.cu.cc``), ``SparseReshape``, and the GPU
rewrites of ``SparseSegment{Sum,Mean,SqrtN}`` (``kernels/segment_reduction_ops_gpu.cu.{h,cc}``) -- SURVEY §2.14 K14 / K16.

CUDA tensors run ``csrc/cuda/sparse_utils.cu`` (every data-dependent size stays on the device until the caller asks for it: ONE host read of the
count per call); CPU tensors use the equivalent torch expressions below, which are also the oracle of the GPU tests."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

from .. import _native
from .._native import check, ptr, stream_ptr
from .embedding_ops import SparseIds

_MODES = {"sum": 0, "mean": 1, "sqrtn": 2}


def _workspace(nnz: int, rows: int, dev) -> torch.Tensor:
    return torch.empty(int(_native.cuda().dr_cuda_sparse_utils_workspace(nnz, rows)), dtype=torch.uint8, device=dev)


# ------------------------------------------------------------------------------------------------------------ prune + fill-empty-rows
def sparse_prune_fill(sp: SparseIds, default_id: Optional[int] = None, prune: bool = True) -> Tuple[SparseIds, torch.Tensor]:
    """Drop invalid entries (``id < 0``, ``weight <= 0``) when ``prune`` and give every row left empty one ``(default_id, weight 1)`` entry when
    ``default_id`` is not None; the result stays row-ordered.  Returns ``(SparseIds, empty_row_indicator [B] bool)`` -- the pair
    ``tf.sparse.retain`` + ``tf.sparse.fill_empty_rows`` computes in ``safe_embedding_lookup_sparse`` (embedding_ops.py:838)."""
    v, r, w, B = sp.values, sp.row_ids, sp.weights, sp.batch_size
    fill = default_id is not None
    if not _native.on_device(v):
        keep = torch.ones_like(v, dtype=torch.bool)
        if prune:
            keep = v >= 0
            if w is not None:
                keep &= w > 0
        v, r = v[keep], r[keep]
        w = w[keep] if w is not None else None
        present = torch.zeros(B, dtype=torch.bool).index_fill_(0, r, True)
        empty = ~present
        if fill and bool(empty.any()):
            e = empty.nonzero(as_tuple=True)[0]
            v, r = torch.cat([v, torch.full_like(e, default_id)]), torch.cat([r, e])
            if w is not None:
                w = torch.cat([w, torch.ones(e.numel(), dtype=w.dtype)])
            order = torch.argsort(r, stable=True)
            v, r = v[order], r[order]
            w = w[order] if w is not None else None
        return SparseIds(v, r, B, w), empty
    dev, nnz = v.device, v.numel()
    v, r = v.contiguous(), r.contiguous()
    wf = w.contiguous().float() if w is not None else None
    cap = nnz + B
    ov, orow = torch.empty(cap, dtype=torch.int64, device=dev), torch.empty(cap, dtype=torch.int64, device=dev)
    ow = torch.empty(cap, dtype=torch.float32, device=dev) if wf is not None else None
    empty = torch.empty(B, dtype=torch.int32, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    ws = _workspace(nnz, B, dev)
    check(_native.cuda().dr_cuda_sparse_prune_fill(ptr(v), ptr(r), ptr(wf), nnz, B, int(prune), int(fill), int(default_id or 0), ptr(ov), ptr(orow), ptr(ow), ptr(empty),
                                                   ptr(count), ptr(ws), stream_ptr()), "sparse_prune_fill")
    n = int(count.item())                                   # the one host read of this op
    return SparseIds(ov[:n], orow[:n], B, ow[:n].to(w.dtype) if ow is not None else None), empty.bool()


def sparse_fill_empty_rows(sp: SparseIds, default_id: int) -> Tuple[SparseIds, torch.Tensor]:
    """``tf.sparse.fill_empty_rows``: no pruning, one ``default_id`` entry per empty row."""
    return sparse_prune_fill(sp, default_id, prune=False)


# ------------------------------------------------------------------------------------------------------------ COO slice / reshape
def sparse_slice(indices: torch.Tensor, values: torch.Tensor, shape: Sequence[int], start: Sequence[int], size: Sequence[int]):
    """``tf.sparse.slice``: entries of the COO tensor ``(indices [nnz, R], values [nnz], shape)`` inside ``[start, start + size)``, indices
    re-based to the slice.  Returns ``(indices, values, shape)``."""
    R = indices.shape[1]
    assert len(shape) == len(start) == len(size) == R
    out_shape = [max(0, min(int(sz), int(sh) - int(st))) for sh, st, sz in zip(shape, start, size)]
    if not _native.on_device(indices):
        st = torch.tensor(list(start), dtype=torch.int64); sz = torch.tensor(list(size), dtype=torch.int64)
        keep = ((indices >= st) & (indices < st + sz)).all(dim=1)
        return indices[keep] - st, values[keep], out_shape
    if values.element_size() not in (4, 8):
        raise TypeError("sparse_slice: 4- or 8-byte values")
    dev, nnz = indices.device, indices.shape[0]
    idx, val = indices.contiguous(), values.contiguous()
    st = torch.tensor(list(start), dtype=torch.int64, device=dev); sz = torch.tensor(list(size), dtype=torch.int64, device=dev)
    oi, ov = torch.empty_like(idx), torch.empty_like(val)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    ws = _workspace(nnz, 1, dev)
    check(_native.cuda().dr_cuda_sparse_slice(ptr(idx), ptr(val), val.element_size(), nnz, R, ptr(st), ptr(sz), ptr(oi), ptr(ov), ptr(count), ptr(ws), stream_ptr()),
          "sparse_slice")
    n = int(count.item())
    return oi[:n], ov[:n], out_shape


def sparse_reshape(indices: torch.Tensor, shape: Sequence[int], new_shape: Sequence[int]) -> Tuple[torch.Tensor, list]:
    """``tf.sparse.reshape``: re-index ``indices [nnz, R0]`` from ``shape`` to ``new_shape`` (one dimension may be -1)."""
    total = 1
    for d in shape:
        total *= int(d)
    new_shape = [int(d) for d in new_shape]
    if new_shape.count(-1) > 1:
        raise ValueError("sparse_reshape: at most one -1")
    if -1 in new_shape:
        known = 1
        for d in new_shape:
            known *= d if d != -1 else 1
        if known == 0 or total % known:
            raise ValueError(f"sparse_reshape: cannot infer -1 for {shape} -> {new_shape}")
        new_shape[new_shape.index(-1)] = total // known
    prod = 1
    for d in new_shape:
        prod *= d
    if prod != total:
        raise ValueError(f"sparse_reshape: {shape} and {new_shape} hold different numbers of elements")
    R0, R1 = len(shape), len(new_shape)
    if not _native.on_device(indices):
        mul0 = torch.ones(R0, dtype=torch.int64)
        for d in range(R0 - 2, -1, -1):
            mul0[d] = mul0[d + 1] * int(shape[d + 1])
        lin = (indices * mul0).sum(dim=1)
        out = torch.empty(indices.shape[0], R1, dtype=torch.int64)
        for d in range(R1 - 1, -1, -1):
            out[:, d] = lin % new_shape[d]
            lin = lin // new_shape[d]
        return out, new_shape
    dev = indices.device
    idx = indices.contiguous()
    s0 = torch.tensor([int(d) for d in shape], dtype=torch.int64, device=dev); s1 = torch.tensor(new_shape, dtype=torch.int64, device=dev)
    out = torch.empty(idx.shape[0], R1, dtype=torch.int64, device=dev)
    check(_native.cuda().dr_cuda_sparse_reshape(ptr(idx), idx.shape[0], R0, ptr(s0), R1, ptr(s1), ptr(out), stream_ptr()), "sparse_reshape")
    return out, new_shape


# ------------------------------------------------------------------------------------------------------------ sparse segment reductions
def _segment_ref(data, indices, segment_ids, num_segments, mode):
    D = data.shape[1]
    out = torch.zeros(num_segments, D, dtype=data.dtype, device=data.device)
    out.index_add_(0, segment_ids, data[indices])
    if mode != "sum":
        cnt = torch.bincount(segment_ids, minlength=num_segments).clamp(min=1).to(data.dtype).unsqueeze(1)
        out = out / (cnt if mode == "mean" else cnt.sqrt())
    return out


class _SparseSegment(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, indices, segment_ids, num_segments, mode):
        d = data.contiguous().float()
        N, D = d.shape
        out = torch.empty(num_segments, D, dtype=torch.float32, device=d.device)
        check(_native.cuda().dr_cuda_sparse_segment_fwd(ptr(d), N, D, ptr(indices), ptr(segment_ids), indices.numel(), num_segments, mode, ptr(out), stream_ptr()),
              "sparse_segment_fwd")
        ctx.save_for_backward(indices, segment_ids); ctx.N, ctx.mode, ctx.dtype = N, mode, data.dtype
        return out.to(data.dtype)

    @staticmethod
    def backward(ctx, g):
        indices, segment_ids = ctx.saved_tensors
        g2 = g.contiguous().float()
        S, D = g2.shape
        dd = torch.zeros(ctx.N, D, dtype=torch.float32, device=g.device)
        check(_native.cuda().dr_cuda_sparse_segment_bwd(ptr(g2), S, D, ptr(indices), ptr(segment_ids), indices.numel(), ctx.N, ctx.mode, ptr(dd), stream_ptr()),
              "sparse_segment_bwd")
        return dd.to(ctx.dtype), None, None, None, None


def _sparse_segment(data, indices, segment_ids, num_segments, mode):
    if num_segments is None:
        num_segments = int(segment_ids.max().item()) + 1 if segment_ids.numel() else 0
    if _native.on_device(data):
        return _SparseSegment.apply(data, indices.contiguous().long(), segment_ids.contiguous().long(), int(num_segments), _MODES[mode])
    return _segment_ref(data, indices.long(), segment_ids.long(), int(num_segments), mode)


def sparse_segment_sum(data: torch.Tensor, indices: torch.Tensor, segment_ids: torch.Tensor, num_segments: Optional[int] = None) -> torch.Tensor:
    """``tf.sparse.segment_sum``: ``out[s] = sum_{i: segment_ids[i] == s} data[indices[i]]`` (segment ids sorted ascending); differentiable in ``data``."""
    return _sparse_segment(data, indices, segment_ids, num_segments, "sum")


def sparse_segment_mean(data, indices, segment_ids, num_segments: Optional[int] = None) -> torch.Tensor:
    return _sparse_segment(data, indices, segment_ids, num_segments, "mean")


def sparse_segment_sqrt_n(data, indices, segment_ids, num_segments: Optional[int] = None) -> torch.Tensor:
    return _sparse_segment(data, indices, segment_ids, num_segments, "sqrtn")
