"""Unique-first model-parallel embedding pipeline (csrc/cuda/sparse_pipeline.cu) -- Python side.

One :class:`SparsePipeline` per engine owns the requester-side state (dedup scratch, inverse index, per-owner bucket
lists, unique-row / unique-gradient buffers) and the owner-side state (positions and slots of the keys received from every
source).  With ``world > 1`` the peer-visible buffers are CUDA-IPC symmetric allocations (:class:`parallel.p2p.P2PComm`) and
the kernels read / write them over NVLink; with ``world == 1`` the very same kernels run on plain device tensors.

Dataflow replaced: ``unique`` before every EV lookup / apply (python/training/optimizer.py:91, unique_ali_op_gpu.cu.cc) and SOK's
three NCCL all-to-alls (all2all_input_dispatcher.cu:227-285, all2all_output_dispatcher.cu:159-246).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import torch

from .. import _native
from .._cuda_sigs import Peers, SpBags, SpGeom, SpSync
from .._native import check, ptr, stream_ptr

vp = C.c_void_p
CH_DEDUP, CH_ROWS, CH_GRAD, CH_DENSE = 0, 1, 2, 3


MAX_TABLES = 256          # kSpMaxTables in csrc/cuda/sparse_pipeline.cu


COMBINERS = {"sum": 0, "mean": 1, "sqrtn": 2}


class Bags:
    """Multi-hot bags over the id columns: ``bags`` lists ``(n_cols, combiner)`` in column order, bag f pools the next ``n_cols`` columns into
    activation slot f with ``sum | mean | sqrtn`` (padding neither adds nor counts).  The geometry lives in device tensors, built once."""

    def __init__(self, dev: torch.device, bags: Sequence[tuple], num_cols: int):
        bags = [(int(n), str(c)) for n, c in bags]
        if not bags:
            raise ValueError("bags: at least one bag")
        for n, c in bags:
            if n < 1:
                raise ValueError(f"bags: a bag needs at least one id column, got {n}")
            if c not in COMBINERS:
                raise ValueError(f"bags: combiner must be one of {'|'.join(COMBINERS)}, got {c!r}")
        if sum(n for n, _ in bags) != num_cols:
            raise ValueError(f"bags: the column counts sum to {sum(n for n, _ in bags)}, the engine has {num_cols} id columns")
        off = [0]
        for n, _ in bags:
            off.append(off[-1] + n)
        self.F, self.spec = len(bags), bags
        self.off = torch.tensor(off, dtype=torch.int32, device=dev)
        self.comb = torch.tensor([COMBINERS[c] for _, c in bags], dtype=torch.int32, device=dev)
        self.col_bag = torch.tensor([f for f, (n, _) in enumerate(bags) for _ in range(n)], dtype=torch.int32, device=dev)
        s = SpBags()
        s.off, s.comb, s.col_bag, s.F = self.off.data_ptr(), self.comb.data_ptr(), self.col_bag.data_ptr(), self.F
        self.struct = s

    def ref(self):
        return C.byref(self.struct)


def _next_pow2(n: int) -> int:
    p = 1
    while p < n:
        p <<= 1
    return p


class _LocalBuffer:
    """world == 1 stand-in for parallel.p2p.SymmetricBuffer: a plain device allocation that is its own (only) peer."""

    def __init__(self, dev: torch.device, nbytes: int):
        self._raw = torch.zeros(max(16, nbytes), dtype=torch.uint8, device=dev)
        self.nbytes = nbytes
        self.local = self._raw.data_ptr()
        self.peers = Peers()
        self.peers.ptr[0] = self.local

    def tensor(self, dtype: torch.dtype, shape) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= s
        nb = n * torch.empty((), dtype=dtype).element_size()
        assert nb <= max(16, self.nbytes)
        return self._raw[:nb].view(dtype).view(*shape)

    def peers_ref(self):
        return C.byref(self.peers)


class SparsePipeline:
    def __init__(self, dev: torch.device, rank: int, world: int, col_table: Sequence[int], num_tables: int, batch: int, dim: int, comm=None,
                 pad_key: int = -1, with_grad: bool = True):
        self.dev, self.rank, self.W, self.comm = dev, rank, world, comm
        self.lib = _native.cuda()
        self.C, self.T, self.B, self.dim = len(col_table), num_tables, batch, dim
        self.ldinv = (self.C + 3) // 4 * 4
        if world > 1 and comm is None:
            raise ValueError("world > 1 needs a P2PComm for the symmetric buffers")
        # limits of the kernels (csrc/cuda/sparse_pipeline.cu): per-peer pointer tables hold 16 ranks (one NVSwitch domain of 8 today), the per-table
        # chunk prefix lives in shared memory, rows move as 8-byte bf16 groups
        if world > 16:
            raise ValueError(f"SparsePipeline: world size {world} > 16 ranks of one peer-memory domain")
        if num_tables > MAX_TABLES:
            raise ValueError(f"SparsePipeline: {num_tables} tables > {MAX_TABLES}; merge small tables (PartitionedEmbeddingVariable / one table with a feature-id prefix)")
        if dim % 4 or dim <= 0:
            raise ValueError(f"SparsePipeline: embedding dim {dim} must be a positive multiple of 4")
        if any(t < 0 or t >= num_tables for t in col_table):
            raise ValueError("SparsePipeline: col_table entry outside [0, num_tables)")
        ncols = [0] * num_tables
        for t in col_table:
            ncols[t] += 1
        hoff, boff = [0], [0]
        for t in range(num_tables):
            n = max(1, ncols[t]) * batch
            hoff.append(hoff[-1] + _next_pow2(2 * n))
            boff.append(boff[-1] + n)
        self.Htot, self.Btot = hoff[-1], boff[-1]
        self.max_bcap = max(b - a for a, b in zip(boff[:-1], boff[1:]))
        if self.Htot >= (1 << 31):
            raise ValueError("dedup scratch exceeds int32 indexing; lower the batch size")
        i32t, i64t = torch.int32, torch.int64
        self.col_table = torch.tensor(list(col_table), dtype=i32t, device=dev)
        self.hoff = torch.tensor(hoff, dtype=i64t, device=dev)
        self.boff = torch.tensor(boff, dtype=i64t, device=dev)
        g = SpGeom()
        g.col_table, g.hoff, g.boff = self.col_table.data_ptr(), self.hoff.data_ptr(), self.boff.data_ptr()
        g.C, g.T, g.W, g.rank, g.B, g.dim, g.ldinv, g.pad_key = self.C, num_tables, world, rank, batch, dim, self.ldinv, pad_key
        self.geom = g
        sym = (lambda nb: comm.symmetric(nb)) if world > 1 else (lambda nb: _LocalBuffer(dev, nb))
        # ---- peer-visible (requester side)
        self.scr_buf = sym(self.Htot * 16)
        self.urow_buf = sym(self.Htot * dim * 2)
        self.ugrad_buf = sym(self.Htot * dim * 8) if with_grad else None       # int64 fixed point (csrc/cuda/sparse_pipeline.cu)
        self.bkt_key_buf = sym(self.Btot * world * 8)
        self.bkt_gs_buf = sym(self.Btot * world * 4)
        self.bcnt_buf = sym(max(64, num_tables * world) * 4)
        self.flags_buf = sym(8 * 16 * 4)
        self.urow = self.urow_buf.tensor(torch.bfloat16, (self.Htot, dim))
        self.ugrad = self.ugrad_buf.tensor(torch.int64, (self.Htot, dim)) if with_grad else None
        self.bcnt = self.bcnt_buf.tensor(i32t, (num_tables, world))
        # ---- local
        self.state = torch.zeros(16, dtype=i32t, device=dev)
        self.inv = torch.full((batch, self.ldinv), -1, dtype=i32t, device=dev)          # [B][ldinv]: sample-major (interaction gathers)
        self.invT = torch.full((self.C, batch), -1, dtype=i32t, device=dev) if with_grad else None   # [C][B]: column-major (segment-sum)
        self.own_pos = torch.zeros(self.Btot * world, dtype=i32t, device=dev)
        self.own_gs = torch.zeros(self.Btot * world, dtype=i32t, device=dev)
        self.own_cnt = torch.zeros(num_tables * world, dtype=i32t, device=dev)
        self._stats = torch.zeros(2, dtype=i64t, device=dev)
        s = SpSync()
        s.flags, s.state, s.rank, s.W = self.flags_buf.peers, self.state.data_ptr(), rank, world
        self.sync = s
        check(self.lib.dr_sp_init_scratch(vp(self.scr_buf.local), self.Htot, stream_ptr(self.dev)), "init_scratch")
        if not _native.emu_active():
            torch.cuda.synchronize(dev)
        if world > 1:
            comm.host_barrier()
        self.launches = 0

    # ------------------------------------------------------------------------------------------------------------------
    def sync_ref(self):
        return C.byref(self.sync)

    def geom_ref(self):
        return C.byref(self.geom)

    def dedup(self, ids: torch.Tensor) -> None:
        """ids: int64 [C, B] (column-major id columns of the local batch)."""
        assert ids.shape == (self.C, self.B) and ids.dtype == torch.int64
        check(self.lib.dr_sp_dedup(ptr(ids), self.geom_ref(), vp(self.scr_buf.local), ptr(self.inv), ptr(self.invT), vp(self.bkt_key_buf.local), vp(self.bkt_gs_buf.local),
                                   vp(self.bcnt_buf.local), ptr(self.ugrad) if self.ugrad is not None else None, self.sync_ref(), stream_ptr(self.dev)), "dedup")
        self.launches += 1

    def lookup(self, ctx, table_map: torch.Tensor, train: bool) -> None:
        """Owner side: probe / insert the keys every source bucketed for this rank and push their rows into the sources' urow."""
        check(self.lib.dr_sp_lookup(ptr(ctx.structs()), ptr(table_map), self.geom_ref(), self.max_bcap, self.bkt_key_buf.peers_ref(),
                                    self.bkt_gs_buf.peers_ref(), self.bcnt_buf.peers_ref(), self.scr_buf.peers_ref(), self.urow_buf.peers_ref(),
                                    int(train), ptr(self.own_pos), ptr(self.own_gs), ptr(self.own_cnt),
                                    ptr(ctx.ulist) if train else None, ptr(ctx.nuniq) if train else None,
                                    ctx.ulist.numel() if train else 0, self.sync_ref(), stream_ptr(self.dev)), "lookup")
        self.launches += 1

    def gather(self, out: torch.Tensor) -> None:
        """Requester side: out[b, c, :] = urow[inv[b, c]] (bf16 [B, C, dim]); the kernel waits for every owner's ROWS flag."""
        assert out.shape == (self.B, self.C, self.dim) and out.dtype == torch.bfloat16 and out.is_contiguous()
        check(self.lib.dr_sp_gather(ptr(self.urow), ptr(self.inv), self.geom_ref(), ptr(out), self.sync_ref(), stream_ptr(self.dev)), "gather")
        self.launches += 1

    def gather_pitched(self, out: torch.Tensor) -> None:
        """gather into the first C * dim columns of a wider row: out[b, c * dim: (c + 1) * dim] = urow[inv[b, c]] (out: a bf16 [B, >= C * dim]
        view whose rows may be longer, e.g. the embedding columns of DLRM-DCNv2's x0)."""
        assert out.dim() == 2 and out.shape[0] == self.B and out.shape[1] >= self.C * self.dim and out.dtype == torch.bfloat16 and out.stride(1) == 1
        check(self.lib.dr_sp_gather_pitched(ptr(self.urow), ptr(self.inv), self.geom_ref(), C.c_void_p(out.data_ptr()), out.stride(0),
                                            self.sync_ref(), stream_ptr(self.dev)), "gather_pitched")
        self.launches += 1

    def segsum(self, demb: torch.Tensor) -> None:
        """Requester side: pre-reduce the per-sample gradient rows (bf16 [C, B, dim]) per distinct key into ugrad; raises GRAD."""
        assert demb.shape == (self.C, self.B, self.dim) and demb.dtype == torch.bfloat16
        check(self.lib.dr_sp_segsum(ptr(demb), ptr(self.invT), self.geom_ref(), ptr(self.ugrad), self.sync_ref(), stream_ptr(self.dev)), "segsum")
        self.launches += 1

    def pool(self, out: torch.Tensor, w: torch.Tensor, bags: Bags) -> None:
        """Requester side: out[b, f, :] = w[f, b] * sum of the live rows urow[inv[b, c]] of bag f (bf16 [B, F, dim], fp32 sum in column order);
        w (fp32 [F, B]) = 1, 1/n or 1/sqrt(n) over the bag's n live ids, 0 for an empty bag.  Takes the place of gather; waits for ROWS."""
        assert out.shape == (self.B, bags.F, self.dim) and out.dtype == torch.bfloat16 and out.is_contiguous()
        assert w.shape == (bags.F, self.B) and w.dtype == torch.float32 and w.is_contiguous()
        assert bags.col_bag.numel() == self.C
        check(self.lib.dr_sp_pool(ptr(self.urow), ptr(self.inv), self.geom_ref(), bags.ref(), ptr(out), ptr(w), self.sync_ref(), stream_ptr(self.dev)), "pool")
        self.launches += 1

    def pool_segsum(self, dpool: torch.Tensor, w: torch.Tensor, bags: Bags) -> None:
        """Requester side: segsum of the pooled bags' gradient (bf16 [F, B, dim]): every live column c of sample b adds dpool[bag(c), b] *
        w[bag(c), b] to the per-key sums in ugrad; raises GRAD.  Takes the place of segsum."""
        assert dpool.shape == (bags.F, self.B, self.dim) and dpool.dtype == torch.bfloat16 and dpool.is_contiguous()
        assert w.shape == (bags.F, self.B) and w.dtype == torch.float32 and w.is_contiguous()
        assert bags.col_bag.numel() == self.C and self.ugrad is not None
        check(self.lib.dr_sp_pool_segsum(ptr(dpool), ptr(w), ptr(self.invT), self.geom_ref(), bags.ref(), ptr(self.ugrad), self.sync_ref(), stream_ptr(self.dev)),
              "pool_segsum")
        self.launches += 1

    def linear_fwd(self, out: torch.Tensor) -> None:
        """Requester side: out[b] = sum over the id columns c of float(urow[inv[b, c], 0]) (fp32 [B], summed in column order); padding adds
        nothing.  The linear (wide) logit read in place from the unique rows; the kernel waits for every owner's ROWS flag."""
        assert out.shape == (self.B,) and out.dtype == torch.float32 and out.is_contiguous()
        check(self.lib.dr_sp_linear_fwd(ptr(self.urow), ptr(self.inv), self.geom_ref(), ptr(out), self.sync_ref(), stream_ptr(self.dev)), "linear_fwd")
        self.launches += 1

    def linear_bwd(self, dlogit: torch.Tensor) -> None:
        """Requester side: add the fp32 gradient of every sample's linear logit to element 0 of ugrad[inv[b, c]] for every live id (exact
        64-bit fixed-point sums, elements 1.. stay zero); raises GRAD.  Takes the place of segsum for a linear group."""
        assert dlogit.shape == (self.B,) and dlogit.dtype == torch.float32 and dlogit.is_contiguous()
        assert self.ugrad is not None, "linear_bwd needs a pipeline built with with_grad=True"
        check(self.lib.dr_sp_linear_bwd(ptr(dlogit), ptr(self.invT), self.geom_ref(), ptr(self.ugrad), self.sync_ref(), stream_ptr(self.dev)), "linear_bwd")
        self.launches += 1

    def ugrad_rows(self) -> torch.Tensor:
        """The pre-reduced per-key gradient rows as fp32 (ugrad holds them in 64-bit fixed point, units of 2^-40)."""
        return (self.ugrad.double() * 2.0 ** -40).float()

    def grad(self, ctx, table_map: torch.Tensor) -> None:
        """Owner side: pull the sources' pre-reduced gradient rows into gsum[unique] (k_apply follows)."""
        check(self.lib.dr_sp_grad(ptr(ctx.structs()), ptr(table_map), self.geom_ref(), self.max_bcap, self.ugrad_buf.peers_ref(), ptr(self.own_pos),
                                  ptr(self.own_gs), ptr(self.own_cnt), ptr(ctx.gsum), self.sync_ref(), stream_ptr(self.dev)), "grad")
        self.launches += 1

    def reset(self) -> None:
        check(self.lib.dr_sp_reset(self.geom_ref(), self.max_bcap, vp(self.scr_buf.local), vp(self.bkt_gs_buf.local), vp(self.bcnt_buf.local),
                                   ptr(self.state), stream_ptr(self.dev)), "reset")
        self.launches += 1

    def signal(self, channel: int) -> None:
        check(self.lib.dr_sp_signal(self.sync_ref(), channel, stream_ptr(self.dev)), "signal")
        self.launches += 1

    def step_end(self) -> None:
        check(self.lib.dr_sp_step_end(ptr(self.state), stream_ptr(self.dev)), "step_end")
        self.launches += 1

    def unique_count(self) -> int:
        """Distinct (table, key) pairs of the batch last deduplicated (valid between dedup() and reset(); host sync)."""
        check(self.lib.dr_sp_stats(self.geom_ref(), vp(self.bcnt_buf.local), ptr(self._stats), stream_ptr(self.dev)), "stats")
        return int(self._stats[0].item())
