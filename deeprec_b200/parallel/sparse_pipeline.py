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
from .._native import ptr

vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
CH_DEDUP, CH_ROWS, CH_GRAD, CH_DENSE = 0, 1, 2, 3


MAX_TABLES = 256          # kSpMaxTables in csrc/cuda/sparse_pipeline.cu


class Peers(C.Structure):
    """Mirror of DrPeers (csrc/cuda/sp_sync.cuh)."""
    _fields_ = [("ptr", vp * 16)]


class SpSync(C.Structure):
    """Mirror of DrSpSync."""
    _fields_ = [("flags", Peers), ("state", vp), ("rank", i32), ("W", i32)]


class SpGeom(C.Structure):
    """Mirror of DrSpGeom."""
    _fields_ = [("col_table", vp), ("hoff", vp), ("boff", vp), ("C", i32), ("T", i32), ("W", i32), ("rank", i32), ("B", i64),
                ("dim", i32), ("ldinv", i32), ("pad_key", i64)]


def _next_pow2(n: int) -> int:
    p = 1
    while p < n:
        p <<= 1
    return p


def _chk(rc, what):
    if rc != 0:
        raise RuntimeError(f"deeprec_cuda sparse pipeline: {what} failed with code {rc}")


def bind(lib):
    if getattr(lib, "_sp_bound", False):
        return lib
    INT, P = C.c_int, vp
    GP, SP, PP = C.POINTER(SpGeom), C.POINTER(SpSync), C.POINTER(Peers)
    sigs = {
        "dr_sp_init_scratch": [P, i64, P],
        "dr_sp_dedup": [P, GP, P, P, P, P, P, P, P, SP, P],
        "dr_sp_segsum": [P, P, GP, P, SP, P],
        "dr_sp_gather": [P, P, GP, P, SP, P],
        "dr_sp_lookup": [P, P, GP, i64, PP, PP, PP, PP, PP, INT, P, P, P, P, P, i64, SP, P],
        "dr_sp_grad": [P, P, GP, i64, PP, P, P, P, P, SP, P],
        "dr_sp_reset": [GP, i64, P, P, P, P, P],
        "dr_sp_signal": [SP, INT, P],
        "dr_sp_step_end": [P, P],
        "dr_sp_stats": [GP, P, P, P],
        "dr_cuda_dot_interaction_fwd_u": [P, i64, P, P, INT, INT, INT, i64, P, i64, SP, P],
        "dr_cuda_dot_interaction_bwd_u": [P, i64, P, i64, P, P, INT, INT, INT, i64, P, i64, P, i64, i64, P],
        "dr_cuda_dlrm_inter_gemm": [P, i64, P, P, INT, INT, INT, i64, P, i64, INT, P, P, i64, P, i64, SP, P],
        "dr_comm_allreduce_apply_sync": [PP, INT, P, P, P, i64, P, P, SP, P],
    }
    for name, args in sigs.items():
        if not hasattr(lib, name) and _native.emu_active():
            continue                             # wgmma translation units are not part of the emulation build
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, INT
    lib._sp_bound = True
    return lib


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
        self.lib = bind(_native.cuda())
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
        _chk(self.lib.dr_sp_init_scratch(vp(self.scr_buf.local), self.Htot, self._s()), "init_scratch")
        if not _native.emu_active():
            torch.cuda.synchronize(dev)
        if world > 1:
            comm.host_barrier()
        self.launches = 0

    # ------------------------------------------------------------------------------------------------------------------
    def _s(self):
        if _native.emu_active():
            return None
        return vp(torch.cuda.current_stream(self.dev).cuda_stream)

    def sync_ref(self):
        return C.byref(self.sync)

    def geom_ref(self):
        return C.byref(self.geom)

    def dedup(self, ids: torch.Tensor) -> None:
        """ids: int64 [C, B] (column-major id columns of the local batch)."""
        assert ids.shape == (self.C, self.B) and ids.dtype == torch.int64
        _chk(self.lib.dr_sp_dedup(ptr(ids), self.geom_ref(), vp(self.scr_buf.local), ptr(self.inv), ptr(self.invT), vp(self.bkt_key_buf.local), vp(self.bkt_gs_buf.local),
                                  vp(self.bcnt_buf.local), ptr(self.ugrad) if self.ugrad is not None else None, self.sync_ref(), self._s()), "dedup")
        self.launches += 1

    def lookup(self, ctx, table_map: torch.Tensor, train: bool) -> None:
        """Owner side: probe / insert the keys every source bucketed for this rank and push their rows into the sources' urow."""
        _chk(self.lib.dr_sp_lookup(ptr(ctx.structs()), ptr(table_map), self.geom_ref(), self.max_bcap, self.bkt_key_buf.peers_ref(),
                                   self.bkt_gs_buf.peers_ref(), self.bcnt_buf.peers_ref(), self.scr_buf.peers_ref(), self.urow_buf.peers_ref(),
                                   int(train), ptr(self.own_pos), ptr(self.own_gs), ptr(self.own_cnt),
                                   ptr(ctx.ulist) if train else None, ptr(ctx.nuniq) if train else None,
                                   ctx.ulist.numel() if train else 0, self.sync_ref(), self._s()), "lookup")
        self.launches += 1

    def gather(self, out: torch.Tensor) -> None:
        """Requester side: out[b, c, :] = urow[inv[b, c]] (bf16 [B, C, dim]); the kernel waits for every owner's ROWS flag."""
        assert out.shape == (self.B, self.C, self.dim) and out.dtype == torch.bfloat16 and out.is_contiguous()
        _chk(self.lib.dr_sp_gather(ptr(self.urow), ptr(self.inv), self.geom_ref(), ptr(out), self.sync_ref(), self._s()), "gather")
        self.launches += 1

    def segsum(self, demb: torch.Tensor) -> None:
        """Requester side: pre-reduce the per-sample gradient rows (bf16 [C, B, dim]) per distinct key into ugrad; raises GRAD."""
        assert demb.shape == (self.C, self.B, self.dim) and demb.dtype == torch.bfloat16
        _chk(self.lib.dr_sp_segsum(ptr(demb), ptr(self.invT), self.geom_ref(), ptr(self.ugrad), self.sync_ref(), self._s()), "segsum")
        self.launches += 1

    def ugrad_rows(self) -> torch.Tensor:
        """The pre-reduced per-key gradient rows as fp32 (ugrad holds them in 64-bit fixed point, units of 2^-40)."""
        return (self.ugrad.double() * 2.0 ** -40).float()

    def grad(self, ctx, table_map: torch.Tensor) -> None:
        """Owner side: pull the sources' pre-reduced gradient rows into gsum[unique] (k_apply follows)."""
        _chk(self.lib.dr_sp_grad(ptr(ctx.structs()), ptr(table_map), self.geom_ref(), self.max_bcap, self.ugrad_buf.peers_ref(), ptr(self.own_pos),
                                 ptr(self.own_gs), ptr(self.own_cnt), ptr(ctx.gsum), self.sync_ref(), self._s()), "grad")
        self.launches += 1

    def reset(self) -> None:
        _chk(self.lib.dr_sp_reset(self.geom_ref(), self.max_bcap, vp(self.scr_buf.local), vp(self.bkt_gs_buf.local), vp(self.bcnt_buf.local),
                                  ptr(self.state), self._s()), "reset")
        self.launches += 1

    def signal(self, channel: int) -> None:
        _chk(self.lib.dr_sp_signal(self.sync_ref(), channel, self._s()), "signal")
        self.launches += 1

    def step_end(self) -> None:
        _chk(self.lib.dr_sp_step_end(ptr(self.state), self._s()), "step_end")
        self.launches += 1

    def unique_count(self) -> int:
        """Distinct (table, key) pairs of the batch last deduplicated (valid between dedup() and reset(); host sync)."""
        _chk(self.lib.dr_sp_stats(self.geom_ref(), vp(self.bcnt_buf.local), ptr(self._stats), self._s()), "stats")
        return int(self._stats[0].item())
