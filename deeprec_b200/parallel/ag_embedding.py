"""All-gather -> lookup -> reduce-scatter model-parallel embedding over peer memory (``csrc/cuda/ag_embedding.cu``) -- the fused-kernel form of SOK
v1's ``DistributedEmbedding`` dataflow (SURVEY 2.15 C5 / C6: 3 x ncclAllGather of the ids, local lookup + partial combine, ncclReduceScatter of the
partial sums, ncclAllGather of the top gradients in the backward).  No gathered copy of the ids exists: owners read every peer's list in place,
requesters pull and sum the owners' partial rows, owners pull the top gradients -- all synchronised by the in-kernel flags of ``sp_sync.cuh``.

One :class:`AllGatherEmbedding` per (table, rank).  Per step::

    ag.load_ids(values, row_ids)        # this rank's sparse batch: key + sample index per entry
    ag.lookup(ctx, train=True)          # owner side: every rank's entries that hash to me
    out = ag.reduce(combiner="mean")    # requester side: [B, D] combined embeddings of MY samples
    ...dense forward / backward...
    ag.stage_grad(dout)                 # top gradients of my samples
    ag.grad(ctx); ctx.apply(...)        # owner side: per-key gradient sums -> row optimizer
    ag.step_end()

``parallel/sok.py::DistributedEmbedding`` keeps the module-level NCCL form (any device / backend); the engines use the unique-first pipeline
(``parallel/sparse_pipeline.py``), which moves strictly less data for one-hot columns."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from .. import _native
from .._cuda_sigs import AgGeom, AgPeers, SpSync
from .._native import check, ptr, stream_ptr
from .sparse_pipeline import _LocalBuffer

CH_IDS, CH_ROWS, CH_GRAD, CH_DONE = 0, 1, 2, 4


class AllGatherEmbedding:
    def __init__(self, dev: torch.device, rank: int, world: int, table, batch: int, nnz_cap: int, comm=None):
        """``table``: this rank's shard (a :class:`ops.device_table.DeviceTable` registered in a StepContext); ``nnz_cap``: most entries a rank's
        batch may have; ``comm``: :class:`parallel.p2p.P2PComm` (or the emulation's ``EmuComm``) when ``world > 1``."""
        if world > 1 and comm is None:
            raise ValueError("world > 1 needs a communicator for the symmetric buffers")
        if world > 16:
            raise ValueError("one peer-memory domain: at most 16 ranks")
        self.dev, self.rank, self.W, self.table, self.B, self.D, self.nnz_cap = dev, rank, world, table, int(batch), int(table.dim), int(nnz_cap)
        self.lib = _native.cuda()
        sym = (lambda nb: comm.symmetric(nb)) if world > 1 else (lambda nb: _LocalBuffer(dev, nb))
        self.keys_buf, self.rows_buf, self.meta_buf = sym(self.nnz_cap * 8), sym(self.nnz_cap * 4), sym(64)
        self.partial_buf, self.grad_buf, self.flags_buf = sym(world * self.B * self.D * 4), sym(self.B * self.D * 4), sym(8 * 16 * 4)
        self.keys = self.keys_buf.tensor(torch.int64, (self.nnz_cap,))
        self.rows = self.rows_buf.tensor(torch.int32, (self.nnz_cap,))
        self.meta = self.meta_buf.tensor(torch.int32, (4,))
        self.grad_stage = self.grad_buf.tensor(torch.float32, (self.B, self.D))
        p = AgPeers()
        p.keys, p.rows, p.meta, p.partial, p.grad = self.keys_buf.peers, self.rows_buf.peers, self.meta_buf.peers, self.partial_buf.peers, self.grad_buf.peers
        self.peers = p
        g = AgGeom()
        g.W, g.rank, g.dim, g.table_index, g.B, g.nnz_cap = world, rank, self.D, int(table.gid), self.B, self.nnz_cap
        self.geom = g
        self.state = torch.zeros(16, dtype=torch.int32, device=dev)
        s = SpSync()
        s.flags, s.state, s.rank, s.W = self.flags_buf.peers, self.state.data_ptr(), rank, world
        self.sync = s
        self.own_pos = torch.zeros(world * self.nnz_cap, dtype=torch.int32, device=dev)
        self.own_row = torch.zeros(world * self.nnz_cap, dtype=torch.int32, device=dev)
        self.own_cnt = torch.zeros(world, dtype=torch.int32, device=dev)
        self._scale: Optional[torch.Tensor] = None
        if world > 1:
            comm.host_barrier()

    def _signal(self, ch: int) -> None:
        check(self.lib.dr_sp_signal(C.byref(self.sync), ch, stream_ptr(self.dev)), "signal")

    # ---- requester side -------------------------------------------------------------------------------------------------------------------
    def load_ids(self, values: torch.Tensor, row_ids: torch.Tensor) -> None:
        """Stage this rank's sparse batch (``values`` int64 keys, ``row_ids`` sample index of every entry) where the owners read it."""
        n = int(values.numel())
        if n > self.nnz_cap:
            raise ValueError(f"{n} entries > nnz_cap {self.nnz_cap}")
        self.keys[:n].copy_(values.reshape(-1)); self.rows[:n].copy_(row_ids.reshape(-1).to(torch.int32))
        self.meta[0] = n
        self._rows_now = row_ids.reshape(-1)
        self._signal(CH_IDS)

    def reduce(self, combiner: str = "sum") -> torch.Tensor:
        """[B, D] fp32: for every sample of this rank the combined rows of its entries (pulled from all owners' partial sums)."""
        self._scale = None
        if combiner != "sum":
            cnt = torch.bincount(self._rows_now.to(torch.int64), minlength=self.B).clamp(min=1).to(torch.float32)
            self._scale = (1.0 / cnt if combiner == "mean" else cnt.rsqrt()).to(self.dev).contiguous()
        out = torch.empty(self.B, self.D, dtype=torch.float32, device=self.dev)
        check(self.lib.dr_ag_reduce(C.byref(self.geom), C.byref(self.peers), ptr(self._scale), ptr(out), C.byref(self.sync), stream_ptr(self.dev)), "reduce")
        return out

    def stage_grad(self, dout: torch.Tensor) -> None:
        """Top gradients [B, D] of this rank's samples (scaled by the combiner here, so that owners add them as they are)."""
        g = dout.to(torch.float32)
        if self._scale is not None:
            g = g * self._scale.unsqueeze(1)
        self.grad_stage.copy_(g)
        self._signal(CH_GRAD)

    # ---- owner side -----------------------------------------------------------------------------------------------------------------------
    def lookup(self, ctx, train: bool) -> None:
        if train:
            ctx.ensure(self.W * self.nnz_cap)
        check(self.lib.dr_ag_lookup(ptr(ctx.structs()), C.byref(self.geom), C.byref(self.peers), int(train), ptr(self.own_pos), ptr(self.own_row), ptr(self.own_cnt),
                                    ptr(ctx.ulist) if train else None, ptr(ctx.nuniq) if train else None, ctx.ulist.numel() if train else 0, C.byref(self.sync), stream_ptr(self.dev)),
              "lookup")

    def grad(self, ctx) -> None:
        check(self.lib.dr_ag_grad(ptr(ctx.structs()), C.byref(self.geom), C.byref(self.peers), ptr(self.own_pos), ptr(self.own_row), ptr(self.own_cnt), ptr(ctx.gsum),
                                  ctx.ulist.numel(), C.byref(self.sync), stream_ptr(self.dev)), "grad")

    def step_end(self) -> None:
        check(self.lib.dr_sp_step_end(ptr(self.state), stream_ptr(self.dev)), "step_end")
