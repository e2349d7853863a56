"""Device-resident EmbeddingVariable storage (HBM tier) and the fused multi-table lookup.

Python owns the buffers (torch tensors, so HBM goes through one allocator); the sm_90a kernels in
csrc/cuda/{table,embedding,optimizer}_kernels.cu receive POD ``DrDeviceTable`` descriptors.
Parity: GPUHashTable / GPUHashMapKV / HbmStorage (framework/embedding/gpu_hash_table.h:33-133,
gpu_hash_map_kv.h:29-340, single_tier_storage.h HbmStorage) and the GPU Kv* ops
(kv_variable_lookup_ops.cc:255-305, training_ali_ops.cc:214,690,1578,2547,3207).

Dedup design: every table belongs to a :class:`StepContext` (one per device x dim x optimizer).
The training forward claims a per-step unique index for each touched key inside the probe kernel;
the backward scatter-adds gradients into ``gsum[unique]``; ``apply_step`` runs ONE fused
admit/allocate/initialise/update kernel over all tables of the context.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional

import torch

from .. import _native
from .._cuda_sigs import DeviceTableStruct
from .._native import EvConfig, OptHyper, ptr, stream_ptr

EMPTY_KEY = -(1 << 63)
_COMB = {"sum": 0, "mean": 1, "sqrtn": 2}


def _next_pow2(n: int) -> int:
    p = 1
    while p < n:
        p <<= 1
    return p


def _chk(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"deeprec_cuda: {what} failed with code {rc}")


class StepContext:
    """Per-step dedup state shared by all device tables of one (device, dim, owner)."""

    def __init__(self, device: torch.device, dim: int):
        self.device, self.dim = device, dim
        self.lib = _native.cuda()
        self.tables: List["DeviceTable"] = []
        self.struct_all = None
        self._ptrs = None
        self.ulist = None
        self.gsum = None
        self.nuniq = torch.zeros(1, dtype=torch.int32, device=device)
        self.claimed_upper = 0
        self.pending = False
        # hyper-parameters + step live in device memory so captured graphs read live values
        self.hp_dev = torch.zeros(C.sizeof(OptHyper), dtype=torch.uint8, device=device)
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=device)

    def set_hyper(self, hp: OptHyper) -> None:
        self.hp_dev.copy_(torch.frombuffer(bytearray(bytes(hp)), dtype=torch.uint8), non_blocking=True)

    def set_step(self, step: int) -> None:
        self.step_dev.fill_(int(step))

    def register(self, t: "DeviceTable") -> int:
        self.tables.append(t)
        self._ptrs = None
        return len(self.tables) - 1

    def unregister(self, t: "DeviceTable") -> None:
        # keep indices stable: replace by a tombstone (never referenced by new lookups)
        for i, x in enumerate(self.tables):
            if x is t:
                self.tables[i] = None
        self._ptrs = None

    def structs(self) -> torch.Tensor:
        ptrs = tuple(t.struct_version if t is not None else -1 for t in self.tables)
        if ptrs != self._ptrs or self.struct_all is None:
            size = C.sizeof(DeviceTableStruct)
            parts = [t.struct_dev if t is not None else torch.zeros(size, dtype=torch.uint8, device=self.device) for t in self.tables]
            new = torch.cat(parts).contiguous()
            if self.struct_all is not None and self.struct_all.numel() == new.numel():
                self.struct_all.copy_(new)        # IN PLACE: a captured CUDA graph holds this buffer's address (tables re-hash / grow at step boundaries)
            else:
                self.struct_all = new
            self._ptrs = ptrs
        return self.struct_all

    def ensure(self, n: int) -> None:
        need = self.claimed_upper + n
        cap = 0 if self.ulist is None else self.ulist.numel()
        if need > cap:
            new_cap = max(1 << 16, _next_pow2(need))
            ul = torch.zeros(new_cap, dtype=torch.int64, device=self.device)
            gs = torch.zeros(new_cap, self.dim, dtype=torch.float32, device=self.device)
            if self.ulist is not None and self.pending:
                ul[:cap].copy_(self.ulist)
                gs[:cap].copy_(self.gsum)
            self.ulist, self.gsum = ul, gs
        self.claimed_upper = need

    def apply_step(self, hp: OptHyper) -> None:
        if not self.pending:
            return
        self.set_hyper(hp)
        _chk(self.lib.dr_cuda_sparse_apply(ptr(self.structs()), ptr(self.ulist), ptr(self.nuniq), self.ulist.numel(), ptr(self.gsum),
                                           self.dim, ptr(self.hp_dev), self.claimed_upper, 1, stream_ptr()), "sparse_apply")
        self.pending = False
        self.claimed_upper = 0


_CONTEXTS: Dict[tuple, StepContext] = {}


def get_context(device: torch.device, dim: int, owner: int = 0) -> StepContext:
    key = (str(device), dim, owner)
    c = _CONTEXTS.get(key)
    if c is None:
        c = _CONTEXTS[key] = StepContext(device, dim)
    return c


class DeviceTable:
    def __init__(self, cfg: EvConfig, default_matrix: torch.Tensor, device: torch.device,
                 capacity: Optional[int] = None, row_capacity: Optional[int] = None, owner: int = 0):
        self.lib = _native.cuda()
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        if self.device.type == "cuda":
            _native.set_device(self.device.index)
        elif not _native.emu_active():
            raise ValueError("DeviceTable lives on a CUDA device (CPU tensors only inside _native.cuda_emulation())")
        self.dim = int(cfg.dim)
        if self.dim % 4:
            raise ValueError("device EmbeddingVariable needs embedding_dim % 4 == 0")
        self.num_slots = int(cfg.num_slots)
        self.stride = (self.dim * (1 + self.num_slots) + (4 if cfg.has_scalars else 0) + 3) // 4 * 4
        self.default_matrix = default_matrix.to(self.device, torch.float32).contiguous()
        cap = capacity or _next_pow2(max(1024, 2 * int(cfg.init_capacity)))
        self.bloom = None
        self.bloom_k = 0
        if cfg.filter_type == 2:
            p, n = float(cfg.bloom_fpp), int(cfg.bloom_max_elements)
            self.bloom_k = max(1, math.ceil(math.log2(1.0 / p)))
            m = max(8, math.ceil(n * abs(math.log(p)) / (math.log(2.0) ** 2)))
            self.bloom = torch.zeros(m, dtype=torch.int32, device=self.device)
        self.struct_version = 0
        self._alloc_keys(cap)
        self._alloc_rows(row_capacity or max(1024, int(cfg.init_capacity)))
        self.counters = torch.zeros(8, dtype=torch.int32, device=self.device)
        self._refresh_struct()
        self._keys_upper = 0
        self._rows_upper = 0
        self.ctx = get_context(self.device, self.dim, owner)
        self.gid = self.ctx.register(self)
        self._map = torch.tensor([self.gid], dtype=torch.int32, device=self.device)

    def close(self) -> None:
        self.ctx.unregister(self)

    # ------------------------------------------------------------------------------------------
    def _alloc_keys(self, capacity: int) -> None:
        d = self.device
        self.capacity = capacity
        # array-of-structs: one 32-byte DrSlot {key, freq, version, row_of, tag, dirty, pad} per position (csrc/cuda/table.cuh);
        # the per-field tensors below are strided VIEWS of it (multi-tier victim selection, tests, debugging)
        self.slots = torch.empty(capacity * 4, dtype=torch.int64, device=d)
        _chk(self.lib.dr_cuda_table_init_slots(ptr(self.slots), capacity, stream_ptr()), "init_slots")
        s32 = self.slots.view(torch.int32).view(capacity, 8)
        self.keys = self.slots.view(capacity, 4)[:, 0]
        self.freq, self.version, self.row_of, self.tag, self.dirty = s32[:, 2], s32[:, 3], s32[:, 4], s32[:, 5], s32[:, 6]

    def _alloc_rows(self, row_capacity: int) -> None:
        self.row_capacity = row_capacity
        self.rows = torch.zeros(row_capacity, self.stride, dtype=torch.float32, device=self.device)
        self.free_list = torch.zeros(row_capacity, dtype=torch.int32, device=self.device)

    def _refresh_struct(self) -> None:
        s = DeviceTableStruct()
        c = self.cfg
        s.slots = self.slots.data_ptr()
        s.rows, s.free_list, s.counters = self.rows.data_ptr(), self.free_list.data_ptr(), self.counters.data_ptr()
        s.default_matrix = self.default_matrix.data_ptr()
        s.bloom = self.bloom.data_ptr() if self.bloom is not None else None
        s.capacity, s.row_capacity = self.capacity, self.row_capacity
        s.default_value_dim = self.default_matrix.shape[0]
        s.bloom_m = self.bloom.numel() if self.bloom is not None else 0
        s.dim, s.stride, s.num_slots, s.has_scalars = self.dim, self.stride, self.num_slots, int(c.has_scalars)
        s.filter_type, s.filter_freq, s.bloom_k = int(c.filter_type), int(c.filter_freq), self.bloom_k
        s.is_inference = int(c.is_inference)
        s.no_permission = float(c.default_value_no_permission)
        for i in range(4):
            s.slot_init[i] = float(c.slot_init[i])
        s.steps_to_live = int(c.steps_to_live)
        s.l2_weight_threshold = float(c.l2_weight_threshold)
        self.struct = s
        self.struct_dev = torch.frombuffer(bytearray(bytes(s)), dtype=torch.uint8).to(self.device)
        self.struct_version += 1

    # ---- capacity management (device-side rehash, no per-insert host sync) ------------------------
    def reserve(self, n_new_keys: int) -> None:
        self._keys_upper += n_new_keys
        self._rows_upper += n_new_keys
        if self._keys_upper * 2 > self.capacity or self._rows_upper > self.row_capacity:
            cnt = self.counters.cpu()
            n_keys, n_rows = int(cnt[2]), int(cnt[0])
            self._keys_upper, self._rows_upper = n_keys + n_new_keys, n_rows + n_new_keys
            new_cap, new_rows = self.capacity, self.row_capacity
            while self._keys_upper * 2 > new_cap:
                new_cap *= 2
            while self._rows_upper > new_rows:
                new_rows *= 2
            if new_cap != self.capacity or new_rows != self.row_capacity:
                self._grow(new_cap, new_rows)

    def _grow(self, new_cap: int, new_rows: int) -> None:
        old_struct = self.struct
        keep = (self.slots, self.rows, self.free_list)
        if new_rows != self.row_capacity:
            old_rows, old_fl, old_rc = self.rows, self.free_list, self.row_capacity
            self._alloc_rows(new_rows)
            self.rows[:old_rc].copy_(old_rows)
            self.free_list[:old_rc].copy_(old_fl)
        rehash = new_cap != self.capacity
        if rehash:
            self._alloc_keys(new_cap)
        self._refresh_struct()
        if rehash:
            _chk(self.lib.dr_cuda_table_rehash(C.byref(old_struct), C.byref(self.struct), stream_ptr()), "rehash")
        _native.stream_sync()
        del keep

    # ---- queries ------------------------------------------------------------------------------------
    def _keys(self, keys: torch.Tensor) -> torch.Tensor:
        return keys.to(self.device, torch.int64).contiguous().view(-1)

    def size(self) -> int:
        return int(self.counters[3].item())

    def total_keys(self) -> int:
        return int(self.counters[2].item())

    def overflowed(self) -> int:
        return int(self.counters[4].item())

    def lookup(self, keys: torch.Tensor, out_dtype: torch.dtype = torch.float32) -> torch.Tensor:
        """Read-only gather (eval / inference)."""
        k = self._keys(keys)
        n = k.numel()
        pos = torch.empty(n, dtype=torch.int32, device=self.device)
        out = torch.empty(n, self.dim, dtype=out_dtype, device=self.device)
        if n == 0:
            return out
        s, st = stream_ptr(), self.ctx.structs()
        _chk(self.lib.dr_cuda_table_lookup(ptr(st), ptr(self._map), 1, ptr(k), None, n, n, 0, None, ptr(pos), None, None, 0, s), "lookup")
        _chk(self.lib.dr_cuda_table_gather(ptr(st), ptr(self._map), 1, self.dim, ptr(k), ptr(pos), None, n, n, ptr(out),
                                           int(out_dtype == torch.bfloat16), 0, 0, 1, s), "gather")
        return out

    def lookup_train(self, keys: torch.Tensor, step: int, out_dtype: torch.dtype = torch.float32):
        """Training forward: insert/admit bookkeeping + dedup claim + gather.  Returns (rows, pos)."""
        k = self._keys(keys)
        n = k.numel()
        self.reserve(n)
        ctx = self.ctx
        ctx.ensure(n)
        pos = torch.empty(n, dtype=torch.int32, device=self.device)
        out = torch.empty(n, self.dim, dtype=out_dtype, device=self.device)
        if n == 0:
            return out, pos
        s, st = stream_ptr(), ctx.structs()
        ctx.set_step(step)
        _chk(self.lib.dr_cuda_table_lookup(ptr(st), ptr(self._map), 1, ptr(k), None, n, n, 1, ptr(ctx.step_dev), ptr(pos), ptr(ctx.ulist),
                                           ptr(ctx.nuniq), ctx.ulist.numel(), s), "lookup_train")
        _chk(self.lib.dr_cuda_table_gather(ptr(st), ptr(self._map), 1, self.dim, ptr(k), ptr(pos), None, n, n, ptr(out),
                                           int(out_dtype == torch.bfloat16), 0, 0, 1, s), "gather")
        ctx.pending = True
        return out, pos

    def accumulate(self, pos: torch.Tensor, grads: torch.Tensor) -> None:
        """Backward: scatter-add per-occurrence gradients into the per-unique-key buffer."""
        n = pos.numel()
        if n == 0:
            return
        g = grads.contiguous().view(n, self.dim)
        if g.dtype not in (torch.float32, torch.bfloat16):
            g = g.float()
        _chk(self.lib.dr_cuda_sparse_accumulate(ptr(self.ctx.structs()), ptr(self._map), 1, self.dim, ptr(pos), None, n, n, ptr(g),
                                                int(g.dtype == torch.bfloat16), 0, 0, 1, None, None, ptr(self.ctx.gsum), stream_ptr()),
             "sparse_accumulate")

    def apply_step(self, hp: OptHyper) -> None:
        self.ctx.apply_step(hp)

    def apply_raw(self, ids: torch.Tensor, grads: torch.Tensor, hp: OptHyper) -> None:
        """HostTable-compatible entry: (ids, per-occurrence grads) -> dedup + apply."""
        _, pos = self.lookup_train(ids, int(hp.global_step))
        self.accumulate(pos, grads.to(self.device))
        self.apply_step(hp)

    def apply(self, keys: torch.Tensor, grads: torch.Tensor, counts: Optional[torch.Tensor], hp: OptHyper) -> None:
        """Pre-deduplicated (keys, summed grads, counts): counts only advance the frequency."""
        k = self._keys(keys)
        g = grads.to(self.device, torch.float32)
        if counts is not None:
            reps = counts.to(self.device, torch.int64)
            idx = torch.repeat_interleave(torch.arange(k.numel(), device=self.device), reps)
            first = torch.ones_like(idx, dtype=torch.bool)
            first[1:] = idx[1:] != idx[:-1]
            k, g = k[idx], g[idx] * first.unsqueeze(-1)
        self.apply_raw(k, g, hp)

    def get_freq(self, keys: torch.Tensor) -> torch.Tensor:
        k = self._keys(keys)
        out = torch.empty(k.numel(), dtype=torch.int64, device=self.device)
        _chk(self.lib.dr_cuda_table_get_meta(C.byref(self.struct), ptr(k), k.numel(), ptr(out), None, None, stream_ptr()), "get_meta")
        return out.cpu()

    def get_version(self, keys: torch.Tensor) -> torch.Tensor:
        k = self._keys(keys)
        out = torch.empty(k.numel(), dtype=torch.int64, device=self.device)
        _chk(self.lib.dr_cuda_table_get_meta(C.byref(self.struct), ptr(k), k.numel(), None, ptr(out), None, stream_ptr()), "get_meta")
        return out.cpu()

    def lookup_slot(self, keys: torch.Tensor, slot: int) -> torch.Tensor:
        k = self._keys(keys)
        out = torch.empty(k.numel(), self.dim, dtype=torch.float32, device=self.device)
        _chk(self.lib.dr_cuda_table_gather_slot(C.byref(self.struct), ptr(k), k.numel(), int(slot), ptr(out), stream_ptr()), "gather_slot")
        return out.cpu()

    # ---- lifecycle -------------------------------------------------------------------------------------
    def shrink(self, step: int) -> int:
        n = torch.zeros(1, dtype=torch.int32, device=self.device)
        _chk(self.lib.dr_cuda_table_shrink(C.byref(self.struct), int(step), ptr(n), stream_ptr()), "shrink")
        removed = int(n.item())
        if removed:
            self._purge_tombstones()
        return removed

    def _purge_tombstones(self) -> None:
        old_struct = self.struct
        keep = (self.slots,)
        self._alloc_keys(self.capacity)
        self._refresh_struct()
        _chk(self.lib.dr_cuda_table_rehash(C.byref(old_struct), C.byref(self.struct), stream_ptr()), "rehash")
        _native.stream_sync()
        del keep

    def remove(self, keys: torch.Tensor) -> int:
        k = self._keys(keys)
        n = torch.zeros(1, dtype=torch.int32, device=self.device)
        _chk(self.lib.dr_cuda_table_remove(C.byref(self.struct), ptr(k), k.numel(), ptr(n), stream_ptr()), "remove")
        removed = int(n.item())
        self._tombstones = getattr(self, "_tombstones", 0) + removed
        if self._tombstones * 4 > self.capacity:      # probes skip tombstones; rebuild only when they pile up
            self._purge_tombstones()
            self._tombstones = 0
        return removed

    def clear_dirty(self) -> None:
        _chk(self.lib.dr_cuda_table_clear_dirty(C.byref(self.struct), stream_ptr()), "clear_dirty")

    def snapshot(self, dirty_only: bool = False, part_id: int = 0, part_num: int = 1) -> Dict[str, torch.Tensor]:
        d, s = self.device, stream_ptr()
        counts = torch.zeros(2, dtype=torch.int32, device=d)
        _chk(self.lib.dr_cuda_table_snapshot(C.byref(self.struct), int(dirty_only), part_id, part_num, ptr(counts),
                                             None, None, None, None, None, None, None, s), "snapshot(count)")
        na, nf = [int(x) for x in counts.cpu()]
        keys = torch.empty(na, dtype=torch.int64, device=d); rows = torch.empty(na, self.stride, dtype=torch.float32, device=d)
        freqs = torch.empty(na, dtype=torch.int64, device=d); vers = torch.empty(na, dtype=torch.int64, device=d)
        fkeys = torch.empty(nf, dtype=torch.int64, device=d); ffreqs = torch.empty(nf, dtype=torch.int64, device=d)
        fvers = torch.empty(nf, dtype=torch.int64, device=d)
        counts.zero_()
        _chk(self.lib.dr_cuda_table_snapshot(C.byref(self.struct), int(dirty_only), part_id, part_num, ptr(counts), ptr(keys), ptr(rows),
                                             ptr(freqs), ptr(vers), ptr(fkeys), ptr(ffreqs), ptr(fvers), s), "snapshot(fill)")

        def order(k):
            if k.numel() == 0:
                return torch.empty(0, dtype=torch.int64, device=d), torch.zeros(1001, dtype=torch.int64)
            b = torch.remainder(k, 1000)
            o = torch.argsort(k, stable=True)             # by key ...
            o = o[torch.argsort(b[o], stable=True)]       # ... then (stable) by bucket
            off = torch.zeros(1001, dtype=torch.int64)
            off[1:] = torch.cumsum(torch.bincount(b, minlength=1000), 0).cpu()
            return o, off
        oa, offa = order(keys)
        of, offf = order(fkeys)
        return dict(keys=keys[oa].cpu(), rows=rows[oa].cpu(), freqs=freqs[oa].cpu(), versions=vers[oa].cpu(), partition_offset=offa,
                    keys_filtered=fkeys[of].cpu(), freqs_filtered=ffreqs[of].cpu(), versions_filtered=fvers[of].cpu(),
                    partition_filter_offset=offf)

    def import_(self, keys, rows, freqs, versions, part_id=0, part_num=1, reset_version=False) -> int:
        k = self._keys(keys)
        n = k.numel()
        if n == 0:
            return 0
        self.reserve(n)
        r = rows.to(self.device, torch.float32).contiguous() if rows is not None else None
        f = freqs.to(self.device, torch.int64).contiguous() if freqs is not None else None
        v = versions.to(self.device, torch.int64).contiguous() if versions is not None else None
        kept = torch.zeros(1, dtype=torch.int32, device=self.device)
        _chk(self.lib.dr_cuda_table_import(C.byref(self.struct), ptr(k), ptr(r), r.shape[1] if r is not None else 0, ptr(f), ptr(v), n,
                                           part_id, part_num, int(reset_version), ptr(kept), stream_ptr()), "import")
        return int(kept.item())

    def bloom_state(self):
        return self.bloom.cpu() if self.bloom is not None else None

    def load_bloom_state(self, state: torch.Tensor) -> None:
        if self.bloom is not None:
            self.bloom.copy_(state.to(self.device).view_as(self.bloom))


class _GroupLookupFn(torch.autograd.Function):
    """N tables, one probe launch + one gather/combine launch; backward = one scatter launch."""

    @staticmethod
    def forward(ctx, anchor, tables, keys, bag_offsets, weights, combiners, B, step, train):
        t0 = tables[0]
        sc, lib, dev, T, dim = t0.ctx, t0.lib, t0.device, len(tables), t0.dim
        nnz = keys.numel()
        s = stream_ptr()
        tmap = torch.tensor([t.gid for t in tables], dtype=torch.int32, device=dev)
        offs = bag_offsets[::B][: T + 1].contiguous()          # per-table nnz offsets
        pos = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
        if train:
            for t in tables:
                t.reserve(nnz // max(T, 1) + 1)
            sc.ensure(nnz)
        st = sc.structs()
        sc.set_step(step)
        _chk(lib.dr_cuda_table_lookup(ptr(st), ptr(tmap), T, ptr(keys), ptr(offs), 0, nnz, int(train), ptr(sc.step_dev), ptr(pos),
                                      ptr(sc.ulist) if train else None, ptr(sc.nuniq) if train else None,
                                      sc.ulist.numel() if train else 0, s), "group lookup")
        out = torch.empty(B, T, dim, dtype=torch.float32, device=dev)
        nnz_scale = torch.empty(max(nnz, 1), dtype=torch.float32, device=dev)
        nnz_row = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
        _chk(lib.dr_cuda_combine_fwd(ptr(st), ptr(tmap), T, B, dim, ptr(keys), ptr(pos), ptr(bag_offsets), ptr(weights), ptr(combiners),
                                     ptr(out), 0, T * dim, dim, ptr(nnz_scale), ptr(nnz_row), s), "combine_fwd")
        if train:
            sc.pending = True
        ctx.sc, ctx.meta = sc, (B, T, dim, nnz)
        ctx.save_for_backward(pos, offs, nnz_scale, nnz_row, tmap)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        pos, offs, nnz_scale, nnz_row, tmap = ctx.saved_tensors
        B, T, dim, nnz = ctx.meta
        sc = ctx.sc
        g = grad_out.contiguous().float()
        _chk(sc.lib.dr_cuda_sparse_accumulate(ptr(sc.structs()), ptr(tmap), T, dim, ptr(pos), ptr(offs), 0, nnz, ptr(g), 0, T * dim, dim, 0,
                                              ptr(nnz_row), ptr(nnz_scale), ptr(sc.gsum), stream_ptr()), "group accumulate")
        return (None,) * 9


_ONEHOT_CACHE: Dict[tuple, tuple] = {}


def group_lookup_dense_device(params, ids: torch.Tensor) -> Optional[torch.Tensor]:
    """One id per (table, sample) -- the Criteo case: ``ids`` [T, B] feature-major -> [B, T, D] through the same two launches as
    ``group_lookup_sparse_device`` but without building bags (no per-table bincount / cumsum / cat: every bag is one id, the offsets
    are an iota that is cached per shape).  Returns None when the tables do not share one (dim, step context)."""
    from ..optim.optimizers import get_or_create_global_step
    tables = [p.table for p in params]
    if len({t.dim for t in tables}) != 1 or len({id(t.ctx) for t in tables}) != 1:
        return None
    T, B = ids.shape
    dev = tables[0].device
    key = (T, B, dev.index)
    cached = _ONEHOT_CACHE.get(key)
    if cached is None:
        cached = _ONEHOT_CACHE[key] = (torch.arange(T * B + 1, dtype=torch.int64, device=dev), torch.zeros(T, dtype=torch.int32, device=dev))   # bags, "sum"
    keys = ids.to(dev, torch.int64).reshape(-1).contiguous()
    train = bool(torch.is_grad_enabled() and any(p.trainable and not p._inference for p in params))
    return _GroupLookupFn.apply(params[0]._anchor, tables, keys, cached[0], None, cached[1], B, int(get_or_create_global_step()), train)


def group_lookup_sparse_device(params, sp_ids, combiners, sp_weights) -> List[torch.Tensor]:
    """All device tables of equal dim -> one probe launch + one gather/combine launch."""
    from ..optim.optimizers import get_or_create_global_step
    tables = [p.table for p in params]
    dims = {t.dim for t in tables}
    ctxs = {id(t.ctx) for t in tables}
    if len(dims) != 1 or len(ctxs) != 1:
        # mixed dims: split into per-dim groups (embedding_ops.py:1640 groups tables by dim)
        outs: List[Optional[torch.Tensor]] = [None] * len(params)
        groups: Dict[int, List[int]] = {}
        for i, t in enumerate(tables):
            groups.setdefault(id(t.ctx), []).append(i)
        for idxs in groups.values():
            res = group_lookup_sparse_device([params[i] for i in idxs], [sp_ids[i] for i in idxs], [combiners[i] for i in idxs],
                                             [sp_weights[i] for i in idxs])
            for i, r in zip(idxs, res):
                outs[i] = r
        return outs
    dev = tables[0].device
    B = sp_ids[0].batch_size
    vals, offs, ws, base = [], [], [], 0
    any_w = any(w is not None or s.weights is not None for s, w in zip(sp_ids, sp_weights))
    for s_, w in zip(sp_ids, sp_weights):
        v = s_.values.to(dev, torch.int64)
        r = s_.row_ids.to(dev)
        counts = torch.bincount(r, minlength=B)
        o = torch.zeros(B, dtype=torch.int64, device=dev)
        o[1:] = torch.cumsum(counts, 0)[:-1]
        offs.append(o + base)
        base += v.numel()
        vals.append(v)
        if any_w:
            ww = w if w is not None else s_.weights
            ws.append(ww.to(dev, torch.float32) if ww is not None else torch.ones(v.numel(), device=dev))
    keys = torch.cat(vals).contiguous()
    bag_offsets = torch.cat(offs + [torch.tensor([base], dtype=torch.int64, device=dev)]).contiguous()
    weights = torch.cat(ws).contiguous() if any_w else None
    comb = torch.tensor([_COMB[c] for c in combiners], dtype=torch.int32, device=dev)
    train = bool(torch.is_grad_enabled() and any(p.trainable and not p._inference for p in params))
    out = _GroupLookupFn.apply(params[0]._anchor, tables, keys, bag_offsets, weights, comb, B, int(get_or_create_global_step()), train)
    return [out[:, t, :] for t in range(len(params))]
