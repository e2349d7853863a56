"""EmbeddingVariable: the dynamic-shape (hash-keyed) embedding table and its variants.

API parity: ``tf.get_embedding_variable`` (python/ops/variable_scope.py:2147),
``EmbeddingVariable`` (python/ops/kv_variable_ops.py:48-985: total_count, get_frequency,
get_version, export, sparse_read, lookup_tier), ``MultiHashVariable`` (:986),
``DynamicEmbeddingVariable`` (:1000).

A table lives in one of two native engines behind the same interface:
  * host  -- csrc/host/host_engine.cc (CPU training / DRAM tier), storage DRAM
  * device -- csrc/cuda/table_kernels.cu (sm_90a hash table + slab rows), storage HBM / HBM_DRAM
Forward lookups never insert (post-2306 semantics, embedding_var.h:202-219): unseen keys read
their default row; creation, admission, frequency and version stamping happen in the apply.
"""
from __future__ import annotations

import zlib

import ctypes as C
from typing import Dict, List, Optional, Sequence

import torch
from torch import nn

from . import _native
from ._native import EvConfig, OptHyper, ptr
from .config import (CBFFilter, CounterFilter, EmbeddingVariableOption, FilterType, GlobalStepEvict,
                     InitializerOption, L2WeightEvict, StorageType, inference_mode)

_REGISTRY: Dict[str, "EmbeddingVariable"] = {}


def _i64(t: torch.Tensor) -> torch.Tensor:
    return t.to(dtype=torch.int64, device="cpu").contiguous()


class HostTable:
    """ctypes wrapper over dr::HostEV."""

    def __init__(self, cfg: EvConfig, default_matrix: torch.Tensor):
        self.lib = _native.host()
        self.cfg = cfg
        self.h = self.lib.dr_host_ev_create(C.byref(cfg))
        self.dim = int(cfg.dim)
        self.stride = int(self.lib.dr_host_ev_stride(self.h))
        dm = default_matrix.to(torch.float32).contiguous()
        self.lib.dr_host_ev_set_default(self.h, ptr(dm))
        self.device = torch.device("cpu")

    def __del__(self):
        try:
            if self.h:
                self.lib.dr_host_ev_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # ---- queries -------------------------------------------------------------------------
    def size(self) -> int:
        return int(self.lib.dr_host_ev_size(self.h))

    def total_keys(self) -> int:
        return int(self.lib.dr_host_ev_total_keys(self.h))

    def lookup(self, keys: torch.Tensor) -> torch.Tensor:
        k = _i64(keys).view(-1)
        out = torch.empty(k.numel(), self.dim, dtype=torch.float32)
        self.lib.dr_host_ev_lookup(self.h, ptr(k), k.numel(), ptr(out))
        return out

    def lookup_slot(self, keys: torch.Tensor, slot: int) -> torch.Tensor:
        k = _i64(keys).view(-1)
        out = torch.empty(k.numel(), self.dim, dtype=torch.float32)
        self.lib.dr_host_ev_lookup_slot(self.h, ptr(k), k.numel(), int(slot), ptr(out))
        return out

    def get_freq(self, keys: torch.Tensor) -> torch.Tensor:
        k = _i64(keys).view(-1)
        out = torch.empty(k.numel(), dtype=torch.int64)
        self.lib.dr_host_ev_get_freq(self.h, ptr(k), k.numel(), ptr(out))
        return out

    def get_version(self, keys: torch.Tensor) -> torch.Tensor:
        k = _i64(keys).view(-1)
        out = torch.empty(k.numel(), dtype=torch.int64)
        self.lib.dr_host_ev_get_version(self.h, ptr(k), k.numel(), ptr(out))
        return out

    # ---- training ------------------------------------------------------------------------
    def apply(self, keys: torch.Tensor, grads: torch.Tensor, counts: Optional[torch.Tensor], hp: OptHyper) -> None:
        k = _i64(keys).view(-1)
        g = grads.to(torch.float32).contiguous().view(k.numel(), self.dim)
        c = _i64(counts).view(-1) if counts is not None else None
        self.lib.dr_host_ev_apply(self.h, ptr(k), ptr(g), ptr(c), k.numel(), C.byref(hp))

    def apply_raw(self, ids: torch.Tensor, grads: torch.Tensor, hp: OptHyper) -> None:
        """Dedup (unique-with-counts + segment-sum, optimizer.py:91) then apply -- one native call; a row-strided ``grads`` view
        (e.g. ``g[:, t, :]`` of a grouped lookup) is consumed in place."""
        k = _i64(ids).view(-1)
        n = k.numel()
        if n == 0:
            return
        g = grads if grads.dtype == torch.float32 else grads.to(torch.float32)
        g = g.reshape(n, self.dim) if g.is_contiguous() else g
        if g.dim() != 2 or g.stride(1) != 1:
            g = g.reshape(n, self.dim).contiguous()
        self.lib.dr_host_ev_apply_raw(self.h, ptr(k), n, C.c_void_p(g.data_ptr()), int(g.stride(0)), C.byref(hp))

    def apply_segments(self, segs, hp: OptHyper) -> None:
        """ONE de-duplicated apply for everything the table received in a step.  ``segs`` = [(ids, grads, group)]: occurrence i of a segment
        uses gradient row ``i // group`` (group 1 = plain lookup; group L = sum-pooled bags of L ids sharing one row)."""
        keep, ids_p, n_p, g_p, st_p, gr_p = [], [], [], [], [], []
        for ids, grads, group in segs:
            k = _i64(ids).view(-1)
            if k.numel() == 0:
                continue
            g = grads if grads.dtype == torch.float32 else grads.to(torch.float32)
            if g.dim() != 2 or g.stride(1) != 1:
                g = g.reshape(-1, self.dim).contiguous()
            keep += [k, g]
            ids_p.append(k.data_ptr()); n_p.append(k.numel()); g_p.append(g.data_ptr()); st_p.append(int(g.stride(0))); gr_p.append(int(group))
        m = len(ids_p)
        if m == 0:
            return
        vp, i64 = C.c_void_p, C.c_int64
        self.lib.dr_host_ev_apply_multi(self.h, m, (vp * m)(*ids_p), (i64 * m)(*n_p), (vp * m)(*g_p), (i64 * m)(*st_p), (i64 * m)(*gr_p), C.byref(hp))

    def lookup_pooled(self, ids: torch.Tensor) -> torch.Tensor:
        """ids [B, L] (PAD_KEY = unused position) -> [B, dim]: per-sample sum of rows, no [B, L, dim] intermediate."""
        k = _i64(ids)
        B, L = k.shape
        out = torch.empty(B, self.dim, dtype=torch.float32)
        self.lib.dr_host_ev_lookup_pooled(self.h, ptr(k), B, L, ptr(out), self.dim)
        return out

    # ---- lifecycle -----------------------------------------------------------------------
    def shrink(self, step: int) -> int:
        return int(self.lib.dr_host_ev_shrink(self.h, int(step)))

    def remove(self, keys: torch.Tensor) -> int:
        k = _i64(keys).view(-1)
        return int(self.lib.dr_host_ev_remove(self.h, ptr(k), k.numel()))

    def clear_dirty(self) -> None:
        self.lib.dr_host_ev_clear_dirty(self.h)

    def snapshot(self, dirty_only: bool = False, part_id: int = 0, part_num: int = 1) -> Dict[str, torch.Tensor]:
        na, nf = C.c_int64(0), C.c_int64(0)
        self.lib.dr_host_ev_snapshot_begin(self.h, int(dirty_only), part_id, part_num, C.byref(na), C.byref(nf))
        na, nf = na.value, nf.value
        out = dict(
            keys=torch.empty(na, dtype=torch.int64), rows=torch.empty(na, self.stride, dtype=torch.float32),
            freqs=torch.empty(na, dtype=torch.int64), versions=torch.empty(na, dtype=torch.int64),
            partition_offset=torch.zeros(1001, dtype=torch.int64),
            keys_filtered=torch.empty(nf, dtype=torch.int64), freqs_filtered=torch.empty(nf, dtype=torch.int64),
            versions_filtered=torch.empty(nf, dtype=torch.int64), partition_filter_offset=torch.zeros(1001, dtype=torch.int64))
        self.lib.dr_host_ev_snapshot_read(
            self.h, ptr(out["keys"]), ptr(out["rows"]), ptr(out["freqs"]), ptr(out["versions"]), ptr(out["partition_offset"]),
            ptr(out["keys_filtered"]), ptr(out["freqs_filtered"]), ptr(out["versions_filtered"]), ptr(out["partition_filter_offset"]))
        self.lib.dr_host_ev_snapshot_end(self.h)
        return out

    def import_(self, keys, rows, freqs, versions, part_id=0, part_num=1, reset_version=False) -> int:
        k = _i64(keys).view(-1)
        r = rows.to(torch.float32).contiguous() if rows is not None else None
        ncols = r.shape[1] if r is not None else 0
        f = _i64(freqs) if freqs is not None else None
        v = _i64(versions) if versions is not None else None
        return int(self.lib.dr_host_ev_import(self.h, ptr(k), ptr(r), ncols, ptr(f), ptr(v), k.numel(), part_id, part_num, int(reset_version)))

    def export_keys(self, keys: torch.Tensor):
        """(rows [n, stride], freqs, versions, found) of specific keys (multi-tier promotion path)."""
        k = _i64(keys).view(-1)
        n = k.numel()
        rows = torch.empty(n, self.stride, dtype=torch.float32)
        f = torch.empty(n, dtype=torch.int64); v = torch.empty(n, dtype=torch.int64); found = torch.zeros(n, dtype=torch.uint8)
        if n:
            self.lib.dr_host_ev_export_keys(self.h, ptr(k), n, ptr(rows), ptr(f), ptr(v), ptr(found))
        return rows, f, v, found.bool()

    def bloom_state(self) -> Optional[torch.Tensor]:
        k, m, b = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        nb = int(self.lib.dr_host_bloom_info(self.h, C.byref(k), C.byref(m), C.byref(b)))
        if nb == 0:
            return None
        out = torch.empty(nb, dtype=torch.uint8)
        self.lib.dr_host_bloom_read(self.h, ptr(out))
        return out

    def load_bloom_state(self, state: torch.Tensor) -> None:
        self.lib.dr_host_bloom_write(self.h, ptr(state.contiguous()))


class _EVLookup(torch.autograd.Function):
    """Gather rows; backward records (ids, grad rows) on the variable as a sparse gradient
    (the IndexedSlices analogue) for the optimizer's dedup + sparse apply."""

    @staticmethod
    def forward(ctx, anchor: torch.Tensor, ev: "EmbeddingVariable", ids: torch.Tensor):
        ctx.ev = ev
        out, pos = ev._gather_train(ids)
        ctx.pos = pos
        ctx.save_for_backward(ids)
        return out

    @staticmethod
    def backward(ctx, grad_out: torch.Tensor):
        (ids,) = ctx.saved_tensors
        if ctx.pos is not None:       # device table: scatter straight into the per-unique buffer
            ctx.ev.table.accumulate(ctx.pos, grad_out)
        else:
            ctx.ev._record_grad(ids, grad_out)
        return None, None, None


class _EVLookupPooled(torch.autograd.Function):
    """Sum-pooled lookup of a dense ``[B, L]`` id tensor on a host table; the backward records ONE gradient row per bag."""

    @staticmethod
    def forward(ctx, anchor: torch.Tensor, ev: "EmbeddingVariable", ids: torch.Tensor):
        ctx.ev, ctx.ids = ev, ids
        return ev.table.lookup_pooled(ids)

    @staticmethod
    def backward(ctx, grad_out: torch.Tensor):
        ids = ctx.ids
        ctx.ev._pending.append((ids.reshape(-1), grad_out.contiguous(), ids.shape[1]))      # (ids, [B, D] rows, group = L)
        return None, None, None


class EmbeddingVariable(nn.Module):
    """A hash-keyed embedding table with admission, eviction, optimizer slots in-row and
    (optionally) multi-tier storage."""

    def __init__(self, name: str, embedding_dim: int, key_dtype: torch.dtype = torch.int64,
                 value_dtype: torch.dtype = torch.float32, initializer=None, trainable: bool = True,
                 ev_option: Optional[EmbeddingVariableOption] = None, device: Optional[torch.device] = None,
                 seed: Optional[int] = None):
        super().__init__()
        self.name = name
        self.embedding_dim = int(embedding_dim)
        self.key_dtype = key_dtype
        self.value_dtype = value_dtype
        self.trainable = trainable
        self.option = ev_option or EmbeddingVariableOption()
        if initializer is not None:
            self.option.init_option = InitializerOption(initializer, self.option.init_option.default_value_dim,
                                                        self.option.init_option.default_value_no_permission)
        st = self.option.storage_option.storage_type
        if device is None:
            device = (torch.device("cuda", torch.cuda.current_device()) if st in (StorageType.HBM, StorageType.HBM_DRAM, StorageType.HBM_DRAM_SSDHASH)
                      else torch.device("cpu"))
        self.device = torch.device(device)
        if self.device.type == "cuda" and st == StorageType.DRAM:
            # kv_variable_ops.cc:225-232: a GPU variable needs an HBM first tier
            self.option.storage_option.storage_type = StorageType.HBM
        # zero-size parameter: gives autograd a leaf so backward reaches _EVLookup
        self._anchor = nn.Parameter(torch.zeros(0, device=self.device), requires_grad=trainable)
        self._num_slots = 0
        self._slot_init = [0.0, 0.0, 0.0, 0.0]
        self._has_scalars = 0
        self._slot_names: List[str] = []
        self._table = None
        self._owner = 0
        self._pending: List = []
        self._group_pending = []          # grouped sparse gradients (ops/host_group.py), drained by the optimizer
        self._seed = seed
        self._inference = inference_mode()
        g = torch.Generator().manual_seed(seed if seed is not None else (zlib.crc32(name.encode()) & 0x7FFFFFFF))
        dvd = max(1, int(self.option.init_option.default_value_dim))
        dm = torch.empty(dvd, self.embedding_dim, dtype=torch.float32)
        init = self.option.init_option.initializer
        if init is None:
            dm.normal_(0.0, 1.0 / (self.embedding_dim ** 0.5), generator=g)   # truncated-normal-like default
            dm.clamp_(-2.0 / (self.embedding_dim ** 0.5), 2.0 / (self.embedding_dim ** 0.5))
        else:
            init(dm)
        self.default_matrix = dm
        _REGISTRY[name] = self

    # ------------------------------------------------------------------------------------
    def _make_config(self) -> EvConfig:
        o = self.option
        cfg = EvConfig()
        cfg.dim = self.embedding_dim
        cfg.num_slots = self._num_slots
        cfg.has_scalars = self._has_scalars
        cfg.init_capacity = int(o.init_capacity)
        f = o.filter_option
        cfg.filter_type = FilterType.NONE
        cfg.bloom_counter_bits = 32
        if isinstance(f, CounterFilter) and f.filter_freq > 0:
            cfg.filter_type, cfg.filter_freq = FilterType.COUNTER, f.filter_freq
        elif isinstance(f, CBFFilter) and f.filter_freq > 0:
            if f.max_element_size > 0 and 0 < f.false_positive_probability < 1:
                cfg.filter_type, cfg.filter_freq = FilterType.BLOOM, f.filter_freq
                cfg.bloom_max_elements, cfg.bloom_fpp = f.max_element_size, f.false_positive_probability
                cfg.bloom_counter_bits = f.counter_bits()
            else:   # CBF without sizing degenerates to the exact counter (variables.py CBFFilter doc)
                cfg.filter_type, cfg.filter_freq = FilterType.COUNTER, f.filter_freq
        e = o.evict_option
        cfg.steps_to_live = e.steps_to_live if isinstance(e, GlobalStepEvict) else 0
        cfg.l2_weight_threshold = e.l2_weight_threshold if isinstance(e, L2WeightEvict) else -1.0
        cfg.default_value_no_permission = o.init_option.default_value_no_permission
        cfg.default_value_dim = self.default_matrix.shape[0]
        cfg.record_freq, cfg.record_version = int(o.record_freq), int(o.record_version)
        cfg.is_inference = int(self._inference)
        cfg.storage_type = int(o.storage_option.storage_type)
        row_bytes = 4 * (self.embedding_dim * (1 + self._num_slots) + (4 if self._has_scalars else 0))
        cfg.hbm_cache_rows = max(1, int(o.storage_option.storage_size[0]) // row_bytes)   # multi_tier_storage.h:58-62
        cfg.cache_strategy = int(o.storage_option.cache_strategy)
        cfg.num_partitions = int(o.ht_partition_num)
        for i in range(4):
            cfg.slot_init[i] = float(self._slot_init[i])
        return cfg

    @property
    def table(self):
        if self._table is None:
            cfg = self._make_config()
            so = self.option.storage_option
            row_bytes = 4 * (self.embedding_dim * (1 + self._num_slots) + (4 if self._has_scalars else 0))
            if self.device.type == "cuda" and int(cfg.storage_type) in (int(StorageType.HBM_DRAM), int(StorageType.HBM_DRAM_SSDHASH)):
                from .ops.multi_tier import MultiTierTable
                ssd = None
                if int(cfg.storage_type) == int(StorageType.HBM_DRAM_SSDHASH):
                    sz = so.storage_size[1] if len(so.storage_size) > 1 else (1 << 30)
                    ssd = dict(dram_rows=max(64, int(sz) // row_bytes), path=so.storage_path)
                self._table = MultiTierTable(cfg, self.default_matrix, self.device, owner=self._owner, ssd=ssd)
            elif self.device.type == "cpu" and int(cfg.storage_type) == int(StorageType.DRAM_SSDHASH):
                from .ops.host_tiers import DramSsdTable
                self._table = DramSsdTable(cfg, self.default_matrix, dram_rows=max(64, int(so.storage_size[0]) // row_bytes), path=so.storage_path,
                                           strategy=int(so.cache_strategy))
            elif self.device.type == "cuda":
                from .ops.device_table import DeviceTable
                self._table = DeviceTable(cfg, self.default_matrix, self.device, owner=self._owner)
            else:
                self._table = HostTable(cfg, self.default_matrix)
            self._warm_start()
        return self._table

    def _warm_start(self) -> None:
        """``CheckpointOption`` (ops/variables.py:217-227, kv_variable_ops.py:636-705): initialise this variable from a tensor of
        ANOTHER checkpoint (``ckpt_to_load_from`` + ``tensor_name_in_ckpt``; keys / values / freqs / versions, optimizer slots are
        not taken over) or from an external ``init_data_source`` (a ``.pt`` / ``.npz`` file or a dict with ``keys`` and ``values``).
        Runs once, when the table is first materialised, unless ``always_load_from_specific_ckpt`` asks for every re-creation."""
        co = self.option.ckpt
        if co is None or (getattr(self, "_warm_started", False) and not co.always_load_from_specific_ckpt):
            return
        keys = vals = freqs = vers = None
        if co.ckpt_to_load_from:
            from .checkpoint.saver import BundleReader, latest_checkpoint
            import os
            prefix = co.ckpt_to_load_from
            if os.path.isdir(prefix):
                prefix = latest_checkpoint(prefix) or prefix
            r = BundleReader(prefix)
            name = co.tensor_name_in_ckpt or self.name
            if not r.has(f"{name}-keys"):
                raise KeyError(f"checkpoint {prefix} has no EmbeddingVariable named {name!r}")
            keys, vals = r.read(f"{name}-keys"), r.read(f"{name}-values")
            freqs = r.read(f"{name}-freqs") if r.has(f"{name}-freqs") else None
            vers = r.read(f"{name}-versions") if r.has(f"{name}-versions") else None
            r.close()
        elif co.init_data_source is not None:
            src = co.init_data_source
            if isinstance(src, str):
                if src.endswith(".npz"):
                    import numpy as np
                    z = np.load(src)
                    src = {k: torch.from_numpy(z[k]) for k in z.files}
                else:
                    src = torch.load(src)
            keys, vals = torch.as_tensor(src["keys"]), torch.as_tensor(src["values"])
            freqs, vers = src.get("freqs"), src.get("versions")
        if keys is None:
            return
        if vals.shape[1] != self.embedding_dim:
            raise ValueError(f"warm start of {self.name}: source dim {vals.shape[1]} != embedding_dim {self.embedding_dim}")
        n = keys.numel()
        self._table.import_(keys.to(torch.int64), vals.to(torch.float32).contiguous(),
                            freqs if freqs is not None else torch.zeros(n, dtype=torch.int64),
                            vers if vers is not None else torch.full((n,), -1, dtype=torch.int64))
        self._warm_started = True

    def _set_slots(self, slot_names: Sequence[str], slot_init: Sequence[float], has_scalars: bool, owner: int = 0) -> None:
        """Called by the optimizer: reserve in-row optimizer slots (slot_creator.py:86-134).
        If rows already exist they are migrated (embedding kept, slots re-initialised)."""
        n = len(slot_names)
        init = list(slot_init) + [0.0] * (4 - len(slot_init))
        same_owner = owner == self._owner or self.device.type != "cuda"
        if n == self._num_slots and init == self._slot_init and int(has_scalars) == self._has_scalars and (same_owner or self._table is None):
            self._slot_names = list(slot_names)
            self._owner = owner
            return
        self._owner = owner
        old = self._table
        snap = old.snapshot() if old is not None and old.total_keys() > 0 else None
        self._num_slots, self._slot_init, self._has_scalars = n, init, int(has_scalars)
        self._slot_names = list(slot_names)
        if old is not None and hasattr(old, "close"):
            old.close()
        self._table = None
        if snap is not None:
            t = self.table
            t.import_(snap["keys"], snap["rows"][:, : self.embedding_dim].contiguous(), snap["freqs"], snap["versions"])
            if snap["keys_filtered"].numel():
                t.import_(snap["keys_filtered"], None, snap["freqs_filtered"], snap["versions_filtered"])

    # ------------------------------------------------------------------------------------
    def _gather(self, ids: torch.Tensor) -> torch.Tensor:
        flat = ids.reshape(-1)
        out = self.table.lookup(flat)
        return out.view(*ids.shape, self.embedding_dim).to(self.device)

    def _gather_train(self, ids: torch.Tensor):
        t = self.table
        if self.device.type == "cuda":
            from .optim.optimizers import get_or_create_global_step
            rows, pos = t.lookup_train(ids.reshape(-1), int(get_or_create_global_step()))
            return rows.view(*ids.shape, self.embedding_dim), pos
        return self._gather(ids), None

    def _record_grad(self, ids: torch.Tensor, grad: torch.Tensor) -> None:
        self._pending.append((ids.reshape(-1), grad.reshape(-1, self.embedding_dim), 1))

    def forward(self, ids: torch.Tensor) -> torch.Tensor:
        return self.lookup(ids)

    def lookup(self, ids: torch.Tensor) -> torch.Tensor:
        """``sparse_read`` (kv_variable_ops.py:855): [..] int64 ids -> [.., dim] rows."""
        if self.trainable and torch.is_grad_enabled() and not self._inference:
            return _EVLookup.apply(self._anchor, self, ids)
        return self._gather(ids)

    sparse_read = lookup

    def lookup_pooled(self, ids: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``embedding_lookup_sparse(combiner="sum")`` for a dense ``[B, L]`` id tensor whose valid positions are given by ``mask``
        (or marked with ``config.PAD_KEY``): -> ``[B, dim]``.  Plain host tables do it in one native pass (no ``[B, L, dim]``
        intermediate in the forward, one gradient row per bag in the backward); every other table type falls back to
        lookup + mask + sum."""
        from .config import PAD_KEY
        if self.device.type == "cpu" and isinstance(self.table, HostTable) and ids.dim() == 2:
            k = ids if mask is None else torch.where(mask, ids, PAD_KEY)
            if self.trainable and torch.is_grad_enabled() and not self._inference:
                return _EVLookupPooled.apply(self._anchor, self, k.contiguous())
            return self.table.lookup_pooled(k.contiguous())
        if mask is None:
            mask = ids != PAD_KEY
        rows = self.lookup(torch.where(mask, ids, torch.zeros_like(ids)))
        return (rows * mask.unsqueeze(-1).to(rows.dtype).to(rows.device)).sum(1)

    def pop_sparse_grads(self):
        """Concatenated (ids, grads) accumulated by backward since the last step."""
        if not self._pending:
            return None
        segs = [(i, g if grp == 1 else g.repeat_interleave(grp, dim=0)) for i, g, grp in self._pending]   # pooled bags: one row per occurrence
        if len(segs) == 1:                              # the common case: one lookup per step -> no copy
            ids, grads = segs[0]
        else:
            ids = torch.cat([p[0] for p in segs])
            grads = torch.cat([p[1] for p in segs])
        self._pending.clear()
        return ids, grads

    def pop_sparse_segments(self):
        """[(ids, grads, group)] recorded since the last step, without concatenating or expanding anything (HostTable.apply_segments)."""
        segs, self._pending = self._pending, []
        return segs

    # ---- introspection (EVGetFrequency / EVGetVersion / KvVariableShape) ---------------------
    def total_count(self) -> int:
        return self.table.size()

    def get_frequency(self, ids: torch.Tensor) -> torch.Tensor:
        return self.table.get_freq(ids).view(ids.shape)

    def get_version(self, ids: torch.Tensor) -> torch.Tensor:
        return self.table.get_version(ids).view(ids.shape)

    def export(self):
        """(keys, values, versions, freqs) of admitted keys (KvResourceExport)."""
        s = self.table.snapshot()
        return s["keys"], s["rows"][:, : self.embedding_dim].contiguous(), s["versions"], s["freqs"]

    @torch.no_grad()
    def scatter_add(self, ids: torch.Tensor, updates: torch.Tensor) -> None:
        """``KvResourceScatterAdd``: rows[id] += update (creates / admits keys like an SGD apply with lr = -1)."""
        hp = OptHyper()
        hp.kind, hp.lr = 0, -1.0
        from .optim.optimizers import get_or_create_global_step
        hp.global_step = int(get_or_create_global_step())
        self.table.apply_raw(ids.reshape(-1), updates.reshape(-1, self.embedding_dim), hp)

    def lookup_tier(self, ids: torch.Tensor) -> torch.Tensor:
        """KvResourceLookupTier: 0 = first tier (HBM/DRAM), 1 = second tier, -1 = absent."""
        t = self.table
        if hasattr(t, "lookup_tier"):
            return t.lookup_tier(ids)
        present = t.get_version(ids) != -1
        present |= t.get_freq(ids) > 0
        return torch.where(present.view(ids.shape), torch.zeros_like(ids), -torch.ones_like(ids))

    def slot_values(self, ids: torch.Tensor, slot_name: str) -> torch.Tensor:
        return self.table.lookup_slot(ids, 1 + self._slot_names.index(slot_name))

    def extra_repr(self) -> str:
        return f"name={self.name}, dim={self.embedding_dim}, storage={StorageType(self.option.storage_option.storage_type).name}"


def get_embedding_variable(name: str, embedding_dim: int, key_dtype: torch.dtype = torch.int64,
                           value_dtype: torch.dtype = torch.float32, initializer=None, trainable: bool = True,
                           partitioner=None, ev_option: Optional[EmbeddingVariableOption] = None,
                           device=None, seed: Optional[int] = None):
    """``tf.get_embedding_variable`` (variable_scope.py:2147).  ``partitioner`` =
    ``fixed_size_partitioner(N)`` returns a :class:`PartitionedEmbeddingVariable`."""
    if partitioner is not None:
        n = partitioner if isinstance(partitioner, int) else partitioner.num_shards
        if n > 1:
            return PartitionedEmbeddingVariable(name, embedding_dim, n, key_dtype, value_dtype, initializer, trainable,
                                                ev_option, device, seed)
    return EmbeddingVariable(name, embedding_dim, key_dtype, value_dtype, initializer, trainable, ev_option, device, seed)


class fixed_size_partitioner:
    def __init__(self, num_shards: int):
        self.num_shards = int(num_shards)


class PartitionedEmbeddingVariable(nn.Module):
    """N EVs ``name/part_i``; ids routed by ``id % N`` (embedding_ops.py:214-330,
    dynamic_partition + dynamic_stitch)."""

    def __init__(self, name, embedding_dim, num_shards, key_dtype, value_dtype, initializer, trainable, ev_option, device, seed):
        super().__init__()
        import copy
        self.name, self.embedding_dim, self.num_shards = name, int(embedding_dim), int(num_shards)
        self.parts = nn.ModuleList([
            EmbeddingVariable(f"{name}/part_{i}", embedding_dim, key_dtype, value_dtype, initializer, trainable,
                              copy.deepcopy(ev_option) if ev_option else None, device, seed)
            for i in range(num_shards)])
        # all shards draw from the same default matrix so a key's initial value does not
        # depend on the shard count (N->M re-sharding keeps semantics)
        for p in self.parts[1:]:
            p.default_matrix = self.parts[0].default_matrix

    def lookup(self, ids: torch.Tensor) -> torch.Tensor:
        flat = ids.reshape(-1)
        shard = torch.remainder(flat, self.num_shards)
        out = torch.empty(flat.numel(), self.embedding_dim, dtype=torch.float32, device=self.parts[0].device)
        for i, p in enumerate(self.parts):
            m = (shard == i).nonzero(as_tuple=True)[0]
            if m.numel():
                out = out.index_copy(0, m.to(out.device), p.lookup(flat[m]))
        return out.view(*ids.shape, self.embedding_dim)

    forward = lookup

    def total_count(self) -> int:
        return sum(p.total_count() for p in self.parts)

    def get_frequency(self, ids):
        flat = ids.reshape(-1)
        out = torch.zeros_like(flat)
        for i, p in enumerate(self.parts):
            m = torch.remainder(flat, self.num_shards) == i
            if m.any():
                out[m] = p.get_frequency(flat[m])
        return out.view(ids.shape)


class MultiHashVariable(nn.Module):
    """Q-R trick (``tf.get_multihash_variable``, variable_scope.py:2317; embedding_ops.py:148-170):
    two small static tables indexed by ``id // size0`` ("Q") and ``id % size1`` ("R"), combined by
    add / mult / concat."""

    def __init__(self, name: str, dims: Sequence[Sequence[int]], num_of_partitions: int = 2,
                 complementary_strategy: str = "Q-R", operation: str = "add", device=None, initializer=None):
        super().__init__()
        if complementary_strategy != "Q-R" or num_of_partitions != 2:
            raise ValueError("only the Q-R strategy with 2 partitions is defined (variable_scope.py:2330)")
        if operation not in ("add", "mult", "mul", "concat"):
            raise ValueError("operation must be add | mult | concat")
        self.name, self.operation = name, "mult" if operation == "mul" else operation
        (q_rows, q_dim), (r_rows, r_dim) = dims
        if self.operation != "concat" and q_dim != r_dim:
            raise ValueError("add/mult need equal dims")
        self.q = nn.Embedding(q_rows, q_dim, device=device)
        self.r = nn.Embedding(r_rows, r_dim, device=device)
        if initializer is not None:
            initializer(self.q.weight.data); initializer(self.r.weight.data)
        self.embedding_dim = q_dim + r_dim if self.operation == "concat" else q_dim

    def lookup(self, ids: torch.Tensor) -> torch.Tensor:
        q = torch.remainder(torch.div(ids, self.r.num_embeddings, rounding_mode="floor"), self.q.num_embeddings)
        r = torch.remainder(ids, self.r.num_embeddings)
        eq, er = self.q(q), self.r(r)
        if self.operation == "add":
            return eq + er
        if self.operation == "mult":
            return eq * er
        return torch.cat([eq, er], dim=-1)

    forward = lookup


def get_multihash_variable(name, dims, num_of_partitions=2, complementary_strategy="Q-R", operation="add",
                           device=None, initializer=None) -> MultiHashVariable:
    return MultiHashVariable(name, dims, num_of_partitions, complementary_strategy, operation, device, initializer)


class DynamicEmbeddingVariable(nn.Module):
    """Dynamic-dimension EV (``tf.get_dynamic_dimension_embedding_variable``, variable_scope.py:2373;
    embedding_ops.py:176-200 ``_gather_fae``): ``block_num`` sub-tables of ``dim/block_num``; an id owns
    the first ``blocknums[id]`` blocks, the rest of its vector is zero."""

    def __init__(self, name: str, embedding_block_dimension: int, embedding_block_num: int,
                 ev_option: Optional[EmbeddingVariableOption] = None, device=None, initializer=None):
        super().__init__()
        import copy
        self.name = name
        self.block_dim, self.block_num = int(embedding_block_dimension), int(embedding_block_num)
        self.embedding_dim = self.block_dim * self.block_num
        self.blocks = nn.ModuleList([
            EmbeddingVariable(f"{name}/block{i}", self.block_dim, initializer=initializer,
                              ev_option=copy.deepcopy(ev_option) if ev_option else None, device=device)
            for i in range(self.block_num)])

    def lookup(self, ids: torch.Tensor, blocknums: torch.Tensor) -> torch.Tensor:
        outs = []
        for i, b in enumerate(self.blocks):
            e = b.lookup(ids)
            mask = (blocknums > i).to(e.dtype).unsqueeze(-1).to(e.device)
            outs.append(e * mask)
        return torch.cat(outs, dim=-1)

    forward = lookup


def get_dynamic_dimension_embedding_variable(name, embedding_block_dimension, embedding_block_num,
                                             ev_option=None, device=None, initializer=None):
    return DynamicEmbeddingVariable(name, embedding_block_dimension, embedding_block_num, ev_option, device, initializer)


def all_embedding_variables() -> Dict[str, EmbeddingVariable]:
    return dict(_REGISTRY)


def clear_registry() -> None:
    _REGISTRY.clear()
