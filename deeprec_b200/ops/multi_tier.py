"""Multi-tier EmbeddingVariable storage: HBM cache tier over a DRAM (host) tier -- ``StorageType.HBM_DRAM``.

Reference behaviour (SURVEY §2.1 MultiTierStorage / HbmDramStorage / BatchCache / EvictionManager, Appendix A.5):
  * compute always touches tier 0; tier-0 capacity = ``storage_size[0] / row_bytes``; a batch's unique ids must fit;
  * misses are promoted (host rows packed -> pinned H2D -> unpack kernel), cold rows demoted (copy kernel -> D2H -> host commit);
  * LFU / LRU victim selection, ids fetched by the staged (prefetch) pipeline are pinned until consumed
    (``add_to_prefetch_list`` / ``add_to_cache``), hit/miss counters, ``lookup_tier``.
Differences by design: the reference keeps the index of BOTH tiers in a CPU hash map and resolves every GPU lookup on the
host (ids D2H + blocking probe, kv_variable_lookup_ops.cc:404-412).  Here tier 0 has its own device hash table, so hits
never leave the GPU; only the miss list crosses PCIe, and promotion/demotion run on a side stream from ``prefetch()``
(driven one batch ahead by the input pipeline), so the training stream sees a warm cache.  LFU/LRU metadata are the
device table's own ``freq`` / ``version`` columns (no separate cache structure).
"""
from __future__ import annotations

import copy
import ctypes as C
from typing import Dict, Optional

import torch

from .._native import EvConfig, OptHyper, check, ptr, stream_ptr
from ..embedding_variable import HostTable
from .device_table import DeviceTable


class MultiTierTable:
    def __init__(self, cfg: EvConfig, default_matrix: torch.Tensor, device: torch.device, owner: int = 0, ssd: Optional[dict] = None):
        self.cfg = cfg
        self.device = torch.device(device)
        self.dim = int(cfg.dim)
        self.cache_rows = max(1024, int(cfg.hbm_cache_rows))
        self.strategy = int(cfg.cache_strategy)             # 0 LFU, 1 LRU
        hbm_cfg = copy.copy(cfg)
        self.hbm = DeviceTable(hbm_cfg, default_matrix, self.device, capacity=None, row_capacity=self.cache_rows + 1024, owner=owner)
        host_cfg = EvConfig.from_buffer_copy(bytes(cfg))
        host_cfg.filter_type, host_cfg.filter_freq = 0, 0        # admission is decided in tier 0; the host tier stores what it is given
        host_cfg.steps_to_live, host_cfg.l2_weight_threshold = 0, -1.0
        if ssd is not None:                                      # HBM_DRAM_SSDHASH: the host tier itself spills to a log-structured SSD store
            from .host_tiers import DramSsdTable
            self.dram = DramSsdTable(host_cfg, default_matrix, strategy=int(cfg.cache_strategy), **ssd)
        else:
            self.dram = HostTable(host_cfg, default_matrix)
        self.stride = self.hbm.stride
        self.lib = self.hbm.lib
        self.side = torch.cuda.Stream(device=self.device)
        self.hits = 0
        self.misses = 0
        self._pinned: Optional[torch.Tensor] = None           # keys promoted by prefetch() and not yet consumed
        self.ctx = self.hbm.ctx

    # ---- tier movement --------------------------------------------------------------------------------------
    def _promote(self, keys: torch.Tensor) -> None:
        """Bring the listed (unique, HBM-absent) keys up from DRAM if they live there."""
        k = keys.to("cpu", torch.int64).contiguous()
        n = k.numel()
        if n == 0:
            return
        rows, freqs, vers, sel = self.dram.export_keys(k)
        if sel.any():
            self.hbm.import_(k[sel], rows[sel].pin_memory(), freqs[sel], vers[sel])   # pinned H2D + import kernel on the current stream

    def _evict(self, need: int, protect: Optional[torch.Tensor]) -> None:
        """Demote cold rows until ``need`` more rows fit (LFU: lowest freq, LRU: oldest version)."""
        t = self.hbm
        resident = t.size()
        over = resident + need - self.cache_rows
        if over <= 0:
            return
        n_evict = min(resident, over + max(1024, self.cache_rows // 16))       # evict in chunks to amortise
        occupied = t.row_of >= 0
        score = (t.freq if self.strategy == 0 else t.version).to(torch.float32)
        score = torch.where(occupied, score, torch.full_like(score, float("inf")))
        if protect is not None and protect.numel():
            # pinned / in-flight keys must stay: find their positions and lift their score
            pos = torch.empty(protect.numel(), dtype=torch.int32, device=self.device)
            check(self.lib.dr_cuda_table_lookup(ptr(t.ctx.structs()), ptr(t._map), 1, ptr(protect), None, protect.numel(), protect.numel(), 0, None,
                                                ptr(pos), None, None, 0, stream_ptr()), "lookup(protect)")
            ok = pos >= 0
            score[pos[ok].long()] = float("inf")
        n_evict = min(n_evict, int(torch.isfinite(score).sum()))
        if n_evict <= 0:
            raise RuntimeError("HBM tier too small: the batch's unique ids (plus pinned prefetched ids) must fit in tier 0 "
                               "(kv_variable_lookup_ops.cc:198-202)")
        victims_pos = torch.topk(score, n_evict, largest=False).indices
        vkeys = t.keys[victims_pos].contiguous()
        rows = torch.empty(n_evict, self.stride, dtype=torch.float32, device=self.device)
        freqs = torch.empty(n_evict, dtype=torch.int64, device=self.device); vers = torch.empty(n_evict, dtype=torch.int64, device=self.device)
        found = torch.empty(n_evict, dtype=torch.uint8, device=self.device)
        check(self.lib.dr_cuda_table_export_keys(C.byref(t.struct), ptr(vkeys), n_evict, ptr(rows), ptr(freqs), ptr(vers), ptr(found), stream_ptr()), "export_keys")
        self.dram.import_(vkeys.cpu(), rows.cpu(), freqs.cpu(), vers.cpu())     # BatchCommit into the host tier
        t.remove(vkeys)

    def _ensure_resident(self, keys: torch.Tensor, pin: bool) -> None:
        k = keys.to(self.device, torch.int64).reshape(-1)
        uniq = torch.unique(k)
        pos = torch.empty(uniq.numel(), dtype=torch.int32, device=self.device)
        t = self.hbm
        check(self.lib.dr_cuda_table_lookup(ptr(t.ctx.structs()), ptr(t._map), 1, ptr(uniq), None, uniq.numel(), uniq.numel(), 0, None, ptr(pos),
                                            None, None, 0, stream_ptr()), "lookup(presence)")
        miss = uniq[pos < 0]
        self.hits += int(uniq.numel() - miss.numel()); self.misses += int(miss.numel())
        protect = uniq if self._pinned is None else torch.unique(torch.cat([uniq, self._pinned]))
        self._evict(int(miss.numel()), protect)
        self._promote(miss)
        if pin:
            self._pinned = uniq if self._pinned is None else torch.unique(torch.cat([self._pinned, uniq]))

    def prefetch(self, keys: torch.Tensor) -> None:
        """Called by the input pipeline one batch ahead (staged subgraph): promotes/demotes on a side stream and pins the ids."""
        self.side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.side):
            self._ensure_resident(keys, pin=True)
        self._prefetch_event = torch.cuda.Event(); self._prefetch_event.record(self.side)

    # ---- table interface ----------------------------------------------------------------------------------------
    def lookup(self, keys: torch.Tensor, out_dtype=torch.float32) -> torch.Tensor:
        self._sync_prefetch()
        self._ensure_resident(keys, pin=False)
        return self.hbm.lookup(keys, out_dtype)

    def _sync_prefetch(self):
        ev = getattr(self, "_prefetch_event", None)
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
            self._prefetch_event = None

    def lookup_train(self, keys: torch.Tensor, step: int, out_dtype=torch.float32):
        self._sync_prefetch()
        self._ensure_resident(keys, pin=False)
        self._pinned = None                                    # consumed: prefetched ids may be evicted again
        return self.hbm.lookup_train(keys, step, out_dtype)

    def accumulate(self, pos, grads):
        self.hbm.accumulate(pos, grads)

    def apply_step(self, hp: OptHyper):
        self.hbm.apply_step(hp)

    def apply_raw(self, ids, grads, hp):
        self._ensure_resident(ids, pin=False)
        self.hbm.apply_raw(ids, grads, hp)

    def size(self) -> int:
        hk = self.hbm.snapshot()["keys"]
        dk = self.dram.snapshot()["keys"]
        return int(torch.unique(torch.cat([hk, dk])).numel())

    def total_keys(self) -> int:
        return self.size() + int(self.hbm.snapshot()["keys_filtered"].numel())

    def get_freq(self, keys):
        f = self.hbm.get_freq(keys)
        return torch.where(f > 0, f, self.dram.get_freq(keys))

    def get_version(self, keys):
        v = self.hbm.get_version(keys)
        return torch.where(v >= 0, v, self.dram.get_version(keys))

    def lookup_slot(self, keys, slot):
        self._ensure_resident(keys, pin=False)
        return self.hbm.lookup_slot(keys, slot)

    def lookup_tier(self, keys: torch.Tensor) -> torch.Tensor:
        """0 = HBM, 1 = DRAM only, -1 = absent (KvResourceLookupTier)."""
        k = keys.to(self.device, torch.int64).reshape(-1)
        row = torch.empty(k.numel(), dtype=torch.int32, device=self.device)
        check(self.lib.dr_cuda_table_get_meta(C.byref(self.hbm.struct), ptr(k), k.numel(), None, None, ptr(row), stream_ptr()), "get_meta")
        in_hbm = (row >= 0).cpu()
        n = k.numel()
        kc = k.cpu().contiguous()
        out = torch.full((n,), -1, dtype=torch.int64)
        if hasattr(self.dram, "lookup_tier"):                 # 3 tiers: 1 = DRAM, 2 = SSD
            lower = self.dram.lookup_tier(kc)
            out = torch.where(lower >= 0, lower + 1, out)
        else:
            out[self.dram.export_keys(kc)[3]] = 1
        out[in_hbm] = 0
        return out.view(keys.shape)

    def shrink(self, step: int) -> int:
        return self.hbm.shrink(step) + self.dram.shrink(step)

    def clear_dirty(self):
        self.hbm.clear_dirty(); self.dram.clear_dirty()

    def snapshot(self, dirty_only: bool = False, part_id: int = 0, part_num: int = 1) -> Dict[str, torch.Tensor]:
        """Merged view: HBM rows are authoritative for resident keys, DRAM for the rest."""
        h = self.hbm.snapshot(dirty_only, part_id, part_num)
        d = self.dram.snapshot(dirty_only, part_id, part_num)
        keep = ~torch.isin(d["keys"], h["keys"])
        keys = torch.cat([h["keys"], d["keys"][keep]])
        rows = torch.cat([h["rows"], d["rows"][keep]]); freqs = torch.cat([h["freqs"], d["freqs"][keep]]); vers = torch.cat([h["versions"], d["versions"][keep]])
        b = torch.remainder(keys, 1000)
        o = torch.argsort(keys, stable=True); o = o[torch.argsort(b[o], stable=True)]
        off = torch.zeros(1001, dtype=torch.int64); off[1:] = torch.cumsum(torch.bincount(b, minlength=1000), 0)
        out = dict(h)
        out.update(keys=keys[o], rows=rows[o], freqs=freqs[o], versions=vers[o], partition_offset=off)
        return out

    def import_(self, keys, rows, freqs, versions, part_id=0, part_num=1, reset_version=False) -> int:
        """Restore: everything lands in DRAM; the hottest rows (by frequency) refill tier 0 (hbm_dram_storage.h:276-306)."""
        n = self.dram.import_(keys, rows, freqs, versions, part_id, part_num, reset_version)
        if rows is not None and freqs is not None and keys.numel():
            k = keys.to(torch.int64)
            m = torch.remainder(torch.remainder(k, 1000), part_num) == part_id if part_num > 1 else torch.ones_like(k, dtype=torch.bool)
            k, f = k[m], freqs.to(torch.int64)[m]
            top = torch.topk(f, min(k.numel(), self.cache_rows // 2)).indices if k.numel() else torch.empty(0, dtype=torch.int64)
            if top.numel():
                self._promote(k[top])
        return n

    def remove(self, keys):
        return max(self.hbm.remove(keys), self.dram.remove(keys))

    def bloom_state(self):
        return self.hbm.bloom_state()

    def load_bloom_state(self, s):
        self.hbm.load_bloom_state(s)

    def cache_stats(self) -> Dict[str, float]:
        tot = max(1, self.hits + self.misses)
        return {"hits": self.hits, "misses": self.misses, "hit_rate": self.hits / tot, "hbm_rows": self.hbm.size()}
