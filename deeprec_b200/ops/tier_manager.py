"""Native multi-tier storage manager: HBM cache tier (DeviceTable) over the host DRAM tier (HostTable / dr::HostEV), driven by
csrc/cuda/tier_kernels.cu -- device-side miss list, pinned staging, side-stream H2D import, histogram-threshold LFU / LRU eviction with
D2H write-back, and ONE C++ background thread (the EvictionManager / prefetch worker).  Python makes two C calls per step
(``prefetch`` one batch ahead, ``commit`` at the step boundary) and never synchronises with the device.

Reference: multi_tier_storage.h:45-330, hbm_dram_storage.h:229-306, cache.h:133,272 (LRU/LFU + prefetch lists), eviction_manager.h:39-131.
"""
from __future__ import annotations

import copy
import ctypes as C
from typing import Dict, Optional

import torch

from .. import _native
from .._native import EvConfig, check, ptr, stream_ptr
from ..embedding_variable import HostTable
from .device_table import DeviceTable

vp, i64 = C.c_void_p, C.c_int64


class DeviceTierManager:
    """``table``: the HBM tier (its row slab is the cache: ``cache_rows`` rows + head-room for one step's new keys).
    ``host``: the DRAM tier (created here when omitted; admission / eviction policies stay with tier 0).
    ``comm`` (world > 1, row-wise model parallelism): ``table`` is this rank's shard -- the keys with ``dr_sp_owner(key, W) == rank`` -- and so is
    the DRAM tier; ``prefetch`` takes the rank's OWN next-batch ids (``ids_per_prefetch`` of them on every rank) and the kernels find the keys
    this rank owns in every rank's list over peer memory (collective: every rank calls ``prefetch`` / ``commit`` once per step)."""

    def __init__(self, table: DeviceTable, cache_rows: int, host: Optional[HostTable] = None, strategy: int = 0, max_batch_keys: int = 1 << 20,
                 evict_chunk: Optional[int] = None, pad_key: int = -1, low_watermark: float = 0.85, comm=None, ids_per_prefetch: int = 0):
        self.table, self.cache_rows, self.strategy, self.pad_key = table, int(cache_rows), int(strategy), int(pad_key)
        self.comm = comm if (comm is not None and getattr(comm, "world", 1) > 1) else None
        self.world, self.rank = (self.comm.world, self.comm.rank) if self.comm is not None else (1, 0)
        self.n_sym = int(ids_per_prefetch)
        self.dev = table.device
        if host is None:
            hc = EvConfig.from_buffer_copy(bytes(table.cfg))
            hc.filter_type, hc.filter_freq = 0, 0            # the host tier stores what it is given
            hc.steps_to_live, hc.l2_weight_threshold = 0, -1.0
            hc.storage_type = 0
            host = HostTable(hc, table.default_matrix.cpu())
        if host.stride != table.stride:
            raise ValueError(f"tier row layouts differ: host stride {host.stride}, device stride {table.stride}")
        self.host = host
        self.lib = _native.cuda()
        hl = _native.host()
        fexp = C.cast(hl.dr_host_ev_export_keys, vp)
        fimp = C.cast(hl.dr_host_ev_import, vp)
        self.evict_chunk = int(evict_chunk or max(4096, self.cache_rows // 8))
        self.low = int(self.cache_rows * low_watermark)
        self.emu = _native.emu_active()                                  # CPU CI: the kernels and the manager thread on the CUDA-on-CPU emulation
        if not self.emu:
            _native.set_device(self.dev.index)
        self.h = self.lib.dr_tier_create(vp(host.h), fexp, fimp, table.stride, int(max_batch_keys), self.evict_chunk, self.dev.index or 0)
        if not self.h:
            raise RuntimeError("dr_tier_create failed")
        self.side = None if self.emu else torch.cuda.Stream(device=self.dev)
        self._count = torch.zeros(1, dtype=torch.int32)                   # admitted-row count of the HBM tier, refreshed asynchronously
        if not self.emu:
            self._count = self._count.pin_memory()
        self._epoch = 0
        self._keep = None
        self._purged_at = 0
        if self.comm is not None:
            if self.n_sym <= 0:
                raise ValueError("world > 1: ids_per_prefetch (ids handed to prefetch() per rank per step) is required")
            self.ids_sym = self.comm.symmetric(2 * self.n_sym * 8)       # [parity][n] int64, read in place by every peer's probe kernel
            self.flags_sym = self.comm.symmetric(64)                      # uint32 [16]: flags[r] = last epoch rank r published
            self.ids_sym.tensor(torch.int64, (2 * self.n_sym,)).fill_(self.pad_key)
            self.flags_sym.tensor(torch.int32, (16,)).zero_()
            self.comm.host_barrier()

    def close(self) -> None:
        if self.h:
            if not self.emu:
                torch.cuda.synchronize(self.dev)
            self.lib.dr_tier_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- per-step protocol --------------------------------------------------------------------------------------------------
    def prefetch(self, keys: torch.Tensor) -> None:
        """Called with the ids of the NEXT batch (device tensor, duplicates / padding allowed) while the current step runs: probes on a
        side stream, pins the hits, hands the misses to the background thread."""
        k = keys.reshape(-1)
        assert (k.is_cuda or self.emu) and k.dtype == torch.int64 and k.is_contiguous()
        self._keep = k                                                   # alive until the probe kernel has run (commit)
        if self.side is not None:
            self.side.wait_stream(torch.cuda.current_stream(self.dev))   # the ids were produced on the caller's stream
        side = vp(self.side.cuda_stream) if self.side is not None else None
        if self.comm is not None:
            if k.numel() != self.n_sym:
                raise ValueError(f"world > 1: prefetch() takes exactly ids_per_prefetch = {self.n_sym} ids per rank (got {k.numel()}; pad with pad_key)")
            rc = self.lib.dr_tier_prefetch_mp(self.h, C.byref(self.table.struct), ptr(k), k.numel(), self.pad_key, self._epoch + 1,
                                              self.ids_sym.peers_ref(), self.flags_sym.peers_ref(), self.world, self.rank, side)
        else:
            rc = self.lib.dr_tier_prefetch(self.h, C.byref(self.table.struct), ptr(k), k.numel(), self.pad_key, self._epoch + 1, side)
        if rc != 0:
            raise RuntimeError(f"dr_tier_prefetch failed ({rc}): commit() the previous batch first")

    def commit(self, step: int) -> int:
        """Step boundary (before the step that consumes the prefetched batch is launched): promoted rows are imported on the current
        stream; cold rows are demoted when the slab passed its high watermark.  Returns the number of promoted rows."""
        s = stream_ptr(self.dev)
        self._epoch += 1
        n = int(self.lib.dr_tier_commit(self.h, C.byref(self.table.struct), self._epoch, s))
        if n < 0:
            raise RuntimeError(f"dr_tier_commit failed ({n})")
        resident = int(self._count[0])                                   # one step stale by construction: the slab has head-room for that
        if resident > self.cache_rows:
            need = min(self.evict_chunk, resident - self.low)
            rc = self.lib.dr_tier_evict(self.h, C.byref(self.table.struct), need, self._epoch, int(step), self.strategy, s)
            if rc != 0:
                raise RuntimeError(f"dr_tier_evict failed ({rc})")
        self._count.copy_(self.table.counters[3:4], non_blocking=True)   # async D2H of the admitted-row counter (read at the next commit)
        # evicted keys leave tombstones in the open-addressing table: re-hash (device kernel, at this step boundary) when they pile up
        demoted = self.stats()["demoted_rows"]
        if (demoted - self._purged_at) * 4 > self.table.capacity:
            self.drain()
            self.table._purge_tombstones()
            self.table.ctx.structs()
            self._purged_at = demoted
        return n

    def lookup(self, keys: torch.Tensor) -> torch.Tensor:
        """Rows of `keys` wherever they live (HBM tier authoritative, else DRAM tier, else the default row) -- inspection / tests."""
        self.drain()
        k = keys.to(self.dev, torch.int64).reshape(-1)
        row = torch.empty(k.numel(), dtype=torch.int32, device=self.dev)
        check(self.lib.dr_cuda_table_get_meta(C.byref(self.table.struct), ptr(k), k.numel(), None, None, ptr(row), stream_ptr()), "get_meta")
        out = self.table.lookup(k)
        in_hbm = (row >= 0)
        kc = k.cpu()
        rows, _, _, found = self.host.export_keys(kc)
        sel = (~in_hbm.cpu()) & found
        if bool(sel.any()):
            out[sel.to(self.dev)] = rows[sel][:, : self.table.dim].to(self.dev)
        return out

    def drain(self) -> None:
        if not self.emu:
            torch.cuda.synchronize(self.dev)
        self.lib.dr_tier_drain(self.h)

    def stats(self) -> Dict[str, float]:
        out = (i64 * 8)()
        self.lib.dr_tier_stats(self.h, out)
        hits, misses = out[0], out[1]
        return {"hits": int(hits), "misses": int(misses), "hit_rate": hits / max(1, hits + misses), "promoted_rows": int(out[2]), "demoted_rows": int(out[3]),
                "h2d_bytes": int(out[4]), "d2h_bytes": int(out[5]), "evict_passes": int(out[6]), "hbm_rows": int(self._count[0]),
                "dram_rows": int(self.host.size())}
