"""Training-state checkpoints of the fused engines (:class:`models.dlrm_engine.DLRMEngine`, :class:`models.rec_engine.FusedRecEngine`).

Same contract as :class:`checkpoint.saver.Saver` / ``IncrementalSaver`` for framework-API models (reference: SaveV2/SaveV3 with EV
hooks ``core/kernels/save_restore_v2_ops.cc:158-360``, ``IncrSave`` / ``IndicesIncrRecorder`` ``kernels/incr_save_restore_ops.h:347``,
``python/training/incremental_saver.py:420-554``), applied to the engines' sharded device tables:

  * full save   = every rank writes ONE bundle ``<prefix>-<step>-part<rank>-of-<world>``: its shard of every table (keys, full-stride
                  rows = embedding + optimizer slots, frequencies, versions, un-admitted keys, 1000-bucket offsets -- the snapshot kernels
                  of csrc/cuda/table_kernels.cu), and rank 0 also the dense block (flat fp32 parameters + optimizer slots, hyper /
                  global step, BatchNorm running statistics).  GlobalStep / L2 eviction runs inside the save, as in the reference.
  * delta save  = only rows whose dirty bit was set by the apply kernel since the last (full or delta) save + the dense block.
  * restore     = any world size: every rank scans every shard file and imports the keys it owns under the CURRENT world
                  (``hash(key) % world`` -- the sharding function of the sparse pipeline), then replays the delta chain in order.
  * linear group = the dim-4 tables of ``FusedRecEngine(linear=True)`` are saved as ``linear/<t>-...`` with the same tensors as ``table/<t>-...``
                  (and restored the same way), their optimizer's hyper-parameters as ``linear/hyper``.
  * multi-tier  = tables of ``FusedRecEngine(tiered=...)`` save BOTH tiers (the HBM cache and the DRAM tier; rows demoted since the last save
                  carry their dirty bit into the DRAM tier, so delta saves stay complete) and restore each into its tier.
"""
from __future__ import annotations

import glob
import json
import os
import re
from typing import Dict, List, Optional

import torch

from .._native import OptHyper
from .saver import BundleReader, BundleWriter, _register_checkpoint

_M64 = (1 << 64) - 1



def _native_device_sync(dev) -> None:
    from .. import _native
    _native.device_sync(dev)                        # torch.cuda.synchronize on a GPU; a no-op on the CUDA-on-CPU emulation

def _lsr(x: torch.Tensor, n: int) -> torch.Tensor:
    """logical shift right of int64 bit patterns"""
    return (x >> n) & ((1 << (64 - n)) - 1)


def _mul(x: torch.Tensor, c: int) -> torch.Tensor:
    c = c & _M64
    if c >= 1 << 63:
        c -= 1 << 64
    return x * c                                      # int64 multiply wraps (two's complement), same low 64 bits as the uint64 product


def sp_owner(keys: torch.Tensor, world: int) -> torch.Tensor:
    """``hash(key) % world`` exactly as csrc/cuda/sparse_pipeline.cu::sp_owner (dr_mix64((key ^ C) ) >> 33) % W)."""
    if world <= 1:
        return torch.zeros_like(keys)
    c = 0x5bd1e9955bd1e995
    x = keys ^ c
    x = _mul(x ^ _lsr(x, 30), 0xbf58476d1ce4e5b9)
    x = _mul(x ^ _lsr(x, 27), 0x94d049bb133111eb)
    x = x ^ _lsr(x, 31)
    return _lsr(x, 33) % world


def _dense_state(eng) -> Dict[str, torch.Tensor]:
    out = {"dense/params": eng.params, "dense/hyper": eng.hp_dev}
    if eng.s0 is not None:
        out["dense/slot0"] = eng.s0
    if eng.s1 is not None:
        out["dense/slot1"] = eng.s1
    if hasattr(eng, "bot"):                              # DLRMEngine: BatchNorm running statistics live outside the flat buffer
        for L in eng.bot:
            out[f"bn/{L.name}/moving_mean"] = L.running_mean
            out[f"bn/{L.name}/moving_variance"] = L.running_var
    net = getattr(eng, "net", None)
    if net is not None:
        for k, v in net.named_buffers():
            out["buffer/" + k] = v
    for g in eng.groups:                                 # a linear group's own optimizer step / beta powers / decay (the deep group's: dense/hyper)
        if g.is_linear:
            out["linear/hyper"] = g.hp_dev
    return out


def _groups(eng):
    """(name, tables, tiers) of every embedding group of the engine: ``table`` for the deep group, ``linear`` for a linear one."""
    return [("linear" if g.is_linear else "table", g.tables, g.tiers) for g in eng.groups]


def _step_of(eng) -> int:
    raw = bytes(eng.hp_dev.cpu().numpy().tobytes())
    return int(OptHyper.from_buffer_copy(raw).global_step)


def save_engine(eng, save_path: str, incremental: bool = False, max_to_keep: int = 5) -> str:
    """Write this rank's shard; returns the bundle prefix.  Call on every rank (collectively: a barrier follows when world > 1)."""
    _native_device_sync(eng.dev)
    step, W, r = _step_of(eng), eng.world, eng.rank
    d = os.path.dirname(os.path.abspath(save_path))
    base = os.path.basename(save_path)
    if incremental:
        d = os.path.join(d, ".incr")
    os.makedirs(d, exist_ok=True)
    prefix = os.path.join(d, f"{base}-{step}-part{r:05d}-of-{W:05d}")
    w = BundleWriter(prefix)
    w.add("global_step", torch.tensor(step, dtype=torch.int64))
    w.add("meta/world", torch.tensor([W, r, int(incremental)], dtype=torch.int64))
    if r == 0:
        for k, v in _dense_state(eng).items():
            w.add(k, v)
    sfx = "sparse_incr_" if incremental else ""
    for grp, tables, tiers in _groups(eng):
        for t, tbl in tables.items():
            if not incremental and (tbl.cfg.steps_to_live > 0 or tbl.cfg.l2_weight_threshold >= 0):
                tbl.shrink(step)                                      # eviction happens inside a full save (single_tier_storage.h:235-261)
            if t in tiers:
                # multi-tier table: the HBM tier is a cache -- rows demoted to the DRAM tier are training state too (hbm_dram_storage.h:
                # Save() walks both tiers).  In-flight promotions / demotions finish first; the HBM copy of a key wins on restore (imported last).
                mgr = tiers[t][0]
                mgr.drain()
                hs = mgr.host.snapshot(dirty_only=incremental)
                w.add(f"{grp}/{t}-host-{sfx}keys", hs["keys"]); w.add(f"{grp}/{t}-host-{sfx}values", hs["rows"])
                w.add(f"{grp}/{t}-host-{sfx}freqs", hs["freqs"]); w.add(f"{grp}/{t}-host-{sfx}versions", hs["versions"])
            s = tbl.snapshot(dirty_only=incremental)
            w.add(f"{grp}/{t}-{sfx}keys", s["keys"]); w.add(f"{grp}/{t}-{sfx}values", s["rows"])
            w.add(f"{grp}/{t}-{sfx}freqs", s["freqs"]); w.add(f"{grp}/{t}-{sfx}versions", s["versions"])
            w.add(f"{grp}/{t}-{'incr_' if incremental else ''}partition_offset", s["partition_offset"])
            w.add(f"{grp}/{t}-{sfx}keys_filtered", s["keys_filtered"]); w.add(f"{grp}/{t}-{sfx}freqs_filtered", s["freqs_filtered"])
            w.add(f"{grp}/{t}-{sfx}versions_filtered", s["versions_filtered"])
            bloom = tbl.bloom_state()
            if bloom is not None and not incremental:
                w.add(f"{grp}/{t}-bloom", bloom)
    w.close()
    for _, tables, tiers in _groups(eng):
        for tbl in tables.values():
            tbl.clear_dirty()                                     # the recorder restarts at every (full or delta) save
        for mgr, _ in tiers.values():
            mgr.host.clear_dirty()
    if W > 1:
        import torch.distributed as dist
        dist.barrier()
    if not incremental:
        _register_checkpoint(d, prefix, step, base, max_to_keep)
        if r == 0:                                                # a new full checkpoint starts a new delta chain
            for f in glob.glob(os.path.join(d, ".incr", f"{base}-*")):
                os.remove(f)
    return prefix


def _shards(directory: str, base: str, step: int) -> List[str]:
    pat = re.compile(re.escape(base) + rf"-{step}-part(\d+)-of-(\d+)\.index$")
    return sorted(os.path.join(directory, f[:-len(".index")]) for f in os.listdir(directory) if pat.match(f))


def latest_engine_step(directory: str, base: str, incremental: bool = False) -> Optional[int]:
    d = os.path.join(directory, ".incr") if incremental else directory
    if not os.path.isdir(d):
        return None
    steps = [int(m.group(1)) for f in os.listdir(d) if (m := re.match(re.escape(base) + r"-(\d+)-part00000-of-\d+\.index$", f))]
    return max(steps) if steps else None


def _load_tables(eng, prefixes: List[str], incremental: bool) -> int:
    W, r = eng.world, eng.rank
    sfx = "sparse_incr_" if incremental else ""
    n = 0
    for p in prefixes:
        rd = BundleReader(p)
        for grp, tables, tiers in _groups(eng):
            for t, tbl in tables.items():
                hk = f"{grp}/{t}-host-{sfx}keys"
                if rd.has(hk):                                    # DRAM-tier rows of a multi-tier table
                    hkeys = rd.read(hk)
                    if hkeys.numel():
                        mine = sp_owner(hkeys, W) == r
                        if bool(mine.any()):
                            rows, fr, ve = rd.read(f"{grp}/{t}-host-{sfx}values")[mine], rd.read(f"{grp}/{t}-host-{sfx}freqs")[mine], rd.read(f"{grp}/{t}-host-{sfx}versions")[mine]
                            if t in tiers:
                                if incremental:                   # demoted since the base checkpoint: the HBM copy an earlier bundle restored is
                                    tbl.remove(hkeys[mine])       # stale, and the HBM tier is authoritative -- drop it before the DRAM-tier import
                                n += tiers[t][0].host.import_(hkeys[mine], rows, fr, ve)
                            else:                                 # restored into an engine without the DRAM tier: everything lives in HBM
                                n += tbl.import_(hkeys[mine], rows, fr, ve)
                kk = f"{grp}/{t}-{sfx}keys"
                if not rd.has(kk):
                    continue
                keys = rd.read(kk)
                if keys.numel():
                    mine = sp_owner(keys, W) == r
                    if bool(mine.any()):
                        n += tbl.import_(keys[mine], rd.read(f"{grp}/{t}-{sfx}values")[mine], rd.read(f"{grp}/{t}-{sfx}freqs")[mine],
                                         rd.read(f"{grp}/{t}-{sfx}versions")[mine])
                fk = rd.read(f"{grp}/{t}-{sfx}keys_filtered")
                if fk.numel():
                    mine = sp_owner(fk, W) == r
                    if bool(mine.any()):
                        tbl.import_(fk[mine], None, rd.read(f"{grp}/{t}-{sfx}freqs_filtered")[mine], rd.read(f"{grp}/{t}-{sfx}versions_filtered")[mine])
                if rd.has(f"{grp}/{t}-bloom") and len(prefixes) == W:      # counting-Bloom state is per shard: only same-world restores reuse it
                    if p.endswith(f"-part{r:05d}-of-{W:05d}"):
                        tbl.load_bloom_state(rd.read(f"{grp}/{t}-bloom"))
        rd.close()
    return n


def _load_dense(eng, prefix0: str) -> None:
    rd = BundleReader(prefix0)
    for k, v in _dense_state(eng).items():
        if rd.has(k):
            x = rd.read(k).to(v.device)
            if k == "dense/hyper" and x.numel() < v.numel():     # written before dense_decay_power joined DrOptHyper: it restarts at 0
                v.zero_()
                v[:x.numel()].copy_(x.view(-1))
            else:
                v.copy_(x.view_as(v))
    rd.close()
    if hasattr(eng, "_pack_weights"):
        eng._pack_weights()                                        # bf16 shadows of the restored fp32 master weights


def restore_engine(eng, save_path: str, step: Optional[int] = None, replay_incremental: bool = True) -> int:
    """Restore the newest (or the given) full checkpoint written under ``save_path`` by ANY world size, then replay newer deltas.
    Returns the global step the engine continues from."""
    d, base = os.path.dirname(os.path.abspath(save_path)), os.path.basename(save_path)
    step = step if step is not None else latest_engine_step(d, base)
    if step is None:
        raise FileNotFoundError(f"no engine checkpoint {save_path}-*")
    shards = _shards(d, base, step)
    if not shards:
        raise FileNotFoundError(f"no shards for {save_path}-{step}")
    _load_dense(eng, shards[0])
    n = _load_tables(eng, shards, incremental=False)
    last = step
    if replay_incremental and os.path.isdir(os.path.join(d, ".incr")):
        di = os.path.join(d, ".incr")
        steps = sorted({int(m.group(1)) for f in os.listdir(di) if (m := re.match(re.escape(base) + r"-(\d+)-part\d+-of-\d+\.index$", f))})
        for s in steps:
            if s <= step:
                continue
            sh = _shards(di, base, s)
            _load_dense(eng, sh[0])
            n += _load_tables(eng, sh, incremental=True)
            last = s
    for _, tables, _ in _groups(eng):
        for tbl in tables.values():
            tbl.clear_dirty()
    _native_device_sync(eng.dev)
    return last
