#!/usr/bin/env python
"""EmbeddingVariable storage-engine micro-benchmark (the reference's embedding_variable_performance_test.cc / _memory_test.cc):
lookup (hit / miss), lookup-or-create through the optimizer apply (fresh keys / existing keys, with dedup), snapshot (save), eviction and
resident memory per key on the host engine at N keys (default 10 M, the scale of the reference's large tests).  One JSON line per
measurement; ``--out`` appends them to a file.  CPU only (the device table is measured by bench.py).

  python benchmarks/ev_bench.py --keys 10000000 --dim 16 --batch 262144 --out cpu_ev_bench.jsonl
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deeprec_b200 as dr  # noqa: E402
from deeprec_b200.optim.optimizers import AdagradOptimizer  # noqa: E402


def rss_bytes() -> int:
    with open("/proc/self/statm") as f:
        return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")


def best(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    return min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=16)
    ap.add_argument("--batch", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--prefault_gb", type=float, default=0.0,
                    help="touch and release this much memory first: in a micro-VM whose RAM is backed on demand the first touch of a guest "
                         "page costs ~100 us (measured), which would otherwise be billed to whatever allocates fresh memory")
    a = ap.parse_args()
    threads = torch.get_num_threads()
    results = []
    if a.prefault_gb > 0:
        warm = torch.empty(int(a.prefault_gb * (1 << 30)), dtype=torch.uint8)
        warm.view(-1, 4096)[:, 0] = 1
        del warm

    def emit(name, seconds, n, **extra):
        r = {"bench": name, "keys_in_table": a.keys, "dim": a.dim, "n": n, "ms": seconds * 1e3, "ns_per_key": seconds / max(n, 1) * 1e9,
             "mkeys_per_s": n / seconds / 1e6 if seconds > 0 else 0.0, "threads": threads, **extra}
        results.append(r); print(json.dumps(r), flush=True)

    dr.embedding_variable.clear_registry()
    rss0 = rss_bytes()
    ev = dr.get_embedding_variable("bench", a.dim, ev_option=dr.EmbeddingVariableOption(
        evict_option=dr.GlobalStepEvict(steps_to_live=2), storage_option=dr.StorageOption(dr.StorageType.DRAM)), device="cpu")
    opt = AdagradOptimizer([], [ev], lr=0.01)
    table, hp = ev.table, opt._hyper(opt.param_groups[0])
    g = torch.Generator().manual_seed(0)

    # ---- fill: lookup-or-create of fresh keys through the sparse apply (one accumulator slot in the row) ----
    t_fill = 0.0
    perm_mul = 0x9E3779B97F4A7C15 & ((1 << 62) - 1)
    for s in range(0, a.keys, a.batch):
        n = min(a.batch, a.keys - s)
        ids = (torch.arange(s, s + n, dtype=torch.int64) * perm_mul) & ((1 << 62) - 1)      # scattered 62-bit keys, all distinct
        grads = torch.randn(n, a.dim, generator=g)
        hp.global_step = 1 + (s // a.batch) % 2
        t0 = time.perf_counter(); table.apply_raw(ids, grads, hp)
        t_fill += time.perf_counter() - t0
    emit("apply_create_fresh_keys", t_fill, a.keys)
    emit("resident_bytes_per_key", 0.0, 0, bytes_per_key=(rss_bytes() - rss0) / max(ev.total_count(), 1), rows=ev.total_count(),
         payload_bytes_per_key=4 * a.dim * 2 + 8)

    def keys_of(idx):
        return (idx * perm_mul) & ((1 << 62) - 1)

    hit = keys_of(torch.randint(0, a.keys, (a.batch,), generator=g))
    miss = keys_of(torch.randint(a.keys, 2 * a.keys, (a.batch,), generator=g))
    zipf = keys_of((torch.rand(a.batch, generator=g).pow(4) * a.keys).long())                # skewed: many duplicates of hot keys
    grads = torch.randn(a.batch, a.dim, generator=g)
    emit("lookup_hit_uniform", best(lambda: table.lookup(hit), a.reps), a.batch)
    emit("lookup_miss", best(lambda: table.lookup(miss), a.reps), a.batch)
    emit("lookup_hit_skewed", best(lambda: table.lookup(zipf), a.reps), a.batch)
    emit("apply_existing_uniform", best(lambda: table.apply_raw(hit, grads, hp), a.reps), a.batch)
    emit("apply_existing_skewed_dedup", best(lambda: table.apply_raw(zipf, grads, hp), a.reps), a.batch, unique=int(zipf.unique().numel()))
    emit("get_frequency", best(lambda: table.get_freq(hit), a.reps), a.batch)

    # snapshot = scan + bucket sort (begin) and the gather of keys / rows / metadata (read).  The output buffers are allocated and touched
    # BEFORE the timed region: what is measured is the engine, not the page faults of 1.3 GB of fresh memory (see --prefault_gb).
    import ctypes as C
    from deeprec_b200._native import ptr

    def timed_snapshot(name, dirty_only):
        na, nf = C.c_int64(0), C.c_int64(0)
        t0 = time.perf_counter(); table.lib.dr_host_ev_snapshot_begin(table.h, int(dirty_only), 0, 1, C.byref(na), C.byref(nf)); t_begin = time.perf_counter() - t0
        n, m = na.value, max(nf.value, 1)
        keys, rows = torch.zeros(n, dtype=torch.int64), torch.zeros(n, table.stride)
        fr, ve, po = torch.zeros(n, dtype=torch.int64), torch.zeros(n, dtype=torch.int64), torch.zeros(1001, dtype=torch.int64)
        fk, ff, fv, fpo = (torch.zeros(m, dtype=torch.int64) for _ in range(3)), None, None, torch.zeros(1001, dtype=torch.int64)
        fk, ff, fv = list(fk)
        t0 = time.perf_counter()
        table.lib.dr_host_ev_snapshot_read(table.h, ptr(keys), ptr(rows), ptr(fr), ptr(ve), ptr(po), ptr(fk), ptr(ff), ptr(fv), ptr(fpo))
        t_read = time.perf_counter() - t0
        table.lib.dr_host_ev_snapshot_end(table.h)
        emit(name, t_begin + t_read, n, begin_ms=t_begin * 1e3, read_ms=t_read * 1e3, read_gb_per_s=rows.numel() * 4 / max(t_read, 1e-9) / 1e9)
        return keys, rows, fr, ve

    def timed_restore(keys, rows, fr, ve):
        ev2 = dr.get_embedding_variable("bench_restore", a.dim, ev_option=dr.EmbeddingVariableOption(storage_option=dr.StorageOption(dr.StorageType.DRAM)), device="cpu")
        AdagradOptimizer([], [ev2], lr=0.01)                       # same row layout (one slot)
        t0 = time.perf_counter(); kept = ev2.table.import_(keys, rows, fr, ve); t = time.perf_counter() - t0
        emit("restore_import", t, int(kept), rows_after=ev2.total_count())

    snap = timed_snapshot("snapshot_full", False)
    timed_restore(*snap)
    del snap
    table.clear_dirty(); table.apply_raw(hit, grads, hp)
    timed_snapshot("snapshot_incremental", True)
    t0 = time.perf_counter(); removed = table.shrink(1000); t = time.perf_counter() - t0      # every key is older than steps_to_live
    emit("evict_global_step", t, int(removed), remaining=ev.total_count())
    if a.out:
        with open(a.out, "a") as f:
            for r in results:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
