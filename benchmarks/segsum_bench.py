#!/usr/bin/env python
"""k_sp_segsum alone on the bench.py batch (B = 65536, Criteo-Terabyte-shaped power-law ids, alpha 1.05, dim 16): the real k_sp_dedup
builds invT, then the gradient pre-reduction is timed with CUDA events (median of --iters launches) on every SM and inside a green context
of --sparse-sms SMs (the DLRM step's sparse partition, with grids sized to it as the engine sizes them).

It also prints what the kernel has to send to L2, counted from the same ids: the (32-sample tile, key) groups, the scalar 8-byte reductions
one lane per group would issue, the 32-byte sectors of one coalesced row per group, and the lower bound of one row per distinct key; and a
SHA-256 of the ugrad rows ordered by (column, id), so that two builds can be compared bit for bit.

  python benchmarks/segsum_bench.py [--batch 65536] [--dim 16] [--seed 107] [--iters 50] [--sparse-sms R]"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def request_counts(ids: np.ndarray, dim: int) -> dict:
    """L2 reduction requests of one segsum over ids [C][B] (no padding in the bench's stream), counted on the host."""
    Cn, B = ids.shape
    col = np.repeat(np.arange(Cn, dtype=np.int64), B)
    b = np.tile(np.arange(B, dtype=np.int64), Cn)
    key = ids.reshape(-1)
    sectors_per_row = dim * 8 // 32
    tile = col * ((B + 31) // 32) + b // 32
    block = col * ((B + 255) // 256) + b // 256
    n_keys = np.unique(col * (1 << 40) + key).size
    n_groups = np.unique(np.stack([tile, key], 1), axis=0).shape[0]
    n_block_groups = np.unique(np.stack([block, key], 1), axis=0).shape[0]
    return {"ids": int(key.size), "distinct_keys": int(n_keys), "tile_key_groups": int(n_groups),
            "scalar_8B_reductions": int(n_groups * dim), "sectors_one_row_per_group": int(n_groups * sectors_per_row),
            "sectors_one_row_per_block_group": int(n_block_groups * sectors_per_row), "sectors_one_row_per_key": int(n_keys * sectors_per_row)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=16)
    ap.add_argument("--seed", type=int, default=107)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--sparse-sms", type=int, default=None, help="SMs of the green context (default: DLRMConfig.sparse_sms)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("segsum_bench.py times a kernel on a GPU; none is visible")
    from deeprec_b200 import _native
    from deeprec_b200.data.synthetic import criteo_batch
    from deeprec_b200.models.dlrm_engine import CRITEO_TB_CARDINALITIES, DLRMConfig
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _native.cuda()
    cards = list(CRITEO_TB_CARDINALITIES)
    Cn, B, D = len(cards), a.batch, a.dim
    _, ids, _ = criteo_batch(B, 13, cards, seed=a.seed, alpha=1.05)
    counts = request_counts(ids.numpy(), D)
    g = torch.Generator().manual_seed(a.seed)
    demb = (torch.randn(Cn, B, D, generator=g) * 1e-3).bfloat16().to(dev)          # per-sample gradient rows, feature-major
    lib.dr_cuda_set_sparse_blocks_per_sm(4)                                         # bench.py's --sparse-blocks
    sp = SparsePipeline(dev, 0, 1, list(range(Cn)), Cn, B, D)
    ids_d = ids.to(dev)
    sp.dedup(ids_d)
    sp.segsum(demb)                                                                 # ugrad rows were zeroed by the dedup: one clean sum
    torch.cuda.synchronize()
    invT = sp.invT.cpu().numpy()
    ck = (np.arange(Cn, dtype=np.int64)[:, None] << 40) + ids.numpy()
    order_keys, first = np.unique(ck.reshape(-1), return_index=True)
    rows = sp.ugrad.cpu().numpy()[invT.reshape(-1)[first]]
    digest = hashlib.sha256(order_keys.tobytes() + rows.tobytes()).hexdigest()

    def time_on(stream, grid_sms):
        lib.dr_cuda_set_sparse_sms(grid_sms)
        ts = []
        with torch.cuda.stream(stream):
            for _ in range(5):
                sp.segsum(demb)
            for _ in range(a.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); sp.segsum(demb); e1.record()
                e1.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3)
        lib.dr_cuda_set_sparse_sms(0)
        return statistics.median(ts)

    us_all = time_on(torch.cuda.current_stream(dev), 0)
    R = a.sparse_sms if a.sparse_sms is not None else DLRMConfig.sparse_sms
    info, h = (C.c_int * 2)(), (C.c_void_p * 5)()
    if lib.dr_cuda_sm_partition(dev.index, R, info, h) != 0:
        raise SystemExit(f"no green context of {R} SMs on this device")
    us_part = time_on(torch.cuda.ExternalStream(h[0], device=dev), info[0])
    sp.reset(); sp.step_end()
    torch.cuda.synchronize()
    print(json.dumps({"gpu": gpu_info(), "batch": B, "dim": D, "seed": a.seed, "requests": counts,
                      "segsum_us_all_sms": round(us_all, 1), "segsum_us_partition": round(us_part, 1), "partition_sms": info[0],
                      "ugrad_sha256": digest}))


if __name__ == "__main__":
    main()
