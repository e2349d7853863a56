#!/usr/bin/env python
"""CUDA-event timing of the linear (wide) embedding group's kernels, k_sp_linear_fwd and k_sp_linear_bwd (csrc/cuda/sparse_pipeline.cu), at
world 1 after a dedup + lookup of a Criteo-shaped batch.  Prints one JSON line.  python benchmarks/linear_group_bench.py [--batch 65536 --cols 26]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--cols", type=int, default=26)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    from deeprec_b200.data import criteo_batch
    from deeprec_b200.models.rec_engine import FusedRecEngine
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, C = a.batch, a.cols
    cards = [1_000_000] * C
    eng = FusedRecEngine(torch.nn.Linear(1, 1), lambda net, dense, emb, ids, linear: linear, list(range(C)), cards, B, linear=True, device=dev)
    _, ids, _ = criteo_batch(B, 13, cards, seed=0)
    eng.ids.copy_(ids.to(dev))
    sp = eng.linear.sp
    sp.dedup(eng.ids)
    sp.lookup(eng.linear.ctx, eng.linear.tmap, False)
    dl = torch.randn(B, device=dev) / B
    out = eng.lin_out

    def timed(fn):
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.iters * 1e3

    fwd_us = timed(lambda: sp.linear_fwd(out))
    bwd_us = timed(lambda: sp.linear_bwd(dl))
    uniq = sp.unique_count()
    # bytes the kernels must move: fwd reads inv (4 B per id), one 8 B row load per id (L2-resident unique rows) and writes 4 B per sample;
    # bwd reads invT (4 B per id) and dlogit (4 B per id, L1/L2-shared) and adds 8 B per distinct key at least
    fwd_bytes = B * C * 4 + B * 4
    bwd_bytes = B * C * 4 + B * 4 + uniq * 8
    print(json.dumps({"metric": "linear group kernels (CUDA events, mean over launches)", "batch": B, "cols": C, "unique_keys": uniq,
                      "linear_fwd_us": fwd_us, "linear_bwd_us": bwd_us, "linear_fwd_GBps_min_bytes": fwd_bytes / fwd_us / 1e3,
                      "linear_bwd_GBps_min_bytes": bwd_bytes / bwd_us / 1e3, "gpu": torch.cuda.get_device_name(dev)}))
    sp.reset(); sp.step_end()


if __name__ == "__main__":
    main()
