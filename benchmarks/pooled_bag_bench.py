#!/usr/bin/env python
"""CUDA-event timing of multi-hot bags (csrc/cuda/sparse_pipeline.cu) at world 1 on the DSSM layout (id columns [user | item | cat | hist_item x L |
hist_cat x L], bags [1, 1, 1, L, L]) after a dedup + lookup of a Taobao-shaped batch:

  * k_sp_pool against k_sp_gather on the same ids ([B, 5, D] against [B, 3 + 2 L, D]);
  * k_sp_pool_segsum on the pooled gradient against k_sp_segsum on the per-position gradient;
  * the DSSM engine step (CUDA graph) with sum bags against the same net fed by per-position columns pooled with a torch sum(1).

Every figure is the mean over --iters launches (or graph replays) after a warm-up; each pair is timed twice, alternating.  Prints the card name
and power limit and one JSON line.  python benchmarks/pooled_bag_bench.py [--batch 65536 --max_len 50]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def timed(fn, iters: int) -> float:
    """Mean microseconds of fn() over iters launches (CUDA events), after a warm-up."""
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--max_len", type=int, default=50)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    import deeprec_b200 as dr
    from deeprec_b200.data import taobao_batch
    from deeprec_b200.models.rec_engine import FusedRecEngine, _StripTables, din_ids, pooled_seq_engine
    from deeprec_b200.models.zoo import build_model
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    print(f"card: {q or torch.cuda.get_device_name(dev)}")
    B, L, D = a.batch, a.max_len, 16
    rows = (1_000_000, 4_000_000, 10_000)
    b = taobao_batch(B, L, *rows, seed=0)
    ids, y = din_ids(b).to(dev), b["labels"].to(dev)
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    pooled = pooled_seq_engine(build_model("dssm", device=dev), B, L, table_rows=rows, device=dev)
    C, F = pooled.C, pooled.deep.bags.F

    # ---- kernels: one dedup + lookup, then the requester kernels over and over within the same step (their flags stay raised)
    sp = pooled.sp
    pooled.load_batch(ids, y)
    pooled.deep.forward(pooled.ids, True)
    per_pos = torch.zeros(B, C, D, dtype=torch.bfloat16, device=dev)
    g = torch.Generator(device=dev).manual_seed(1)
    demb_pos = (torch.randn(C, B, D, device=dev, generator=g) * 1e-3).bfloat16()
    dpool = (torch.randn(F, B, D, device=dev, generator=g) * 1e-3).bfloat16()
    w, bags = pooled.deep.pool_w, pooled.deep.bags
    res = {"pool_us": [], "gather_us": [], "pool_segsum_us": [], "segsum_us": []}
    for _ in range(2):
        res["pool_us"].append(timed(lambda: sp.pool(pooled.emb_out, w, bags), a.iters))
        res["gather_us"].append(timed(lambda: sp.gather(per_pos), a.iters))
    for _ in range(2):
        res["pool_segsum_us"].append(timed(lambda: sp.pool_segsum(dpool, w, bags), a.iters))
        res["segsum_us"].append(timed(lambda: sp.segsum(demb_pos), a.iters))
    pooled.deep.backward(pooled.demb)                 # close the step: pull, apply, scratch reset
    pooled.deep.end_step()
    torch.cuda.synchronize()

    # ---- engine steps: bags against per-position columns + torch sum(1), the same DSSM net
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    net = _StripTables(build_model("dssm", device=dev))

    def fwd_pos(net, dense, emb, ids):
        u, q = emb[:, 0], torch.cat([emb[:, 1], emb[:, 2]], -1)
        hist = torch.cat([emb[:, 3:3 + L].sum(1), emb[:, 3 + L:3 + 2 * L].sum(1)], -1)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return net.inner.head(u, q, hist)
    per_col = FusedRecEngine(net, fwd_pos, [0, 1, 2] + [1] * L + [2] * L, list(rows), B, device=dev)
    for eng in (pooled, per_col):
        eng.load_batch(ids, y)
        eng.capture()
    res["step_bags_ms"], res["step_per_position_ms"] = [], []
    for _ in range(2):
        res["step_bags_ms"].append(timed(pooled.train_step, a.iters) / 1e3)
        res["step_per_position_ms"].append(timed(per_col.train_step, a.iters) / 1e3)
    print(json.dumps({"metric": "multi-hot bags, DSSM layout (CUDA events, mean over launches; two alternating runs each)", "batch": B, "max_len": L,
                      "dim": D, "id_columns": C, "bags": F, "card": q, "launches_per_step_bags": pooled.launches_per_step,
                      "launches_per_step_per_position": per_col.launches_per_step, **res}))


if __name__ == "__main__":
    main()
