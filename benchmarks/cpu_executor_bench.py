"""Small-batch latency of the CPU Processor's op-program interpreter under the three executor policies (normal / cost_model / inline).

  python benchmarks/cpu_executor_bench.py [--threads 4] [--batches 1,8,32] >> cpu_executor_bench.jsonl

The cost-model executor helps where the program has independent branches (MMoE / PLE experts and towers, ESMM / DSSM towers) and the batch is
too small for an op to use its own team."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deeprec_b200 as dr                                                   # noqa: E402
from deeprec_b200.data import taobao_batch                                  # noqa: E402
from deeprec_b200.models.rec_engine import din_ids                          # noqa: E402
from deeprec_b200.models.zoo import build_model                             # noqa: E402
from deeprec_b200.serving import Processor, export_saved_model_program      # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", type=int, default=4)
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--models", default="mmoe,ple,esmm,dssm,din")
    ap.add_argument("--iters", type=int, default=400)
    a = ap.parse_args()
    L = 50
    for name in a.models.split(","):
        dr.embedding_variable.clear_registry()
        torch.manual_seed(0)
        model = build_model(name, device="cpu")
        root = tempfile.mkdtemp()
        export_saved_model_program(model, os.path.join(root, "v1"), version=1, root=root, max_len=L)
        b = taobao_batch(64, L, 500, 3000, 40, seed=1)
        ids = din_ids(b).numpy(); dense = np.zeros((64, 1), np.float32)
        for B in [int(x) for x in a.batches.split(",")]:
            row = {"model": name, "batch": B, "threads": a.threads}
            for pol in ("normal", "cost_model", "inline"):
                p = Processor(os.path.join(root, "v1"), {"session_num": 1, "max_batch": 64, "model_update_interval_ms": 0, "intra_op_parallelism_threads": a.threads,
                                                         "executor_policy": pol, "start_node_stats_step": 4, "stop_node_stats_step": 36}, device="cpu")
                d, i = dense[:B], np.ascontiguousarray(ids[:, :B])
                for _ in range(60):
                    p.predict(d, i)
                ts = []
                for _ in range(a.iters):
                    t0 = time.perf_counter(); p.predict(d, i); ts.append(time.perf_counter() - t0)
                ts.sort()
                row[pol + "_p50_us"] = round(ts[len(ts) // 2] * 1e6, 1); row[pol + "_p99_us"] = round(ts[int(len(ts) * 0.99)] * 1e6, 1)
                if pol == "cost_model":
                    row["plan"] = {k: v for k, v in p.model_info()["executor"].items() if k != "policy"}
                p.close()
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
