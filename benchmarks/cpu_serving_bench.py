#!/usr/bin/env python
"""CPU Processor benchmark (the reference deploys its processor on CPU hosts): DLRM p50 / p99 latency and samples/s through the native CPU
runtime's C ABI, for a few (sessions, client threads, batch) operating points.  Prints one JSON line per point.

  python benchmarks/cpu_serving_bench.py [--out cpu_serving_bench.jsonl]
"""
import argparse
import json
import os
import sys
import tempfile
import threading
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deeprec_b200 as dr  # noqa: E402
from deeprec_b200.data import criteo_batch  # noqa: E402
from deeprec_b200.models.dlrm_engine import CRITEO_KAGGLE_CARDINALITIES as CARDS  # noqa: E402
from deeprec_b200.models.zoo import build_model  # noqa: E402
from deeprec_b200.serving import Processor, encode_request, export_saved_model_module  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--model", default="dlrm", help="dlrm (native architecture) or an op-program model: wdl, deepfm, dcn, dcnv2, masknet; din, dssm, esmm, mmoe, dbmtl, ple, simple_multitask (Taobao-shaped, 50-step history)")
    a = ap.parse_args()
    torch.manual_seed(0)
    from deeprec_b200.models.zoo import TAOBAO_MODELS
    taobao = a.model in TAOBAO_MODELS                    # din, dssm, esmm, mmoe, dbmtl, ple, simple_multitask: 3 + 2 L id columns, L = 50
    L = 50
    root = tempfile.mkdtemp()
    if taobao:
        from deeprec_b200.data import taobao_batch
        from deeprec_b200.models.rec_engine import din_ids
        from deeprec_b200.serving import export_saved_model_program
        model = build_model(a.model, device="cpu")
        opt = dr.optim.AdagradOptimizer(model, lr=0.05)
        for s in range(4):
            b = taobao_batch(2048, L, 100000, 400000, 1000, seed=s)
            loss = model.loss(b); opt.zero_grad(); loss.backward(); opt.step()
        export_saved_model_program(model, root + "/v1", version=4, max_len=L)

        def request(batch, seed):
            b = taobao_batch(batch, L, 100000, 400000, 1000, seed=seed)
            return encode_request(np.zeros((batch, 1), np.float32), din_ids(b).numpy())
    else:
        model = build_model(a.model, device="cpu", cardinalities=CARDS)
        opt = dr.optim.AdagradOptimizer(model, lr=0.05)
        for s in range(4):
            d, ids, y = criteo_batch(2048, 13, CARDS, seed=s)
            loss = model.loss(d, ids, y); opt.zero_grad(); loss.backward(); opt.step()
        if a.model == "dlrm":
            export_saved_model_module(model, root + "/v1", version=4)
        else:
            from deeprec_b200.serving import export_saved_model_program
            export_saved_model_program(model, root + "/v1", version=4)

        def request(batch, seed):
            return encode_request(*[x.numpy() for x in criteo_batch(batch, 13, CARDS, seed=seed)[:2]])
    lines = []
    points = ((1, 1, 1, 4000, 0), (4, 4, 1, 8000, 0), (4, 4, 32, 3000, 0), (2, 2, 256, 600, 0), (1, 1, 2048, 60, 0),
              (2, 16, 1, 16000, 0), (2, 16, 1, 16000, 32))        # many concurrent single-row callers: without / with request batching
    for sessions, threads, batch, n, batching in points:
        cfg = {"session_num": sessions, "max_batch": max(256, batch), "model_update_interval_ms": 0}
        if batching:
            cfg.update(enable_batching=True, batching_parameters={"max_batch_size": batching, "batch_timeout_micros": 100})
        proc = Processor(root + "/v1", cfg, device="cpu")
        reqs = [request(batch, 100 + i) for i in range(8)]
        for r in reqs:
            assert proc.process(r)[0] == 200
        lat = [[] for _ in range(threads)]

        def client(i):
            for k in range(n // threads):
                t0 = time.perf_counter()
                rc, _ = proc.process(reqs[(i + k) % 8])
                lat[i].append((time.perf_counter() - t0) * 1e3)
                assert rc == 200
        ts = [threading.Thread(target=client, args=(i,)) for i in range(threads)]
        t0 = time.perf_counter()
        [t.start() for t in ts]; [t.join() for t in ts]
        wall = time.perf_counter() - t0
        v = np.sort(np.concatenate([np.array(x) for x in lat]))
        rec = {"metric": f"{a.model} serving, native CPU Processor (C ABI)", "sessions": sessions, "client_threads": threads, "batch": batch, "requests": int(v.size),
               "qps": v.size / wall, "samples_per_s": v.size * batch / wall, "p50_ms": float(v[v.size // 2]), "p99_ms": float(v[min(v.size - 1, int(v.size * 0.99))]),
               "vcpus": os.cpu_count(), "dtype": "fp32", "batching_max_batch_size": batching}
        if batching:
            rec["merged"] = proc.model_info()["batching"]
        print(json.dumps(rec), flush=True)
        lines.append(json.dumps(rec))
        proc.close()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
