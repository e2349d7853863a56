#!/usr/bin/env python
"""CPU stand-alone training throughput of every zoo model -- the one benchmark the reference PUBLISHES in samples/s
(BASELINE.md section B: modelzoo/*/README.md, batch 2048, Alibaba ecs.g8i.4xlarge = 16 vCPU Xeon Platinum 8475B).

  python benchmarks/cpu_zoo_bench.py [--models dlrm,deepfm,...] [--dtype fp32|bf16|both] [--out cpu_zoo_bench.json]

Method: synthetic Criteo- / Taobao-shaped batches generated up front, W warm-up steps, then R repetitions of K timed steps (forward,
backward, optimizer step incl. the sparse EmbeddingVariable apply); the BEST repetition is reported (the box is shared; the reference
reports the mean of a long run on a dedicated VM).  bf16 = ``torch.autocast('cpu', bfloat16)`` (AMX on Sapphire Rapids), the analogue
of the reference's "DeepRec fp32+bf16" column.  The published numbers were measured on 16 vCPUs; the vCPU count of this box is
recorded next to every ratio.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deeprec_b200 as dr  # noqa: E402
from deeprec_b200.data import criteo_batch, taobao_batch  # noqa: E402
from deeprec_b200.models.zoo import TAOBAO_MODELS, build_model  # noqa: E402
from deeprec_b200.optim import make_optimizer  # noqa: E402

# BASELINE.md section B: (community TF fp32, DeepRec fp32, DeepRec fp32+bf16) samples/s on 16 vCPU
PUBLISHED = {
    "dlrm": (110607.49, 129766.90, 141266.06), "deepfm": (61230.80, 74380.35, 95107.32), "din": (18522.65, 59160.78, 59651.75),
    "wdl": (32605.25, 38533.30, 82485.07), "dssm": (98357.70, 182120.67, 191525.84), "dien": (6327.50, 10094.21, 11565.63),
    "esmm": (90890.15, 170830.50, 202675.93), "dbmtl": (63220.87, 77383.54, 137581.54), "mmoe": (67189.94, 105387.94, 142645.17),
    "simple_multitask": (109859.81, 216999.25, 282453.56), "bst": (16924.47, 22143.04, 28686.70), "dcn": (24524.91, 31917.35, 55753.15),
    "ple": (21182.44, 28608.60, 33542.94), "masknet": None, "dcnv2": None,
}


def bench(name: str, batch: int, steps: int, warmup: int, reps: int, bf16: bool, optimizer: str) -> dict:
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    cards = [1000] * 26
    model = build_model(name, dr.EmbeddingVariableOption(), torch.device("cpu"), False, cardinalities=cards)
    opt = make_optimizer(optimizer, model, lr=0.01)
    taobao = name in TAOBAO_MODELS
    gen = (lambda s: taobao_batch(batch, 20, 100000, 200000, 1000, seed=s)) if taobao else (lambda s: criteo_batch(batch, 13, cards, seed=s))
    batches = [gen(s) for s in range(warmup + steps)]

    def step(b):
        with torch.autocast("cpu", dtype=torch.bfloat16, enabled=bf16):
            loss = model.loss(b) if taobao else model.loss(*b)
        opt.zero_grad(); loss.backward(); opt.step()
        return loss

    for b in batches[:warmup]:
        step(b)
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        for b in batches[warmup:]:
            loss = step(b)
        best = min(best, (time.perf_counter() - t0) / steps)
    return {"model": name, "dtype": "bf16" if bf16 else "fp32", "batch": batch, "ms_per_step": best * 1e3, "samples_per_s": batch / best,
            "final_loss": float(loss.detach())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=",".join(PUBLISHED))
    ap.add_argument("--dtype", default="both", choices=["fp32", "bf16", "both"])
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--optimizer", default="adagrad")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    vcpus = os.cpu_count()
    rows = []
    for name in a.models.split(","):
        for bf16 in ([False, True] if a.dtype == "both" else [a.dtype == "bf16"]):
            r = bench(name, a.batch, a.steps, a.warmup, a.reps, bf16, a.optimizer)
            pub = PUBLISHED.get(name)
            if pub:
                ref = pub[2] if bf16 else pub[1]
                r.update(published_deeprec_16vcpu=ref, ratio=r["samples_per_s"] / ref, ratio_per_vcpu=(r["samples_per_s"] / vcpus) / (ref / 16),
                         published_stock_tf_16vcpu=pub[0])
            r["vcpus"] = vcpus
            rows.append(r)
            print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"threads": torch.get_num_threads(), "vcpus": vcpus, "cpu": _cpu_name(), "results": rows}, f, indent=1)


def _cpu_name() -> str:
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return "unknown"


if __name__ == "__main__":
    main()
