#!/usr/bin/env python
"""Per-kernel device time of eager DLRM training steps at the bench.py configuration (one GPU, B = 65536, fresh power-law batches), from
torch.profiler with CUDA activities only, in a run of its own.  For every kernel name it prints the calls and the device microseconds per
step; the ordered batch reductions (k_det_colsum) are also split by the kernel that wrote their partials (the kernel before them on the
same stream) and that kernel's grid, which for k_colstats, k_bn_bwd_apply_v2 and k_head is the number of partial rows summed.  The summed
kernel time overlaps between the main and the side stream, so it is not the step time (benchmarks/step_timing.py gives that per phase).
Writes OUT/step_profile_trace.json (Chrome trace) and OUT/step_profile.json.  Uses only DLRMEngine.

  python benchmarks/step_profile.py OUT [--steps 10] [--warmup 5] [--batch 65536]"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def short_name(name: str) -> str:
    """Kernel name without return type, namespaces and parameter list (template arguments kept: they select different kernels)."""
    name = name.replace("(anonymous namespace)::", "").replace("drc::", "")
    name = re.sub(r"^void\s+", "", name)
    depth = 0
    for i, ch in enumerate(name):
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=65536)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    from torch.profiler import ProfilerActivity, profile

    from deeprec_b200.data.synthetic import criteo_batch
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = DLRMConfig(batch_size=a.batch, sparse_blocks_per_sm=4)          # bench.py's defaults (adagrad, side-stream embeddings)
    eng = DLRMEngine(cfg, dev)
    batches = [criteo_batch(cfg.batch_size, cfg.num_dense, cfg.cardinalities, seed=99 + i, alpha=1.05) for i in range(a.warmup + a.steps)]
    batches = [tuple(t.to(dev) for t in b) for b in batches]
    for b in batches[: a.warmup]:
        eng.load_batch(*b); eng.train_step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for b in batches[a.warmup:]:
            eng.load_batch(*b); eng.train_step()
        torch.cuda.synchronize()
    trace = os.path.join(a.out, "step_profile_trace.json")
    prof.export_chrome_trace(trace)

    with open(trace) as fh:
        events = [e for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    per_name = collections.defaultdict(lambda: [0, 0.0])
    by_producer = collections.defaultdict(lambda: [0, 0.0])
    last_on_stream = {}
    for e in sorted(events, key=lambda e: e["ts"]):
        nm, args = short_name(e["name"]), e.get("args", {})
        per_name[nm][0] += 1
        per_name[nm][1] += e["dur"]
        stream = args.get("stream")
        if "det_colsum" in nm:
            prev = last_on_stream.get(stream)
            key = f"after {prev[0]} (grid {prev[1]})" if prev else "first on its stream"
            by_producer[key][0] += 1
            by_producer[key][1] += e["dur"]
        last_on_stream[stream] = (nm, (args.get("grid") or [0])[0])
    n = a.steps

    def table(d):
        return [{"kernel": k, "calls_per_step": c / n, "us_per_step": round(t / n, 2)} for k, (c, t) in sorted(d.items(), key=lambda kv: -kv[1][1])]

    rep = {"gpu": gpu_info(), "batch": a.batch, "profiled_steps": n, "kernels": table(per_name), "det_colsum_by_producer": table(by_producer),
           "kernel_us_per_step_total": round(sum(t for _, t in per_name.values()) / n, 1),
           "det_colsum_us_per_step": round(sum(t for k, (_, t) in per_name.items() if "det_colsum" in k) / n, 2)}
    with open(os.path.join(a.out, "step_profile.json"), "w") as fh:
        json.dump(rep, fh, indent=1)
    print(f"# {rep['gpu']}  B={a.batch}  {n} eager steps profiled")
    print(f"{'calls/step':>10} {'us/step':>10}  kernel")
    for r in rep["kernels"]:
        print(f"{r['calls_per_step']:10.1f} {r['us_per_step']:10.2f}  {r['kernel'][:110]}")
    print("# k_det_colsum by producer")
    for r in rep["det_colsum_by_producer"]:
        print(f"{r['calls_per_step']:10.1f} {r['us_per_step']:10.2f}  {r['kernel'][:110]}")
    print(json.dumps({k: rep[k] for k in ("gpu", "kernel_us_per_step_total", "det_colsum_us_per_step")}))


if __name__ == "__main__":
    main()
