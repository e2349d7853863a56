#!/usr/bin/env python
"""Per-stream timeline of DLRM training steps at the bench.py configuration (one GPU, B = 65536, fresh power-law batches): how much of the
step's two overlap windows really runs on two streams at once.  torch.profiler with CUDA activities, in a run of its own, over eager steps
and, in a second profiler session, over CUDA-graph replays (graph kernels are reported with the stream they ran on).

  forward window   fork .. f_join: the embedding forward (k_sp_dedup, k_sp_lookup) beside the bottom MLP, up to the dot-interaction kernel
  backward window  b_dot .. b_join: the embedding backward (k_sp_segsum .. k_apply) beside the bottom-MLP backward, up to k_dense_apply

For each window it reports the busy intervals of every stream (step-relative microseconds), the time both streams had a kernel running and
the time only one did.  Every main-chain GEMM (k_gemm_tn, the eleven calls of benchmarks/step_gemms.py, in the same order) gets its in-step
duration, next to its isolated time when --isolated names the JSON lines step_gemms.py printed.  The card name and power limit are read in
the same run.  Writes OUT/step_streams_{eager,graph}_trace.json (Chrome traces) and OUT/step_streams.json.

  python benchmarks/step_streams.py OUT [--steps 10] [--warmup 5] [--batch 65536] [--isolated gemms.jsonl] [--sparse-sms R]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

GEMM_CALLS = ["bot0_fwd", "bot1_fwd", "bot2_fwd", "bot3_fwd", "top0_fwd", "top1_fwd", "top1_dX", "top0_dX", "bot3_dX", "bot2_dX", "bot1_dX"]


def gpu_info() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    line = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    f = [x.strip() for x in line.split(",")] if line else [torch.cuda.get_device_name(), None, None]
    return {"name": f[0], "power_limit": f[1], "sm_clock_max": f[2]}


def union(iv):
    """Sorted, merged [start, end) intervals."""
    out = []
    for a, b in sorted(iv):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def length(iv) -> float:
    return sum(b - a for a, b in iv)


def intersect(x, y):
    out, i, j = [], 0, 0
    while i < len(x) and j < len(y):
        a, b = max(x[i][0], y[j][0]), min(x[i][1], y[j][1])
        if a < b:
            out.append([a, b])
        if x[i][1] < y[j][1]:
            i += 1
        else:
            j += 1
    return out


def clip(iv, lo, hi):
    return [[max(a, lo), min(b, hi)] for a, b in iv if b > lo and a < hi]


def analyse(trace_path: str) -> dict:
    with open(trace_path) as fh:
        ev = [e for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    ev.sort(key=lambda e: e["ts"])
    k = [(e["ts"], e["ts"] + e["dur"], e["name"], e.get("args", {}).get("stream")) for e in ev]
    ends = [i for i, x in enumerate(k) if "k_dense_apply" in x[2]]
    steps, lo = [], 0
    for hi in ends:
        seg = k[lo:hi + 1]
        lo = hi + 1
        try:
            cast = next(x for x in seg if "k_cast_pad" in x[2])
            dfwd = next(x for x in seg if "k_dot_fwd" in x[2])
            dbwd = next(x for x in seg if "k_dot_bwd" in x[2])
        except StopIteration:
            continue
        sparse_stream = next(x[3] for x in seg if "k_sp_dedup" in x[2])
        first_sp = next(x for x in seg if "k_sp_dedup" in x[2])
        t0 = min(cast[0], first_sp[0])
        windows = {"forward": (t0, dfwd[0]), "backward": (dbwd[1], seg[-1][0])}
        rec = {"step_us": seg[-1][1] - seg[0][0]}
        for wn, (a, b) in windows.items():
            streams = {}
            for x in seg:
                if x[1] > a and x[0] < b:
                    streams.setdefault(x[3], []).append([x[0], x[1]])
            busy = {s: clip(union(v), a, b) for s, v in streams.items()}
            sp = busy.get(sparse_stream, [])
            others = union([iv for s, v in busy.items() if s != sparse_stream for iv in v])
            both = length(intersect(sp, others))
            anyb = length(union(sp + others))
            rec[wn] = {"window_us": b - a, "both_us": both, "one_us": anyb - both, "idle_us": (b - a) - anyb,
                       "sparse_busy_us": length(sp), "dense_busy_us": length(others),
                       "busy": {("sparse" if s == sparse_stream else f"stream {s}"): [[round(p - seg[0][0], 1), round(q - seg[0][0], 1)] for p, q in v]
                                for s, v in busy.items()}}
        gemms = [x for x in seg if "k_gemm_tn" in x[2]]
        rec["gemm_us"] = [x[1] - x[0] for x in gemms] if len(gemms) == len(GEMM_CALLS) else None
        steps.append(rec)
    if not steps:
        raise SystemExit(f"no complete step found in {trace_path}")

    def med(f):
        return round(statistics.median(f(s) for s in steps), 1)

    out = {"steps": len(steps), "step_us": med(lambda s: s["step_us"])}
    for wn in ("forward", "backward"):
        out[wn] = {key: med(lambda s, key=key: s[wn][key]) for key in ("window_us", "both_us", "one_us", "idle_us", "sparse_busy_us", "dense_busy_us")}
        out[wn]["busy_last_step"] = steps[-1][wn]["busy"]
    g = [s["gemm_us"] for s in steps if s["gemm_us"]]
    out["gemm_in_step_us"] = {n: round(statistics.median(x[i] for x in g), 1) for i, n in enumerate(GEMM_CALLS)} if g else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--isolated", default=None, help="JSON lines of benchmarks/step_gemms.py (isolated time of each GEMM call)")
    ap.add_argument("--sparse-sms", type=int, default=None, help="DLRMConfig.sparse_sms (default: the config's default)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_streams.py profiles the step on a GPU; none is visible")
    os.makedirs(a.out, exist_ok=True)
    from torch.profiler import ProfilerActivity, profile

    from deeprec_b200.data.synthetic import criteo_batch
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    kw = {} if a.sparse_sms is None else {"sparse_sms": a.sparse_sms}
    cfg = DLRMConfig(batch_size=a.batch, sparse_blocks_per_sm=4, **kw)          # bench.py's configuration
    eng = DLRMEngine(cfg, dev)
    n = a.warmup + a.steps
    batches = [tuple(t.to(dev) for t in criteo_batch(cfg.batch_size, cfg.num_dense, cfg.cardinalities, seed=99 + i, alpha=1.05)) for i in range(2 * n + 1)]
    rep = {"gpu": info, "batch": a.batch, "sparse_sms": getattr(cfg, "sparse_sms", 0), "partition": getattr(eng, "partition_sms", None)}
    it = iter(batches)
    for mode in ("eager", "graph"):
        if mode == "graph":
            eng.load_batch(*next(it))
            eng.capture()
        for _ in range(a.warmup):
            eng.load_batch(*next(it)); eng.train_step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                eng.load_batch(*next(it)); eng.train_step()
            torch.cuda.synchronize()
        trace = os.path.join(a.out, f"step_streams_{mode}_trace.json")
        prof.export_chrome_trace(trace)
        rep[mode] = analyse(trace)
    if a.isolated:
        iso = {}
        with open(a.isolated) as fh:
            for line in fh:
                if line.startswith("{"):
                    r = json.loads(line)
                    iso[r["call"]] = r["us"]
        for mode in ("eager", "graph"):
            g = rep[mode]["gemm_in_step_us"]
            if g:
                rep[mode]["gemm_vs_isolated"] = {c: {"in_step_us": g[c], "isolated_us": iso.get(c), "ratio": round(g[c] / iso[c], 2) if iso.get(c) else None}
                                                 for c in GEMM_CALLS}
    with open(os.path.join(a.out, "step_streams.json"), "w") as fh:
        json.dump(rep, fh, indent=1)
    for mode in ("eager", "graph"):
        r = rep[mode]
        print(json.dumps({"mode": mode, "gpu": info, "sparse_sms": rep["sparse_sms"], "partition": rep["partition"], "step_us": r["step_us"],
                          **{w: {k: v for k, v in r[w].items() if k != "busy_last_step"} for w in ("forward", "backward")},
                          "gemm": r.get("gemm_vs_isolated") or r["gemm_in_step_us"]}))


if __name__ == "__main__":
    main()
