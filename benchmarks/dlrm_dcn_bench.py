#!/usr/bin/env python
"""DLRM-DCNv2 training step on DLRMEngine at MLPerf shapes, and one low-rank cross layer against a torch autograd composite.

  python benchmarks/dlrm_dcn_bench.py [--batch 65536] [--steps 20] [--warmup 5] [--layer-iters 20] [--skip-layer]

Step: bottom 512-256-128 (+BatchNorm), 26 tables of dim 128 with Criteo-Terabyte cardinalities, x0 = [bottom | 26 rows] (3456 wide), 3 low-rank
cross layers of rank 512, top 1024-1024-512-256, logit; Adagrad; one CUDA graph per step; every prefill, warm-up and timed step takes a batch
never seen before (pre-generated into pinned memory, copied to the device before timing).  Reports device-timed ms/step and samples/s,
launches and new keys per step, the GEMM FLOP of one step counted from the shapes, and that count over the step time as a whole-step rate.

Layer: x_{l+1} = x0 * (x_l V^T W^T + b) + x_l forward and backward at [B, 3456], rank 512, through the engine's kernels (plain GEMM, cross
epilogue GEMM, k_cross_bwd, two dW GEMMs, dt GEMM, residual epilogue GEMM) and through torch autograd under bf16 autocast (cuBLAS); both
timed with CUDA events and their outputs compared.  Prints one JSON line; the card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gemm_flops(cfg, B: int) -> dict:
    """FLOP of the step's GEMMs from the shapes (2 per multiply-add): forward, weight gradients and input gradients."""
    f = {"bottom": 0, "cross": 0, "top": 0}
    k = cfg.num_dense
    for i, n in enumerate(cfg.mlp_bot):
        f["bottom"] += 2 * B * k * n * (2 if i == 0 else 3)      # fwd + dW (+ dX, except the first layer)
        k = n
    N, r = (len(cfg.cardinalities) + 1) * cfg.embedding_dim, cfg.dcn_low_rank_dim
    f["cross"] = cfg.dcn_num_layers * 12 * B * N * r             # fwd: 2 GEMMs; bwd: dW, dt, dV, dx_l
    k = N
    for n in cfg.mlp_top:
        f["top"] += 3 * 2 * B * k * n                            # fwd + dW + dX
        k = n
    f["total"] = sum(f.values())
    return f


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        pl, clk = r.stdout.strip().split(",")[:2]
        out.update(power_limit_w=float(pl), max_sm_clock_mhz=float(clk))
    except Exception as e:                                       # noqa: BLE001
        out["power_limit_w"] = f"unavailable ({e!r})"
    return out


def bench_step(args) -> dict:
    from deeprec_b200.data.synthetic import criteo_batch
    from deeprec_b200.models.dlrm_engine import CRITEO_TB_CARDINALITIES, MLPERF_DCNV2, DLRMConfig, DLRMEngine
    # tables start at 2M rows and grow at a step boundary: pre-sized to the 16M-row default, dim-128 rows with Adagrad slots would not fit in 80 GB
    cfg = DLRMConfig(batch_size=args.batch, cardinalities=list(CRITEO_TB_CARDINALITIES), optimizer="adagrad", max_rows_per_table=1 << 21, **MLPERF_DCNV2)
    eng = DLRMEngine(cfg)
    n = args.prefill + args.warmup + args.steps
    batches = [criteo_batch(cfg.batch_size, cfg.num_dense, cfg.cardinalities, seed=7 + i) for i in range(n)]
    dev_b = [[t.pin_memory().cuda(non_blocking=True) for t in b] for b in batches]
    torch.cuda.synchronize()
    eng.load_batch(*dev_b[0]); eng.capture()
    for b in dev_b[1:args.prefill + args.warmup]:
        eng.load_batch(*b); eng.train_step()
    torch.cuda.synchronize()
    keys0 = sum(t.size() for t in eng.tables.values())
    l0 = eng.launches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for b in dev_b[args.prefill + args.warmup:]:
        eng.load_batch(*b); eng.train_step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    keys1 = sum(t.size() for t in eng.tables.values())
    fl = gemm_flops(cfg, cfg.batch_size)
    return {"ms_per_step": ms, "samples_per_s": cfg.batch_size / (ms / 1e3), "launches_per_step": (eng.launches - l0) / args.steps,
            "new_keys_per_step": (keys1 - keys0) / args.steps, "gemm_tflop_per_step": {k: v / 1e12 for k, v in fl.items()},
            "whole_step_gemm_tflops": fl["total"] / (ms / 1e3) / 1e12, "loss": eng.loss_value(), "batch": cfg.batch_size}


def bench_layer(B: int, N: int, r: int, iters: int) -> dict:
    from deeprec_b200 import _native
    lib = _native.cuda()
    bf = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(5)
    x0 = torch.randn(B, N, device="cuda", generator=g).to(bf)
    xl = torch.randn(B, N, device="cuda", generator=g).to(bf)
    gout = (torch.randn(B, N, device="cuda", generator=g) * 1e-3).to(bf)
    V = (torch.rand(r, N, device="cuda", generator=g) * 2 - 1) * (6.0 / (N + r)) ** 0.5
    W = (torch.rand(N, r, device="cuda", generator=g) * 2 - 1) * (6.0 / (N + r)) ** 0.5
    b = torch.randn(N, device="cuda", generator=g) * 0.1
    Vb, Wb, Vt, Wt = V.to(bf), W.to(bf), V.t().contiguous().to(bf), W.t().contiguous().to(bf)
    t, u, out, du, dt, dxl = (torch.empty(B, n, device="cuda", dtype=bf) for n in (r, N, N, N, r, N))
    dx0 = torch.empty(B, N, device="cuda")
    dW, dV, db = torch.zeros(N, r, device="cuda"), torch.zeros(r, N, device="cuda"), torch.zeros(N, device="cuda")
    vp = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None   # noqa: E731

    def ours():
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        dW.zero_(); dV.zero_(); db.zero_()
        rc = [lib.dr_cuda_gemm_tn_ex(vp(xl), N, vp(Vb), N, B, r, N, None, 0, None, 0, 0, vp(t), r, None, None, None, 0, 0, s),
              lib.dr_cuda_gemm_tn_cross(vp(t), r, vp(Wb), r, B, N, r, vp(b), 1, vp(x0), N, vp(xl), N, vp(out), N, vp(u), N, 0, s),
              lib.dr_cuda_cross_bwd(vp(gout), N, vp(x0), N, vp(u), N, B, N, vp(du), N, vp(dx0), N, 1, vp(db), s),
              lib.dr_cuda_gemm_dw(vp(du), N, vp(t), r, B, N, r, vp(dW), r, 0, s),
              lib.dr_cuda_gemm_tn_ex(vp(du), N, vp(Wt), N, B, r, N, None, 0, None, 0, 0, vp(dt), r, None, None, None, 0, 0, s),
              lib.dr_cuda_gemm_dw(vp(dt), r, vp(xl), N, B, r, N, vp(dV), N, 0, s),
              lib.dr_cuda_gemm_tn_cross(vp(dt), r, vp(Vt), r, B, N, r, None, 2, None, 0, vp(gout), N, vp(dxl), N, None, 0, 0, s)]
        assert not any(rc), rc

    Vp, Wp, bp = (p.clone().requires_grad_(True) for p in (V, W, b))
    x0p, xlp = x0.clone().requires_grad_(True), xl.clone().requires_grad_(True)

    def composite():
        for p in (Vp, Wp, bp, x0p, xlp):
            p.grad = None
        with torch.autocast("cuda", dtype=bf):
            y = x0p * torch.nn.functional.linear(torch.nn.functional.linear(xlp, Vp), Wp, bp) + xlp
        y.backward(gout)
        return y

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    ms_ours, ms_torch = timed(ours), timed(composite)
    y = composite(); ours(); torch.cuda.synchronize()

    def rel(a, ref):
        a, ref = a.double(), ref.double()
        return ((a - ref).norm() / ref.norm()).item()

    # both sides against an fp64 evaluation from the same bf16 operands would need another [B, N] x [N, r] fp64 pass per tensor; the two
    # bf16 implementations are compared with each other instead, and each relative difference is of the order of bf16 rounding
    diffs = {"out": rel(out, y), "dx_l": rel(dxl, xlp.grad), "dx0(g*u)": rel(dx0, x0p.grad), "dW": rel(dW, Wp.grad), "dV": rel(dV, Vp.grad),
             "db": rel(db, bp.grad)}
    fl = 12 * B * N * r
    return {"shape": [B, N], "rank": r, "ms_ours": ms_ours, "ms_torch_autocast": ms_torch, "speedup": ms_torch / ms_ours,
            "gemm_tflops_ours": fl / (ms_ours / 1e3) / 1e12, "gemm_tflops_torch": fl / (ms_torch / 1e3) / 1e12, "rel_diff_vs_torch": diffs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prefill", type=int, default=4)
    ap.add_argument("--layer-iters", type=int, default=20)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--skip-layer", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dlrm_dcn_bench: needs a CUDA device (nothing here is measured on the CPU)")
    torch.cuda.set_device(0)
    res = {"benchmark": "dlrm_dcnv2", "card": card()}
    if not args.skip_step:
        res["step"] = bench_step(args)
        torch.cuda.empty_cache()
    if not args.skip_layer:
        res["cross_layer"] = bench_layer(args.batch, 27 * 128, 512, args.layer_iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
