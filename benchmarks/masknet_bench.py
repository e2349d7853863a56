#!/usr/bin/env python
"""MaskNet (zoo.MaskBlockNet) training step on FusedRecEngine, and the LayerNorm GEMM epilogue against GEMM + torch LayerNorm + ReLU.

  python benchmarks/masknet_bench.py [--batch 65536] [--steps 20] [--warmup 3] [--rounds 3] [--op-iters 50]

Step: masknet_parallel (5 blocks) and masknet_serial at B = --batch, Adagrad, one CUDA graph per step, device-timed.  Each round builds the
engine twice in this process, with the MaskBlocks on the fused op (DEEPREC_FUSED_NN=1) and as cuBLAS GEMMs + torch BatchNorm / LayerNorm
(DEEPREC_FUSED_NN=0), alternating; medians over the rounds.  Op: dr_cuda_gemm_tn_ln at M = 65536, K = 432, N = 64 against
dr_cuda_gemm_tn_ex + torch LayerNorm + ReLU (bf16), CUDA events over --op-iters calls.  Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CARDS = [1_000_000] * 26


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                            # noqa: BLE001
        return f"unknown ({e})"


def step_ms(name: str, fused: bool, B: int, steps: int, warmup: int) -> float:
    import deeprec_b200 as dr
    from deeprec_b200.models.rec_engine import criteo_engine
    from deeprec_b200.models.zoo import build_model
    os.environ["DEEPREC_FUSED_NN"] = "1" if fused else "0"
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    eng = criteo_engine(build_model(name, device=dev), B, table_rows=CARDS, device=dev, learning_rate=0.05)
    g = torch.Generator().manual_seed(1)
    batches = [(torch.randint(0, 1_000_000, (26, B), generator=g).to(dev), (torch.rand(B, generator=g) < 0.3).float().to(dev),
                {"dense": (torch.rand(B, 13, generator=g) * 3).to(dev)}) for _ in range(4)]
    eng.load_batch(*batches[0])
    eng.capture()
    for i in range(warmup):
        eng.load_batch(*batches[i % 4]); eng.train_step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        eng.load_batch(*batches[i % 4]); eng.train_step()
    e1.record()
    torch.cuda.synchronize()
    loss = eng.loss_value()
    assert loss == loss, "non-finite loss"
    del eng
    torch.cuda.empty_cache()
    return e0.elapsed_time(e1) / steps


def op_us(iters: int) -> dict:
    from deeprec_b200 import _native
    lib, s = _native.cuda(), _native.stream_ptr()
    M, K, N = 65536, 432, 64
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    A = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    W = (torch.randn(N, K, device="cuda") / K ** 0.5).to(torch.bfloat16)
    gamma, beta = torch.rand(N, device="cuda") + 0.5, torch.randn(N, device="cuda") * 0.1
    y, xh, rs = torch.empty(M, N, dtype=torch.bfloat16, device="cuda"), torch.empty(M, N, dtype=torch.bfloat16, device="cuda"), torch.empty(M, device="cuda")
    h = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    ln = torch.nn.LayerNorm(N, eps=1e-3, device="cuda")
    with torch.no_grad():
        ln.weight.copy_(gamma); ln.bias.copy_(beta)

    def fused():
        assert lib.dr_cuda_gemm_tn_ln(p(A), K, p(W), K, M, N, K, None, p(gamma), p(beta), 1e-3, 1, p(y), N, p(xh), N, p(rs), 0, s) == 0

    def unfused():
        assert lib.dr_cuda_gemm_tn_ex(p(A), K, p(W), K, M, N, K, None, 0, None, 0, 0, p(h), N, None, None, None, 0, 0, s) == 0
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return torch.relu(ln(h))

    out = {}
    for name, fn in (("gemm_tn_ln", fused), ("gemm_then_torch_layernorm_relu", unfused)):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            r = fn()
        e1.record()
        torch.cuda.synchronize()
        out[name + "_us"] = round(e0.elapsed_time(e1) * 1000 / iters, 2)
    ref = unfused().float()
    out["max_abs_diff"] = float((y.float() - ref).abs().max())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--op-iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("masknet_bench: needs a GPU")
    res = {"card": card(), "batch": a.batch, "steps": a.steps, "rounds": a.rounds}
    for name in ("masknet_parallel", "masknet_serial"):
        times = {True: [], False: []}
        for _ in range(a.rounds):
            for fused in (True, False):
                times[fused].append(step_ms(name, fused, a.batch, a.steps, a.warmup))
        res[name] = {"fused_ms": round(statistics.median(times[True]), 3), "torch_ms": round(statistics.median(times[False]), 3),
                     "fused_all": [round(t, 3) for t in times[True]], "torch_all": [round(t, 3) for t in times[False]]}
    os.environ.pop("DEEPREC_FUSED_NN", None)
    res["op"] = op_us(a.op_iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
