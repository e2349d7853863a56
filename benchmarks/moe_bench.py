#!/usr/bin/env python
"""MMoE / PLE on FusedRecEngine: the grouped wgmma GEMMs, the fused softmax-gate mixture and the whole training step, each against what it
replaces.

  python benchmarks/moe_bench.py [--batches 8192,65536] [--steps 20] [--warmup 3] [--rounds 3] [--op-iters 30]

Kernels, at B = 65536 and the MMoE / PLE expert layer shapes: dr_cuda_gemm_tn_grouped against G dr_cuda_gemm_tn_ex calls, and
dr_cuda_gemm_dw_grouped against G dr_cuda_gemm_dw calls (CUDA events over --op-iters calls, alternated over the rounds).  Mixture: one
fused_moe_mix forward + backward against the torch composite (Linear, softmax, stack, multiply, sum and their autograd) for the MMoE and the
PLE gates.  Steps: MMoE with 3 experts (the zoo default) and 4 (the reference's EXPERTS_COUNT) and PLE, Adagrad, one CUDA graph per step,
device-timed; the fused path is pooled_seq_engine, the module path a FusedRecEngine whose forward_fn calls tower_logits(f) without the ops.
Rounds alternate the two; medians.  Prints the card's name and power limit and one JSON line.
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
ROWS = (1_000_000, 1_000_000, 10_000)
L = 50


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                            # noqa: BLE001
        return f"unknown ({e})"


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000 / iters


# ---- kernels --------------------------------------------------------------------------------------------------------------------
GEMM_SHAPES = [("mmoe_l2", 3, 192, 256), ("mmoe_l3", 3, 128, 192), ("mmoe_l4", 3, 64, 128), ("mmoe4_l2", 4, 192, 256), ("ple_l2", 5, 128, 256),
               ("ple_l3", 5, 64, 128)]   # (name, G, N, K): every expert layer after the shared-input first one


def gemm_rounds(iters: int, rounds: int) -> dict:
    from deeprec_b200 import _native
    from deeprec_b200.nn.layers import _i64s, _ptrs
    lib, s = _native.cuda(), _native.stream_ptr()
    M = 65536
    res = {}
    for name, G, N, K in GEMM_SHAPES:
        A = torch.randn(M, G * K, device="cuda").to(torch.bfloat16)
        W = (torch.randn(G, N, K, device="cuda") / K ** 0.5).to(torch.bfloat16)
        b = torch.randn(G, N, device="cuda") * 0.1
        out = torch.empty(M, G * N, dtype=torch.bfloat16, device="cuda")
        dW = torch.zeros(G, N, K, device="cuda")
        a = lambda g: A.data_ptr() + g * K * 2
        o = lambda g: out.data_ptr() + g * N * 2

        def tn_grouped():
            assert lib.dr_cuda_gemm_tn_grouped(G, _ptrs([a(g) for g in range(G)]), _i64s([G * K] * G), _ptrs([W[g].data_ptr() for g in range(G)]),
                                               _i64s([K] * G), M, N, K, _ptrs([b[g].data_ptr() for g in range(G)]), 1, None, None,
                                               _ptrs([o(g) for g in range(G)]), _i64s([G * N] * G), None, 0, s) == 0

        def tn_separate():
            for g in range(G):
                assert lib.dr_cuda_gemm_tn_ex(C.c_void_p(a(g)), G * K, C.c_void_p(W[g].data_ptr()), K, M, N, K, C.c_void_p(b[g].data_ptr()), 1, None, 0,
                                              0, C.c_void_p(o(g)), G * N, None, None, None, 0, 0, s) == 0

        def dw_grouped():
            assert lib.dr_cuda_gemm_dw_grouped(G, _ptrs([o(g) for g in range(G)]), _i64s([G * N] * G), _ptrs([a(g) for g in range(G)]),
                                               _i64s([G * K] * G), M, N, K, _ptrs([dW[g].data_ptr() for g in range(G)]), _i64s([K] * G), 0, s) == 0

        def dw_separate():
            for g in range(G):
                assert lib.dr_cuda_gemm_dw(C.c_void_p(o(g)), G * N, C.c_void_p(a(g)), G * K, M, N, K, C.c_void_p(dW[g].data_ptr()), K, 0, s) == 0

        t = {k: [] for k in ("tn_grouped", "tn_separate", "dw_grouped", "dw_separate")}
        for _ in range(rounds):
            for k, fn in (("tn_grouped", tn_grouped), ("tn_separate", tn_separate), ("dw_grouped", dw_grouped), ("dw_separate", dw_separate)):
                t[k].append(_time(fn, iters))
        res[f"{name}_G{G}_N{N}_K{K}"] = {k + "_us": round(statistics.median(v), 1) for k, v in t.items()}
    return res


def mix_rounds(iters: int, rounds: int) -> dict:
    from deeprec_b200.nn import fused_moe_mix
    M, H, K = 65536, 64, 80
    res = {}
    for name, select in (("mmoe", ([0, 1, 2], [0, 1, 2])), ("ple", ([0, 1, 4], [2, 3, 4], [0, 1, 2, 3, 4]))):
        E = 1 + max(max(s) for s in select)
        X = torch.randn(M, E, H, device="cuda").to(torch.bfloat16).requires_grad_(True)
        xs = [torch.randn(M, K, device="cuda").to(torch.bfloat16).requires_grad_(True) for _ in select]
        gates = [torch.nn.Linear(K, len(s), device="cuda") for s in select]
        dm = [torch.randn(M, H, device="cuda").to(torch.bfloat16) for _ in select]

        def fused():
            torch.autograd.backward(fused_moe_mix(xs, gates, X, select), dm)

        def composite():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                outs = [(torch.softmax(g(x), -1).unsqueeze(-1) * torch.stack([X[:, i] for i in s], 1)).sum(1) for x, g, s in zip(xs, gates, select)]
            torch.autograd.backward(outs, dm)

        t = {"fused": [], "torch": []}
        for _ in range(rounds):
            t["fused"].append(_time(fused, iters))
            t["torch"].append(_time(composite, iters))
        res[name] = {k + "_fwd_bwd_us": round(statistics.median(v), 1) for k, v in t.items()}
    return res


# ---- training steps ---------------------------------------------------------------------------------------------------------------
def _model(name: str, experts: int, dev):
    import deeprec_b200 as dr
    from deeprec_b200.models.zoo import MMoE, build_model
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    return MMoE(num_experts=experts, emb_dim=16, device=dev) if name == "mmoe" else build_model(name, device=dev)


def _module_path_engine(model, B: int, dev):
    """pooled_seq_engine's engine with tower_logits(f) on the plain modules"""
    from deeprec_b200.models.rec_engine import FusedRecEngine, _StripTables
    net = _StripTables(model)

    def fwd(net, dense, emb, ids):
        with torch.autocast(emb.device.type, dtype=torch.bfloat16):
            return net.inner.tower_logits(torch.cat([emb[:, 0], emb[:, 1], emb[:, 2], emb[:, 3], emb[:, 4]], -1))
    bags = [(1, "sum")] * 3 + [(L, "sum")] * 2
    return FusedRecEngine(net, fwd, [0, 1, 2] + [1] * L + [2] * L, list(ROWS), B, embedding_dim=model.emb_dim, bags=bags, label_dim=2,
                          loss_fn=lambda out, y: net.inner.multitask_loss({k: v.float() for k, v in out.items()}, y[:, 0], y[:, 1]), device=dev,
                          learning_rate=0.05)


def step_ms(name: str, experts: int, fused: bool, B: int, steps: int, warmup: int) -> float:
    from deeprec_b200.models.rec_engine import pooled_seq_engine
    dev = torch.device("cuda", 0)
    model = _model(name, experts, dev)
    eng = pooled_seq_engine(model, B, L, table_rows=ROWS, device=dev, learning_rate=0.05) if fused else _module_path_engine(model, B, dev)
    g = torch.Generator().manual_seed(1)
    batches = []
    for _ in range(4):
        ids = torch.cat([torch.randint(0, r, (1, B), generator=g) for r in ROWS] + [torch.randint(0, ROWS[1], (L, B), generator=g),
                                                                                   torch.randint(0, ROWS[2], (L, B), generator=g)], 0)
        y = (torch.rand(B, 2, generator=g) < 0.3).float()
        batches.append((ids.to(dev), y.to(dev)))
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8192,65536")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--op-iters", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_bench: needs a GPU")
    res = {"card": card(), "steps": a.steps, "rounds": a.rounds}
    print("card:", res["card"], flush=True)
    res["gemm"] = gemm_rounds(a.op_iters, a.rounds)
    res["mix"] = mix_rounds(a.op_iters, a.rounds)
    for B in (int(b) for b in a.batches.split(",")):
        for name, experts in (("mmoe", 3), ("mmoe", 4), ("ple", 0)):
            times = {True: [], False: []}
            for _ in range(a.rounds):
                for fused in (True, False):
                    times[fused].append(step_ms(name, experts, fused, B, a.steps, a.warmup))
            key = f"{name}{experts if name == 'mmoe' else ''}_B{B}"
            res[key] = {"fused_ms": round(statistics.median(times[True]), 3), "module_ms": round(statistics.median(times[False]), 3),
                        "fused_all": [round(t, 3) for t in times[True]], "module_all": [round(t, 3) for t in times[False]]}
            print(key, res[key], flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
