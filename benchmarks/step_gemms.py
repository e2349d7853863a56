#!/usr/bin/env python
"""Replay the eleven dense GEMM calls (dr_cuda_gemm_tn_ex) of one DLRM training step at the bench.py configuration (B = 65536) and time each
one alone: CUDA events, L2 flushed before every launch, median of --iters.  The shapes, leading dimensions and epilogues are those of
models/dlrm_engine.py: bias + ReLU in the forward chains, the ReLU-backward mask (aux mode 1) and the BatchNorm-backward partner (aux mode 2)
in the dX chains, fused column statistics (S1 / S2, which includes their k_det_colsum) where the step asks for them.  Inputs come from a
seed.  Per call it prints the time, the HBM bytes the call has to move (A, B, the bf16 output and the aux tile), the achieved GB/s, the
floor at the data-sheet 3.35 TB/s of an H100 SXM and the fraction of that floor reached, plus a SHA-256 of out / S1 / S2 so two builds
can be compared bit for bit.  The last line sums the eleven calls.

    python benchmarks/step_gemms.py [--iters 30] [--seed 0] [--batch 65536]"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12

# name, N, K, lda, bias, relu, aux_mode, S1, S2   (M = batch; ldb = K, ldc = ld_mask = N)
CALLS = [
    ("bot0_fwd", 512, 16, 16, True, True, 0, True, True),
    ("bot1_fwd", 256, 512, 512, True, True, 0, True, True),
    ("bot2_fwd", 64, 256, 256, True, True, 0, True, True),
    ("bot3_fwd", 16, 64, 64, True, True, 0, False, False),
    ("top0_fwd", 512, 368, 368, True, True, 0, False, False),
    ("top1_fwd", 256, 512, 512, True, True, 0, False, False),
    ("top1_dX", 512, 256, 256, False, False, 1, True, False),
    ("top0_dX", 368, 512, 512, False, False, 0, False, False),
    ("bot3_dX", 64, 16, 16, False, False, 2, True, True),
    ("bot2_dX", 256, 64, 64, False, False, 2, True, True),
    ("bot1_dX", 512, 256, 256, False, False, 2, True, True),
]


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def digest(*ts) -> str:
    h = hashlib.sha256()
    for t in ts:
        if t is not None:
            h.update(t.contiguous().view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--batch", type=int, default=65536)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_gemms.py times kernels on a GPU; none is visible")
    from deeprec_b200 import _native
    lib = _native.cuda()
    dev = torch.device("cuda", 0)
    M = a.batch
    g = torch.Generator(device=dev).manual_seed(a.seed)
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    print(f"# {gpu_info()}  M={M}  median of {a.iters}, L2 flushed", flush=True)
    total_us = total_floor = 0.0
    for name, N, K, lda, has_bias, relu, aux, s1, s2 in CALLS:
        A = (torch.randn(M, lda, device=dev, generator=g) * 0.5).bfloat16()
        Bm = (torch.randn(N, K, device=dev, generator=g) * 0.1).bfloat16()
        bias = torch.randn(N, device=dev, generator=g) if has_bias else None
        mask = torch.randn(M, N, device=dev, generator=g).bfloat16() if aux else None
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        S1 = torch.zeros(N, device=dev) if s1 else None
        S2 = torch.zeros(N, device=dev) if s2 else None

        def call():
            rc = lib.dr_cuda_gemm_tn_ex(p(A), lda, p(Bm), K, M, N, K, p(bias), int(relu), p(mask), N, aux, p(out), N, None, p(S1), p(S2), 0, 0,
                                        _native.stream_ptr(dev))
            _native.check(rc, "dr_cuda_gemm_tn_ex")

        call()
        torch.cuda.synchronize()
        if S1 is not None:
            S1.zero_()
        if S2 is not None:
            S2.zero_()
        call()          # out / S1 / S2 of exactly one call on zeroed statistics
        torch.cuda.synchronize()
        sha = digest(out, S1, S2)
        for _ in range(3):
            call()
        ts = []
        for _ in range(a.iters):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); call(); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        ts.sort()
        us = ts[len(ts) // 2]
        nbytes = 2 * (M * K + N * K + M * N + (M * N if aux else 0))
        floor_us = nbytes / HBM_BYTES_PER_S * 1e6
        total_us += us
        total_floor += floor_us
        print(json.dumps({"call": name, "M": M, "N": N, "K": K, "us": round(us, 1), "us_min": round(ts[0], 1), "us_max": round(ts[-1], 1),
                          "MB": round(nbytes / 1e6, 1), "GBps": round(nbytes / us * 1e-3, 0), "floor_us": round(floor_us, 1),
                          "of_floor": round(floor_us / us, 3), "sha": sha}), flush=True)
    print(json.dumps({"call": "sum", "us": round(total_us, 1), "floor_us": round(total_floor, 1), "of_floor": round(total_floor / total_us, 3)}), flush=True)


if __name__ == "__main__":
    main()
