#!/usr/bin/env python
"""A/B of the dense-path GEMM kernels at the flagship MLP shapes (CUDA events, L2 flushed between iterations, median of N): the streaming
bf16 wgmma kernel vs its cluster-of-2 variant (B tile multicast, dr_cuda_set_gemm_2cta) vs its B-resident variant (dr_cuda_set_gemm_bres,
K <= 512) vs block-scaled fp8 (dr_cuda_gemm_mxfp8_tn; quantisation of the activations timed separately).  One JSON line per shape.
    python benchmarks/gemm_ab.py [--iters 30]"""
import argparse
import ctypes as C
import json

import torch

from deeprec_b200 import _native
from deeprec_b200.ops import mxfp8

SHAPES = [(65536, 512, 16), (65536, 256, 512), (65536, 64, 256), (65536, 1024, 368 + 16), (65536, 1024, 1024), (65536, 512, 1024), (65536, 256, 512),
          (8192, 1024, 1024), (2048, 1024, 512)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    lib = _native.cuda()
    lib.dr_cuda_set_gemm_2cta.argtypes, lib.dr_cuda_set_gemm_2cta.restype = [C.c_int], C.c_int
    lib.dr_cuda_set_gemm_bres.argtypes, lib.dr_cuda_set_gemm_bres.restype = [C.c_int], C.c_int
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    s = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def timed(fn):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(args.iters):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) * 1e3)
        return sorted(ts)[len(ts) // 2]

    for M, N, K in SHAPES:
        A = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
        B = (torch.randn(N, K, device="cuda") * 0.1).bfloat16()
        bias = torch.randn(N, device="cuda")
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)

        def bf16():
            assert lib.dr_cuda_gemm_tn_ex(p(A), K, p(B), K, M, N, K, p(bias), 1, None, 0, 0, p(out), N, None, None, None, 0, 0, s()) == 0

        lib.dr_cuda_set_gemm_2cta(0)
        t1 = timed(bf16)
        lib.dr_cuda_set_gemm_2cta(1)
        t2 = timed(bf16)
        lib.dr_cuda_set_gemm_2cta(0)
        tr = None
        if K <= 512:
            lib.dr_cuda_set_gemm_bres(1)
            tr = timed(bf16)
            lib.dr_cuda_set_gemm_bres(0)
        bq, sfb = mxfp8.quantize_mxfp8(B)
        aq, sfa = mxfp8.quantize_mxfp8(A)
        tq = timed(lambda: mxfp8.quantize_mxfp8(A))
        t8 = timed(lambda: mxfp8.mxfp8_gemm(aq, sfa, bq, sfb, N, bias, True))
        fl = 2.0 * M * N * K
        print(json.dumps({"M": M, "N": N, "K": K, "bf16_1cta_us": round(t1, 1), "bf16_2cta_us": round(t2, 1), "bf16_bres_us": round(tr, 1) if tr else None, "mxfp8_gemm_us": round(t8, 1),
                          "mxfp8_quantize_a_us": round(tq, 1), "bf16_1cta_tflops": round(fl / t1 * 1e-6, 1), "bf16_2cta_tflops": round(fl / t2 * 1e-6, 1),
                          "mxfp8_tflops": round(fl / t8 * 1e-6, 1)}), flush=True)


if __name__ == "__main__":
    main()
