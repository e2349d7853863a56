#!/usr/bin/env python
"""nn.fused_encoder_layer (wgmma in_proj / out_proj / FFN GEMMs + the mma.sync attention kernels of csrc/cuda/mha_kernels.cu) against
nn.TransformerEncoderLayer (eager, bf16 autocast): forward + backward of one post-norm encoder layer at BST's size (E = 32, 4 heads, FFN 128),
S = 51 (the history of 50 and the target), B = 4096 and 8192, with a random key mask whose last position is valid.  Timing: CUDA events around
N iterations after a warm-up.

It also times the attention core on its own (dr_cuda_mha_fwd + dr_cuda_mha_bwd on the same qkv) and reports its bytes moved over that time
against 3.35 TB/s (H100 SXM HBM3).  The bytes are what the two kernels must read and write, from the shapes: forward qkv (6 E) + valid (1) +
o (2 E) per token; backward qkv (6 E) + valid (1) + o (2 E) + do (2 E) + dqkv (6 E) per token.  The card name, power limit and max SM clock
are read in the same run.  Prints one JSON line per case."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeprec_b200 import _native  # noqa: E402
from deeprec_b200._native import ptr, stream_ptr  # noqa: E402
from deeprec_b200.nn import fused_encoder_layer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def time_ms(fn, iters, warmup=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="4096,8192")
    ap.add_argument("--seq", type=int, default=51)
    ap.add_argument("--dim", type=int, default=32)
    ap.add_argument("--heads", type=int, default=4)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mha_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = gpu_info()
    lib = _native.cuda()
    S, E, heads = a.seq, a.dim, a.heads
    for B in (int(b) for b in a.batches.split(",")):
        torch.manual_seed(0)
        layer = torch.nn.TransformerEncoderLayer(E, heads, 4 * E, dropout=0.0, batch_first=True, device=dev)
        x = torch.randn(B, S, E, device=dev, requires_grad=True)
        valid = torch.rand(B, S, device=dev) < 0.7
        valid[:, -1] = True
        gy = torch.randn(B, S, E, device=dev)

        def fused():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = fused_encoder_layer(x, layer, valid)
            y.backward(gy)

        def module():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = layer(x, src_key_padding_mask=~valid)
            y.backward(gy.to(y.dtype))

        qkv = torch.randn(B * S, 3 * E, device=dev).to(torch.bfloat16)
        vb = valid.to(torch.uint8).contiguous()
        o = torch.empty(B * S, E, dtype=torch.bfloat16, device=dev)
        do = torch.randn(B * S, E, device=dev).to(torch.bfloat16)
        dqkv = torch.empty_like(qkv)

        def core():
            _native.check(lib.dr_cuda_mha_fwd(ptr(qkv), ptr(vb), B, S, E, heads, ptr(o), stream_ptr()), "mha_fwd")
            _native.check(lib.dr_cuda_mha_bwd(ptr(qkv), ptr(vb), ptr(o), ptr(do), B, S, E, heads, ptr(dqkv), stream_ptr()), "mha_bwd")

        tokens = B * S
        core_bytes = tokens * ((6 * E + 1 + 2 * E) + (6 * E + 1 + 2 * E + 2 * E + 6 * E))
        row = {"B": B, "S": S, "E": E, "heads": heads, "iters": a.iters, "gpu": info}
        for name, fn in (("fused", fused), ("module", module)):
            row[f"{name}_ms_fwd_bwd"] = round(time_ms(fn, a.iters), 4)
        ms = time_ms(core, a.iters)
        row.update({"core_ms_fwd_bwd": round(ms, 4), "core_bytes": core_bytes, "core_tb_s": round(core_bytes / ms / 1e9, 3),
                    "core_share_of_3.35TB_s": round(core_bytes / ms / 1e-3 / HBM_BYTES_PER_S, 4)})
        row["speedup_vs_module"] = round(row["module_ms_fwd_bwd"] / row["fused_ms_fwd_bwd"], 3)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
