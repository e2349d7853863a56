#!/usr/bin/env python
"""nn.fused_gru (wgmma input projection + mma.sync recurrence kernels, csrc/cuda/rnn_kernels.cu) against nn.GRU (cuDNN, eager, bf16
autocast): forward + backward of one GRU layer at DIEN's size (I = H = 32), B = 65536, L = 20 and 50, with every sample L steps long and with
uniform random lengths in 0..L (tail padding).  cuDNN runs every padded step; the fused path stops each sample at its length.  Timing: CUDA
events around N launches after a warm-up.  FLOP/s counts the work a length-aware GRU needs, computed from the shapes and sum(len): the
projection over all B L rows (forward, dx, dW_ih: 3 x 2 B L I 3H) and the recurrence over sum(len) steps (forward h W_hh^T, and in the
backward its recomputation, the carry product and dW_hh: 4 x 2 3H H).  The same count is used for both, so the rates compare directly.
Prints one JSON line per case."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeprec_b200.nn import fused_gru  # noqa: E402


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
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--hidden", type=int, default=32)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    B, I, H = a.batch, a.hidden, a.hidden
    info = gpu_info()
    for L in (20, 50):
        for kind in ("full", "random"):
            torch.manual_seed(0)
            gru = torch.nn.GRU(I, H, batch_first=True, device=dev)
            x = torch.randn(B, L, I, device=dev, requires_grad=True)
            lengths = torch.full((B,), L, device=dev) if kind == "full" else torch.randint(0, L + 1, (B,), device=dev)
            gy = torch.randn(B, L, H, device=dev)

            def fused():
                y = fused_gru(x, gru, lengths)
                y.backward(gy)

            def cudnn():
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    y, _ = gru(x)
                y.backward(gy.to(y.dtype))
            steps = int(lengths.sum())
            flop = 3 * 2 * B * L * I * 3 * H + 4 * 2 * 3 * H * H * steps
            for name, fn in (("fused", fused), ("cudnn", cudnn)):
                ms = time_ms(fn, a.iters)
                print(json.dumps({"impl": name, "B": B, "L": L, "I": I, "H": H, "lengths": kind, "sum_len": steps, "ms_fwd_bwd": round(ms, 4),
                                  "tflops": round(flop / ms / 1e9, 2), "iters": a.iters, "gpu": info}), flush=True)


if __name__ == "__main__":
    main()
