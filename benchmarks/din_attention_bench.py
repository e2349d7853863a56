#!/usr/bin/env python
"""DIN attention unit: nn.fused_din_attention (csrc/cuda/din_att_kernels.cu) against ops.attention.din_attention_composite, forward and
forward + backward under bf16 autocast, at B = 8192, L = 50, D = 32, H1 / H2 = 80 / 40 with tail-padded masks, in both modes (sum: DIN,
weights: DIEN).  CUDA events after warm-up, the two implementations alternated.  FLOPs and bytes come from the shapes; each time is set
against the H100 SXM data-sheet roofline (989 TFLOP/s dense bf16, 3.35 TB/s).  Prints one JSON line per workload and the card's name and
power limit.  The whole-step effect is zoo_bench.py --engine --model din / dien.

  python benchmarks/din_attention_bench.py [--iters 50] [--B 8192]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12


def work(B, L, D, H1, H2, bwd, k_bytes=2):
    """FLOPs of the unit (first layer on [k | q*k], second layer, score; the backward: dh1, dX and the two weight-gradient products) and the
    least bytes it must move (q, k, mask, the output; the backward also reads dout and writes dq, dk)."""
    pos = B * L
    fwd = 2 * pos * (2 * D * H1 + H1 * H2 + H2)
    flops = fwd if not bwd else 2 * fwd + 2 * pos * (H2 * H1 + 2 * D * H1) + 2 * pos * (2 * D * H1 + H1 * H2)
    byts = B * D * 4 + pos * D * k_bytes + pos + B * D * 4
    if bwd:
        byts += B * D * 4 + B * D * 4 + pos * D * k_bytes
    return flops, byts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--B", type=int, default=8192)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("din_attention_bench: needs a CUDA device")
    from deeprec_b200.nn import fused_din_attention
    from deeprec_b200.ops.attention import din_attention_composite
    dev = torch.device("cuda")
    info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": info}))
    B, L, D, H1, H2 = a.B, 50, 32, 80, 40
    torch.manual_seed(0)
    att = torch.nn.Sequential(torch.nn.Linear(4 * D, H1), torch.nn.Sigmoid(), torch.nn.Linear(H1, H2), torch.nn.Sigmoid(), torch.nn.Linear(H2, 1)).to(dev)
    lens = torch.randint(1, L + 1, (B,), device=dev)
    mask = torch.arange(L, device=dev)[None] < lens[:, None]
    q = torch.randn(B, D, device=dev).to(torch.bfloat16).requires_grad_()
    k = (torch.randn(B, L, D, device=dev) * mask.unsqueeze(-1)).to(torch.bfloat16).requires_grad_()

    def composite_weights(q, k, mask, att):
        qe = q.unsqueeze(1).expand_as(k)
        s = att(torch.cat([qe, k, qe - k, qe * k], -1)).squeeze(-1).masked_fill(~mask, -2 ** 31)
        return torch.softmax(s, -1)

    impls = {
        "sum": {"fused": lambda: fused_din_attention(q, k, mask, att), "composite": lambda: din_attention_composite(q, k, mask, att)},
        "weights": {"fused": lambda: fused_din_attention(q, k, mask, att, weights=True), "composite": lambda: composite_weights(q, k, mask, att)},
    }

    def step(fn, bwd):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = fn()
        if bwd:
            out.float().sum().backward()

    for mode, fns in impls.items():
        for bwd in (False, True):
            times = {n: [] for n in fns}
            for n, fn in fns.items():
                for _ in range(5):
                    step(fn, bwd)
            torch.cuda.synchronize()
            for _ in range(3):                  # alternated rounds
                for n, fn in fns.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.iters):
                        step(fn, bwd)
                    e1.record()
                    torch.cuda.synchronize()
                    times[n].append(e0.elapsed_time(e1) / a.iters * 1e3)
            flops, byts = work(B, L, D, H1, H2, bwd)
            floor = max(flops / PEAK_FLOPS, byts / PEAK_BW) * 1e6
            bound = "compute" if flops / PEAK_FLOPS >= byts / PEAK_BW else "memory"
            med = {n: sorted(v)[len(v) // 2] for n, v in times.items()}
            print(json.dumps({"mode": mode, "pass": "fwd+bwd" if bwd else "fwd", "B": B, "L": L, "D": D, "H1": H1, "H2": H2,
                              "us_fused": round(med["fused"], 1), "us_composite": round(med["composite"], 1),
                              "speedup": round(med["composite"] / med["fused"], 2), "gflop": round(flops / 1e9, 2), "mb": round(byts / 1e6, 1),
                              "bound": bound, "fused_share_of_roofline": round(floor / med["fused"], 3),
                              "composite_share_of_roofline": round(floor / med["composite"], 3)}))


if __name__ == "__main__":
    main()
