"""Block-scaled fp8 GEMM (dr_cuda_gemm_mxfp8_tn: one e4m3 wgmma per 32-element scale block, scales applied in registers) and its quantiser
(csrc/cuda/gemm_mxfp8.cu): the CUDA quantiser equals the torch model of the format bit for bit (elements and scale words), and the GEMM
equals the fp32 product of the DEQUANTISED operands (so any error left is the bf16 output rounding -- a wrong scale-word layout would be
off by powers of two), for M / N / K tails and many tiles per CTA.  Runs in a child process under a timeout (a wrong mbarrier protocol
hangs instead of failing)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

_CHILD = r'''
import sys, torch
from deeprec_b200.ops import mxfp8
torch.manual_seed(3)
# ---- quantiser == reference, bit for bit
for R, Cc, dt in [(128, 128, torch.float32), (300, 200, torch.float32), (1000, 368, torch.bfloat16), (5, 13, torch.float32)]:
    x = (torch.randn(R, Cc, device="cuda") * torch.logspace(-3, 3, R, device="cuda").unsqueeze(1)).to(dt)
    x[0] = 0
    q, sf = mxfp8.quantize_mxfp8(x)
    torch.cuda.synchronize()
    q0, sf0 = mxfp8.quantize_mxfp8_reference(x)
    assert torch.equal(sf, sf0), (R, Cc, "scale words")
    assert torch.equal(q, q0), (R, Cc, "elements", (q != q0).sum().item())
print("quantiser ok", flush=True)
# ---- GEMM == fp32 product of the dequantised operands
shapes = [(128, 128, 128), (256, 128, 512), (1000, 256, 200), (4096, 1024, 512), (777, 40, 64), (65536, 512, 368), (130, 8, 1024)]
if len(sys.argv) > 1:
    shapes = shapes[: int(sys.argv[1])]
for M, N, K in shapes:
    A = torch.randn(M, K, device="cuda") * torch.logspace(-2, 2, M, device="cuda").unsqueeze(1)      # per-row magnitudes: the scales matter
    B = torch.randn(N, K, device="cuda") * 0.1 * torch.logspace(-1, 1, N, device="cuda").unsqueeze(1)
    bias = torch.randn(N, device="cuda")
    aq, sfa = mxfp8.quantize_mxfp8(A)
    bq, sfb = mxfp8.quantize_mxfp8(B)
    ref = mxfp8.dequantize_mxfp8(aq, sfa) @ mxfp8.dequantize_mxfp8(bq, sfb).t()
    full = A @ B.t()
    for relu, mc in ((False, 0), (True, 0), (True, 5)):
        out = mxfp8.mxfp8_gemm(aq, sfa, bq, sfb, N, bias, relu, mc).float()
        torch.cuda.synchronize()
        r = ref + bias
        f = full + bias
        if relu:
            r, f = r.relu(), f.relu()
        # row-wise tolerance: rows differ by 4 orders of magnitude
        rs = r.abs().amax(1, keepdim=True) + 1e-6
        e = ((out - r).abs() / rs).max().item()
        assert e < 1e-2, (M, N, K, relu, mc, "vs dequantised operands", e)
        # vs fp32: the kernel adds no error beyond what the e4m3 format itself costs (the dequantised product's own distance to fp32)
        fs = f.abs().amax(1, keepdim=True) + 1e-6
        e2 = ((out - f).abs() / fs).max().item()
        e_fmt = ((r - f).abs() / fs).max().item()
        assert e2 < e_fmt + 1e-2, (M, N, K, relu, mc, "vs fp32", e2, e_fmt)
    print("ok", M, N, K, flush=True)
# ---- the layer
lin = torch.nn.Linear(368, 500).cuda()
x = torch.randn(3000, 368, device="cuda").bfloat16()
y = mxfp8.MXFP8Linear(lin, relu=True)(x).float()
ref = lin(x.float()).relu()
assert y.shape == ref.shape and ((y - ref).abs().max() / ref.abs().max()).item() < 5e-2
print("ALL_OK")
'''


def _run_child(code, *args, timeout=240):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    try:
        r = subprocess.run([sys.executable, "-c", code, *args], cwd=root, env=env, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired as e:
        pytest.fail("MXFP8 child timed out (kernel hang?): " + str(e.stdout)[-2000:])
    assert r.returncode == 0 and "ALL_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


def test_mxfp8_quantiser_and_block_scaled_gemm():
    _run_child(_CHILD)
