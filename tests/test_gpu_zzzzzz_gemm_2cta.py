"""CTA-pair (thread-block cluster of 2, B tile multicast to both CTAs) variant of the wgmma GEMM (DEEPREC_GEMM_2CTA /
dr_cuda_set_gemm_2cta): same results as the single-CTA kernels and as the fp32 reference for the epilogue modes (bias + ReLU,
ReLU-backward mask, fp32 copy), M / N tails, odd numbers of 128-row blocks (the second CTA of the last pair is all out of bounds).

The kernel runs in a child process under a timeout: a wrong mbarrier / cluster protocol hangs instead of failing, and the hang must
cost one test, not the session."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

_CHILD = r'''
import ctypes as C, sys, torch
from deeprec_b200 import _native
lib = _native.cuda()
lib.dr_cuda_set_gemm_2cta.argtypes, lib.dr_cuda_set_gemm_2cta.restype = [C.c_int], C.c_int
s = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
shapes = [(256, 256, 64), (512, 128, 128), (1000, 256, 512), (4096, 1024, 512), (384, 64, 96 + 32), (65536, 512, 368 + 16),
          (777, 200, 64), (128, 512, 1024), (33000, 368, 512)]
if len(sys.argv) > 1:
    shapes = shapes[: int(sys.argv[1])]
for M, N, K in shapes:
    torch.manual_seed(5)
    A = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    B = (torch.randn(N, K, device="cuda") * 0.1).bfloat16()
    bias = torch.randn(N, device="cuda") * 0.1
    act = torch.randn(M, N, device="cuda").relu().bfloat16()
    ref0 = A.float() @ B.float().t()

    def run(mode, max_ctas=0):
        out = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
        o32 = torch.full((M, N), 7.0, device="cuda") if mode == "f32" else None
        if mode == "mask":
            rc = lib.dr_cuda_gemm_tn_ex(p(A), K, p(B), K, M, N, K, None, 0, p(act), N, 1, p(out), N, None, None, None, max_ctas, 0, s())
        else:
            rc = lib.dr_cuda_gemm_tn_ex(p(A), K, p(B), K, M, N, K, p(bias), 1, None, 0, 0, p(out), N, p(o32), None, None, max_ctas, 0, s())
        assert rc == 0, rc
        torch.cuda.synchronize()
        return out, o32

    for mode, ref in (("fwd", (ref0 + bias).relu()), ("mask", ref0 * (act.float() > 0)), ("f32", (ref0 + bias).relu())):
        lib.dr_cuda_set_gemm_2cta(1)
        o1, f1 = run(mode)
        o1b, _ = run(mode, 6)          # 3 pairs: every pair walks many tiles (accumulator ping-pong, smem ring wrap-around)
        lib.dr_cuda_set_gemm_2cta(0)
        o0, f0 = run(mode)
        scale = ref.abs().max().item() + 1e-6
        e = (o1.float() - ref).abs().max().item() / scale
        assert e < 2e-2, (M, N, K, mode, e)
        assert (o1.float() - o0.float()).abs().max().item() <= 8e-3 * scale, (M, N, K, mode)
        assert torch.equal(o1, o1b), (M, N, K, mode, "grid-size dependence")
        if f1 is not None:
            assert (f1 - ref).abs().max().item() / scale < 2e-2 and (f1 - f0).abs().max().item() <= 1e-4 * scale, (M, N, K, mode)
    print("ok", M, N, K, flush=True)
print("ALL_OK")
'''

_ENGINE_CHILD = r'''
import ctypes as C, torch
from deeprec_b200 import _native
from deeprec_b200.data import criteo_batch
from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
lib = _native.cuda()
lib.dr_cuda_set_gemm_2cta.argtypes, lib.dr_cuda_set_gemm_2cta.restype = [C.c_int], C.c_int
cards = [50, 1000, 7, 300] + [97] * 22
def train(flag):
    lib.dr_cuda_set_gemm_2cta(flag)
    torch.manual_seed(0)
    eng = DLRMEngine(DLRMConfig(batch_size=2048, cardinalities=cards, learning_rate=0.05))
    losses = []
    for st in range(6):
        d, ids, y = criteo_batch(eng.B, 13, cards, seed=st)
        eng.load_batch(d.cuda(), ids.cuda(), y.cuda()); eng.train_step()
        losses.append(eng.loss_value())
    return losses
l0, l1 = train(0), train(1)
assert all(abs(a - b) < 5e-3 for a, b in zip(l0, l1)), (l0, l1)
print("ALL_OK")
'''


def _run_child(code, *args, timeout=240):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    try:
        r = subprocess.run([sys.executable, "-c", code, *args], cwd=root, env=env, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired as e:
        pytest.fail("CTA-pair GEMM child timed out (kernel hang?): " + str(e.stdout)[-2000:])
    assert r.returncode == 0 and "ALL_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


def test_gemm_2cta_smallest_shape():
    """One 256 x 256 x 64 tile: one pair, one k block -- separates 'the protocol hangs' from 'a tail case is wrong'."""
    _run_child(_CHILD, "1", timeout=180)


def test_gemm_2cta_matches_reference_and_single_cta_kernels():
    _run_child(_CHILD)


def test_dlrm_engine_step_matches_with_2cta_gemms():
    """The flagship engine trained twice from the same seed, single-CTA vs CTA-pair GEMMs (the graph captures whichever is selected)."""
    _run_child(_ENGINE_CHILD)
