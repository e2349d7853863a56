"""B-resident (weight-stationary) variant of the wgmma GEMM (DEEPREC_GEMM_BRES / dr_cuda_set_gemm_bres): same results as the
streaming kernel and as the fp32 reference, for every epilogue mode.  Opt-in, default off."""
import os
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from deeprec_b200 import _native
    lib = _native.cuda()
    lib.dr_cuda_set_gemm_bres.argtypes, lib.dr_cuda_set_gemm_bres.restype = [C.c_int], C.c_int
    return lib


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


@pytest.fixture
def bres():
    lib = _lib()
    prev = lib.dr_cuda_set_gemm_bres(1)
    yield lib
    lib.dr_cuda_set_gemm_bres(prev)


@pytest.mark.parametrize("M,N,K", [(4096, 512, 16), (5000, 256, 512), (65536, 512, 368), (3000, 64, 256), (2048, 368, 512), (777, 128, 64), (128, 512, 512),
                                   (100000, 256, 256)])
def test_bres_matches_reference_and_streaming_kernel(bres, M, N, K):
    lib = bres
    torch.manual_seed(11)
    A = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    B = (torch.randn(N, K, device="cuda") * 0.1).bfloat16()
    bias = torch.randn(N, device="cuda") * 0.1
    act = torch.randn(M, N, device="cuda").relu().bfloat16()
    ref0 = A.float() @ B.float().t()

    def run(mode):
        out = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
        S1 = torch.zeros(N, device="cuda"); S2 = torch.zeros(N, device="cuda")
        if mode == "fwd":
            rc = lib.dr_cuda_gemm_tn_ex(_p(A), K, _p(B), K, M, N, K, _p(bias), 1, None, 0, 0, _p(out), N, None, _p(S1), _p(S2), 0, 0, _s())
        elif mode == "mask":
            rc = lib.dr_cuda_gemm_tn_ex(_p(A), K, _p(B), K, M, N, K, None, 0, _p(act), N, 1, _p(out), N, None, _p(S1), None, 0, 0, _s())
        else:
            rc = lib.dr_cuda_gemm_tn_ex(_p(A), K, _p(B), K, M, N, K, None, 0, _p(act), N, 2, _p(out), N, None, _p(S1), _p(S2), 0, 0, _s())
        assert rc == 0
        torch.cuda.synchronize()
        return out, S1, S2

    for mode, ref in (("fwd", (ref0 + bias).relu()), ("mask", ref0 * (act.float() > 0)), ("stats", ref0)):
        lib.dr_cuda_set_gemm_bres(1)
        o1, a1, b1 = run(mode)
        lib.dr_cuda_set_gemm_bres(0)
        o0, a0, b0 = run(mode)
        lib.dr_cuda_set_gemm_bres(1)
        scale = ref.abs().max().item() + 1e-6
        assert (o1.float() - ref).abs().max().item() / scale < 2e-2, mode
        assert (o1.float() - o0.float()).abs().max().item() <= 8e-3 * scale, mode      # same K order per output element: equal up to bf16 rounding
        assert (a1 - a0).abs().max().item() <= 1e-3 * (a0.abs().max().item() + 1.0), mode       # column sums: atomics order differs
        assert (b1 - b0).abs().max().item() <= 1e-3 * (b0.abs().max().item() + 1.0), mode


def test_engine_step_matches_with_bres(bres):
    """One DLRM engine trained twice from the same seed, streaming vs B-resident GEMMs: same losses to bf16 noise."""
    from deeprec_b200.data import criteo_batch
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    cards = [50, 1000, 7, 300] + [97] * 22

    def train(flag):
        bres.dr_cuda_set_gemm_bres(flag)
        torch.manual_seed(0)
        eng = DLRMEngine(DLRMConfig(batch_size=2048, cardinalities=cards, learning_rate=0.05))
        losses = []
        for s in range(6):
            d, ids, y = criteo_batch(eng.B, 13, cards, seed=s)
            eng.load_batch(d.cuda(), ids.cuda(), y.cuda()); eng.train_step()
            losses.append(eng.loss_value())
        return losses

    l0, l1 = train(0), train(1)
    assert all(abs(a - b) < 5e-3 for a, b in zip(l0, l1)), (l0, l1)
