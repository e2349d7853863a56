"""The argument and result contract of dr_cuda_gemm_tn_ex, pinned on the CUDA-on-CPU emulation build (csrc/cuda/emu/emu_stubs.cu).
The hardware entry (csrc/cuda/gemm_wgmma.cu) follows the same contract; tests/test_gpu_wgmma_edges.py checks the same cases on an H100:
- return codes: -2 pitch / N not a multiple of 8, -3 misaligned pointer, -5 lda < K / ldb < K / ldc < N, -4 S2 without S1 or aux_mode 2
  without an aux tile; statistics are accepted for every N and together with out_f32;
- out_f32 uses the row pitch ldc, like out;
- S1 / S2 add (+=) the fp32 epilogue values -- after bias, ReLU and mask, before the bf16 rounding of out -- and S2 multiplies by the aux
  value in aux_mode 2."""
import pytest
import torch

from deeprec_b200 import _native


def _p(t):
    return t.data_ptr() if t is not None else None


def _operands(M, N, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K + 8, generator=g).bfloat16()
    B = (torch.randn(N, K + 24, generator=g) * 0.5).bfloat16()
    bias = torch.randn(N, generator=g) * 0.3
    aux = torch.randn(M, N, generator=g).relu().bfloat16()
    return A, B, bias, aux


def _call(lib, A, lda, B, ldb, M, N, K, bias=None, relu=0, aux=None, ldm=0, aux_mode=0, out=None, ldc=None, o32=None, S1=None, S2=None):
    return lib.dr_cuda_gemm_tn_ex(_p(A), lda, _p(B), ldb, M, N, K, _p(bias), relu, _p(aux), ldm, aux_mode, _p(out), ldc, _p(o32),
                                  _p(S1), _p(S2), 0, 0, None)


def test_gemm_tn_ex_return_codes_on_the_emulation():
    M, N, K = 5, 16, 24
    A, B, _, aux = _operands(M, N, K)
    out = torch.zeros(M, N + 8, dtype=torch.bfloat16)
    S1, S2 = torch.zeros(N), torch.zeros(N)
    with _native.cuda_emulation():
        lib = _native.cuda()
        assert _call(lib, A, K + 8, B, K + 24, M, N, K, out=out, ldc=N + 8) == 0
        assert _call(lib, A, K + 4, B, K + 24, M, N, K, out=out, ldc=N + 8) == -2          # lda % 8
        assert _call(lib, A, K + 8, B, K + 24, M, 12, K, out=out, ldc=N + 8) == -2         # N % 8
        assert _call(lib, A, K + 8, B, K + 24, M, N, K, out=out, ldc=N + 4) == -2          # ldc % 8
        a_off = A.view(-1)[4:]                                                            # 8-byte aligned only
        assert _call(lib, a_off, K + 8, B, K + 24, M, N, K, out=out, ldc=N + 8) == -3
        assert _call(lib, A, 16, B, K + 24, M, N, K, out=out, ldc=N + 8) == -5             # lda < K
        assert _call(lib, A, K + 8, B, 16, M, N, K, out=out, ldc=N + 8) == -5              # ldb < K
        assert _call(lib, A, K + 8, B, K + 24, M, 32, K, out=out, ldc=N + 8) == -5         # ldc < N
        assert _call(lib, A, K + 8, B, K + 24, M, N, K, out=out, ldc=N + 8, S2=S2) == -4   # S2 without S1
        assert _call(lib, A, K + 8, B, K + 24, M, N, K, aux_mode=2, out=out, ldc=N + 8, S1=S1, S2=S2) == -4   # aux_mode 2 without aux
        # statistics at N <= 32 and together with out_f32 are part of the contract
        o32 = torch.zeros(M, N + 8)
        assert _call(lib, A, K + 8, B, K + 24, M, N, K, out=out, ldc=N + 8, o32=o32, S1=S1, S2=S2) == 0
        assert _call(lib, A, K + 8, B, K + 24, M, N, K, aux=aux, ldm=N, aux_mode=2, out=out, ldc=N + 8, S1=S1, S2=S2) == 0
        assert _call(lib, A, K + 8, B, K + 24, 0, N, K, out=out, ldc=N + 8) == 0           # empty problem: nothing to do


@pytest.mark.parametrize("aux_mode", [0, 1, 2])
def test_gemm_tn_ex_f32_pitch_and_statistics_on_the_emulation(aux_mode):
    M, N, K = 7, 24, 40
    ldc = N + 8
    A, B, bias, aux = _operands(M, N, K, seed=aux_mode + 1)
    a, b = A[:, :K].double(), B[:, :K].double()
    acc = a @ b.t()
    if aux_mode != 1:
        acc = (acc + bias.double()).relu()
    else:
        acc = acc * (aux.double() > 0)
    out = torch.full((M + 2, ldc), 7.0, dtype=torch.bfloat16)
    o32 = torch.full((M + 2, ldc), 7.0)
    S1, S2 = torch.full((N,), 0.5), torch.full((N,), -0.25)
    with _native.cuda_emulation():
        lib = _native.cuda()
        rc = _call(lib, A, K + 8, B, K + 24, M, N, K, bias=bias if aux_mode != 1 else None, relu=int(aux_mode != 1),
                   aux=aux if aux_mode else None, ldm=N, aux_mode=aux_mode, out=out, ldc=ldc, o32=o32, S1=S1, S2=None if aux_mode == 1 else S2)
    assert rc == 0
    # fp32 copy at pitch ldc; padding columns and extra rows untouched
    tol = 2 * K * 2.0 ** -24 * (a.abs() @ b.abs().t() + bias.double().abs())
    assert ((o32[:M, :N].double() - acc).abs() <= tol).all()
    assert (o32[:M, N:] == 7.0).all() and (o32[M:] == 7.0).all()
    assert torch.equal(out[:M, :N], o32[:M, :N].bfloat16())
    assert (out[:M, N:].float() == 7.0).all() and (out[M:].float() == 7.0).all()
    # statistics add the fp32 values (exactly what o32 holds), not the bf16 out
    v = o32[:M, :N].double()
    want1 = 0.5 + v.sum(0)
    assert torch.allclose(S1.double(), want1, rtol=0, atol=1e-5 * (1 + v.abs().sum(0).max().item()))
    bf_sum = 0.5 + out[:M, :N].double().sum(0)
    if (bf_sum - want1).abs().max() > 1e-3:                # the bf16-rounded sum is distinguishable here: S1 must not be it
        assert (S1.double() - bf_sum).abs().max() > (S1.double() - want1).abs().max()
    if aux_mode != 1:
        partner = aux[:M].double() if aux_mode == 2 else v
        want2 = -0.25 + (v * partner).sum(0)
        assert torch.allclose(S2.double(), want2, rtol=0, atol=1e-5 * (1 + (v * partner).abs().sum(0).max().item()))
    else:
        assert (S2 == -0.25).all()
