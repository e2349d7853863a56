"""The wgmma GEMM family (csrc/cuda/gemm_wgmma.cu) at its edges against float64 references, with per-element bounds.

Every reference is computed from the operands exactly as the kernel sees them (bf16, or e4m3 with its scales) upcast to float64, so the
only error left is the kernel's accumulation and output rounding:
- fp32 values (out_f32, dW) of a K-term dot product accumulated in fp32:  |v - ref| <= 2 K 2^-24 (|A| @ |B|^T + |bias|)
  (each of the <= K + 1 additions rounds with relative error 2^-24 of a partial sum bounded by the sum of absolute terms; factor 2 slack);
- bf16 output adds the final rounding:  |out - ref| <= 2^-8 |ref| + 2 K 2^-24 (|A| @ |B|^T + |bias|);
- column statistics add their own reduction: S = sum over rows of v, added in a 4-level shuffle tree, then 8 warps, then m_tiles tiles in
  order, then into the initial S:  |S - ref| <= sum_m tol_m + (m_tiles + 14) 2^-24 (sum_m |ref_m| + tol_m + |S_0|);
- FP8 / MXFP8: e4m3 x e4m3 products are exact in fp32, but the tensor cores' fp8 accumulation is documented publicly to keep only about
  14 significant bits.  Each wgmma of k = 32 therefore contributes at most 2^-13 (sum of absolute terms it adds) plus the fp32 accumulate:
  |acc - ref| <= (ceil(K / 32) + 1) 2^-13 (|A_q| @ |B_q|^T).  The FP8 epilogue then multiplies by a power-of-two col_scale (exact) and adds
  the bias in an fma (2^-24 |v|).  MXFP8 promotes each block's product into fp32 with one fma per block, so the same bound holds with the
  per-block scales folded into the operands.  An e4m3 output adds relative 2^-4 (3 mantissa bits) plus half the subnormal spacing 2^-10.

Writes outside the output are caught with sentinel bit patterns (a NaN payload the kernel never produces) in the padding columns of a
wider output buffer and in guard rows before and after it.  Grid size and kernel variant (streaming, B-resident, CTA pair) must not change a
single bit: each 128-row tile is accumulated in the same k order whichever CTA computes it.  Anything that could hang on a wrong mbarrier /
cluster protocol (one CTA walking every tile, the CTA-pair kernel) runs in a child process under a timeout."""
import ctypes as C
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
BF16_SENT = 0x7FA5                  # NaN payloads: bf16 / fp32 / e4m3 bit patterns no store of the kernel produces
F32_SENT = 0x7FC0DEAD
E4M3_SENT = 0x7F


def _lib():
    from deeprec_b200 import _native
    lib = _native.cuda()
    for name in ("dr_cuda_set_gemm_2cta", "dr_cuda_set_gemm_bres"):
        getattr(lib, name).argtypes, getattr(lib, name).restype = [C.c_int], C.c_int
    return lib


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ---------------------------------------------------------------------------------------------------------------------------------------
# helpers

class Guarded:
    """An output [rows, cols] at row pitch ld inside a buffer with `guard` sentinel rows before and after it."""

    def __init__(self, rows, cols, ld, dtype, guard=3):
        self.rows, self.cols, self.ld, self.guard = rows, cols, ld, guard
        ity = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.uint8: torch.uint8}[dtype]
        sent = {torch.bfloat16: BF16_SENT, torch.float32: F32_SENT, torch.uint8: E4M3_SENT}[dtype]
        self.raw = torch.full(((rows + 2 * guard) * ld,), sent, dtype=ity, device="cuda")
        self.sent = sent
        self.buf = self.raw.view(dtype).view(rows + 2 * guard, ld)
        self.t = self.buf[guard: guard + rows]

    def ptr(self):
        return _p(self.t)

    def value(self):
        return self.t[:, : self.cols]

    def check_sentinels(self, what=""):
        r = self.raw.view(self.rows + 2 * self.guard, self.ld)
        g = self.guard
        assert (r[:g] == self.sent).all() and (r[g + self.rows:] == self.sent).all(), f"{what}: store outside rows [0, M)"
        assert (r[g: g + self.rows, self.cols:] == self.sent).all(), f"{what}: store into the padding columns [N, ldc)"


def _strided_bf16(rows, cols, pad, scale, gen):
    """A [rows, cols] bf16 column slice of a [rows, cols + pad] tensor (row pitch cols + pad)."""
    w = (torch.randn(rows, cols + pad, device="cuda", generator=gen) * scale).bfloat16()
    return w, w[:, :cols]


def _assert_within(got, ref, tol, what):
    err = (got.double() - ref).abs()
    bad = err > tol
    if bad.any():
        i = bad.nonzero()[0].tolist()
        pytest.fail(f"{what}: {int(bad.sum())} elements outside the bound; first at {i}: got {got[tuple(i)].item()!r} "
                    f"ref {ref[tuple(i)].item()!r} bound {tol[tuple(i)].item()!r}")


def _stat_bound(ref_terms, tol_terms, S0, M):
    m_tiles = (M + 127) // 128
    return tol_terms.sum(0) + (m_tiles + 14) * U * (ref_terms.abs().sum(0) + tol_terms.sum(0) + S0.double().abs())


def _gemm_ex(lib, A, lda, B, ldb, M, N, K, out, ldc, bias=None, relu=0, aux=None, ldm=0, aux_mode=0, o32=None, S1=None, S2=None, max_ctas=0):
    return lib.dr_cuda_gemm_tn_ex(_p(A), lda, _p(B), ldb, M, N, K, _p(bias), relu, _p(aux), ldm, aux_mode, out, ldc, o32,
                                  _p(S1), _p(S2), max_ctas, 0, _s())


# ---------------------------------------------------------------------------------------------------------------------------------------
# dr_cuda_gemm_tn_ex: shapes (a pairwise cover of M x N x K), strided operands, guarded outputs, bias + ReLU + out_f32 + S1 / S2

M_SET = (1, 127, 129, 777, 4096)
N_SET = (8, 16, 24, 40, 64, 72, 136, 200, 512)
K_SET = (8, 24, 64, 72, 200, 512, 520, 1032)
SHAPES = [(1, 8, 8), (127, 16, 24), (129, 24, 64), (777, 40, 72), (4096, 64, 200), (1, 72, 512), (127, 136, 520), (129, 200, 1032),
          (777, 512, 8), (4096, 8, 24), (1, 16, 1032), (127, 40, 64), (4096, 512, 520), (129, 136, 200), (777, 72, 24), (4096, 24, 72),
          (1, 200, 64), (127, 64, 8), (129, 512, 512), (777, 8, 1032), (4096, 16, 512), (1, 40, 200), (129, 64, 72), (777, 200, 520)]
assert {s[0] for s in SHAPES} == set(M_SET) and {s[1] for s in SHAPES} == set(N_SET) and {s[2] for s in SHAPES} == set(K_SET)


def _problem(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Aw, A = _strided_bf16(M, K, 8, 1.0, g)                 # lda = K + 8
    Bw, B = _strided_bf16(N, K, 24, 0.5, g)                # ldb = K + 24
    bias = torch.randn(N, device="cuda", generator=g) * 0.3
    aux = torch.randn(M, N, device="cuda", generator=g).relu().bfloat16()
    a, b = A.double(), B.double()
    return Aw, Bw, bias, aux, a @ b.t(), a.abs() @ b.abs().t()


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_tn_ex_shapes_bias_relu_f32_stats(M, N, K):
    lib = _lib()
    Aw, Bw, bias, _, acc, absacc = _problem(M, N, K, seed=M * 7 + N * 3 + K)
    ldc = N + 8
    out = Guarded(M, N, ldc, torch.bfloat16)
    o32 = Guarded(M, N, ldc, torch.float32)
    S1 = torch.linspace(-1, 1, N, device="cuda"); S2 = torch.linspace(2, 3, N, device="cuda")
    S10, S20 = S1.clone(), S2.clone()
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, out.ptr(), ldc, bias=bias, relu=1, o32=o32.ptr(), S1=S1, S2=S2) == 0
    torch.cuda.synchronize()
    ref = (acc + bias.double()).relu()
    e32 = 2 * K * U * (absacc + bias.double().abs())
    _assert_within(o32.value(), ref, e32, "out_f32")
    _assert_within(out.value(), ref, 2.0 ** -8 * ref.abs() + e32, "out")
    assert torch.equal(out.value(), o32.value().bfloat16()), "out must be the bf16 rounding of out_f32"
    out.check_sentinels("out"); o32.check_sentinels("out_f32")
    _assert_within(S1, S10.double() + ref.sum(0), _stat_bound(ref, e32, S10, M), "S1")
    e2 = e32 * (2 * ref.abs() + e32) + U * ref * ref
    _assert_within(S2, S20.double() + (ref * ref).sum(0), _stat_bound(ref * ref, e2, S20, M), "S2")


# ---------------------------------------------------------------------------------------------------------------------------------------
# epilogue modes

@pytest.mark.parametrize("M,N,K", [(777, 24, 72), (129, 136, 520), (1, 16, 8), (4096, 40, 200)])
def test_gemm_tn_ex_aux_modes_and_statistics(M, N, K):
    """aux mode 1 (ReLU-backward mask) with S1; aux mode 2 (S2 = sum out * aux) with S1 and out_f32; N <= 32 carries statistics too."""
    lib = _lib()
    Aw, Bw, _, aux, acc, absacc = _problem(M, N, K, seed=11 + M + N + K)
    ldc = N + 8
    e32 = 2 * K * U * absacc
    # aux mode 1: out = acc * (aux > 0); S1 = column sums of that
    out = Guarded(M, N, ldc, torch.bfloat16)
    S1 = torch.zeros(N, device="cuda")
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, out.ptr(), ldc, aux=aux, ldm=N, aux_mode=1, S1=S1) == 0
    torch.cuda.synchronize()
    keep = (aux.double() > 0).double()
    ref = acc * keep
    _assert_within(out.value(), ref, 2.0 ** -8 * ref.abs() + e32, "out (mask)")
    out.check_sentinels("out (mask)")
    _assert_within(S1, ref.sum(0), _stat_bound(ref, e32 * keep, S1.new_zeros(N), M), "S1 (mask)")
    # aux mode 2: out = acc, S1 = sum out, S2 = sum out * aux; fp32 copy at pitch ldc
    out = Guarded(M, N, ldc, torch.bfloat16)
    o32 = Guarded(M, N, ldc, torch.float32)
    S1 = torch.zeros(N, device="cuda"); S2 = torch.zeros(N, device="cuda")
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, out.ptr(), ldc, aux=aux, ldm=N, aux_mode=2, o32=o32.ptr(), S1=S1, S2=S2) == 0
    torch.cuda.synchronize()
    _assert_within(o32.value(), acc, e32, "out_f32 (aux 2)")
    _assert_within(out.value(), acc, 2.0 ** -8 * acc.abs() + e32, "out (aux 2)")
    out.check_sentinels("out (aux 2)"); o32.check_sentinels("out_f32 (aux 2)")
    _assert_within(S1, acc.sum(0), _stat_bound(acc, e32, S1.new_zeros(N), M), "S1 (aux 2)")
    w = aux.double()
    _assert_within(S2, (acc * w).sum(0), _stat_bound(acc * w, e32 * w + U * (acc * w).abs(), S2.new_zeros(N), M), "S2 (aux 2)")


@pytest.mark.parametrize("M,N,K", [(777, 24, 72), (129, 200, 64), (1, 8, 24)])
def test_gemm_tn_ex_stats_exclude_rows_past_m(M, N, K):
    """ReLU with a positive bias: the zero-filled rows of the last tile (past M) evaluate to relu(bias) > 0 and must not reach S1 / S2;
    the statistics sum the fp32 values, not the bf16 output."""
    lib = _lib()
    Aw, Bw, _, _, acc, absacc = _problem(M, N, K, seed=21 + M + N)
    bias = torch.rand(N, device="cuda") + 1.0
    ldc = N + 8
    out = Guarded(M, N, ldc, torch.bfloat16)
    o32 = Guarded(M, N, ldc, torch.float32)
    S1 = torch.zeros(N, device="cuda"); S2 = torch.zeros(N, device="cuda")
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, out.ptr(), ldc, bias=bias, relu=1, o32=o32.ptr(), S1=S1, S2=S2) == 0
    torch.cuda.synchronize()
    ref = (acc + bias.double()).relu()
    e32 = 2 * K * U * (absacc + bias.double().abs())
    _assert_within(S1, ref.sum(0), _stat_bound(ref, e32, S1.new_zeros(N), M), "S1")
    _assert_within(S2, (ref * ref).sum(0), _stat_bound(ref * ref, e32 * (2 * ref.abs() + e32) + U * ref * ref, S2.new_zeros(N), M), "S2")
    v = o32.value().double()
    assert ((S1.double() - v.sum(0)).abs() <= (M // 128 + 15) * U * v.abs().sum(0)).all(), "S1 must sum the fp32 epilogue values"


def test_gemm_tn_ex_return_codes():
    """The argument contract shared with the emulation build (tests/test_cuda_emu_gemm_contract.py)."""
    lib = _lib()
    M, N, K = 5, 16, 24
    Aw, Bw, _, aux, _, _ = _problem(M, N, K, seed=3)
    out = torch.zeros(M, N + 8, dtype=torch.bfloat16, device="cuda")
    o = _p(out)
    S1, S2 = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, o, N + 8) == 0
    assert _gemm_ex(lib, Aw, K + 4, Bw, K + 24, M, N, K, o, N + 8) == -2
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, 12, K, o, N + 8) == -2
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, o, N + 4) == -2
    assert _gemm_ex(lib, Aw.view(-1)[4:], K + 8, Bw, K + 24, M, N, K, o, N + 8) == -3
    assert _gemm_ex(lib, Aw, 16, Bw, K + 24, M, N, K, o, N + 8) == -5
    assert _gemm_ex(lib, Aw, K + 8, Bw, 16, M, N, K, o, N + 8) == -5
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, 32, K, o, N + 8) == -5
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, o, N + 8, S2=S2) == -4
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, o, N + 8, aux_mode=2, S1=S1, S2=S2) == -4
    o32 = torch.zeros(M, N + 8, device="cuda")
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, o, N + 8, o32=_p(o32), S1=S1, S2=S2) == 0
    assert _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, o, N + 8, aux=aux, ldm=N, aux_mode=2, S1=S1, S2=S2) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------------------------
# persistence and variants: bitwise identical for every max_ctas and for the streaming / B-resident / CTA-pair kernels (child process)

VARIANT_SHAPES = [(777, 200, 512), (4096, 72, 520), (129, 512, 64), (1, 16, 24), (4096, 512, 200), (300, 40, 1032)]


def _variants_main():
    lib = _lib()
    for M, N, K in VARIANT_SHAPES:
        Aw, Bw, bias, aux, acc, absacc = _problem(M, N, K, seed=M + N + K)
        ldc = N + 8

        def run(mode, max_ctas):
            out = Guarded(M, N, ldc, torch.bfloat16); o32 = Guarded(M, N, ldc, torch.float32)
            S1 = torch.zeros(N, device="cuda"); S2 = torch.zeros(N, device="cuda")
            if mode == "fwd":
                rc = _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, out.ptr(), ldc, bias=bias, relu=1, o32=o32.ptr(), S1=S1, S2=S2, max_ctas=max_ctas)
            else:
                rc = _gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, out.ptr(), ldc, aux=aux, ldm=N, aux_mode=2, o32=o32.ptr(), S1=S1, S2=S2,
                              max_ctas=max_ctas)
            assert rc == 0, rc
            torch.cuda.synchronize()
            out.check_sentinels(f"{M, N, K, mode, max_ctas} out"); o32.check_sentinels(f"{M, N, K, mode, max_ctas} out_f32")
            return out.value().clone(), o32.value().clone(), S1, S2

        for mode in ("fwd", "aux2"):
            runs = {}
            for mc in (0, 1, 2, 5):
                runs[f"max_ctas={mc}"] = run(mode, mc)
            lib.dr_cuda_set_gemm_bres(1)            # K <= 512 takes the B-resident kernel; K = 520 / 1032 must fall back to streaming
            runs["bres"] = run(mode, 0)
            runs["bres,max_ctas=5"] = run(mode, 5)
            lib.dr_cuda_set_gemm_bres(0)
            lib.dr_cuda_set_gemm_2cta(1)            # N >= 64 takes the CTA-pair kernel
            runs["2cta"] = run(mode, 0)
            runs["2cta,max_ctas=2"] = run(mode, 2)
            lib.dr_cuda_set_gemm_2cta(0)
            base = runs["max_ctas=0"]
            ref = (acc + bias.double()).relu() if mode == "fwd" else acc
            _assert_within(base[1], ref, 2 * K * U * (absacc + bias.double().abs()), f"{M, N, K, mode} out_f32")
            for name, r in runs.items():
                for i, what in enumerate(("out", "out_f32", "S1", "S2")):
                    assert torch.equal(r[i], base[i]), (M, N, K, mode, name, what, (r[i].float() - base[i].float()).abs().max().item())
        print("ok", M, N, K, flush=True)
    print("ALL_OK")


def _mxfp8_one_cta_main():
    _mxfp8_cases(max_ctas_set=(1, 0))
    print("ALL_OK")


def _run_child(fn_name, timeout=300):
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    code = f"import sys; sys.path.insert(0, {here!r}); import test_gpu_wgmma_edges as T; T.{fn_name}()"
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    try:
        r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired as e:
        pytest.fail(f"{fn_name} timed out (kernel hang?): " + str(e.stdout)[-2000:])
    assert r.returncode == 0 and "ALL_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


def test_gemm_tn_ex_bitwise_across_grid_sizes_and_variants():
    _run_child("_variants_main")


# ---------------------------------------------------------------------------------------------------------------------------------------
# dr_cuda_gemm_dw: split-K weight gradient, accumulated into a strided, non-zero, guarded dW

DW_SHAPES = [(1, 8, 8), (63, 200, 72), (64, 512, 368), (65, 8, 368), (4097, 200, 8), (4097, 512, 72), (65, 512, 8), (1, 200, 368),
             (63, 8, 72), (64, 200, 8)]


@pytest.mark.parametrize("batch,N_out,K_in", DW_SHAPES)
def test_gemm_dw_edges(batch, N_out, K_in):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(batch + N_out + K_in)
    dYw, dY = _strided_bf16(batch, N_out, 8, 0.5, g)
    Xw, X = _strided_bf16(batch, K_in, 16, 1.0, g)
    y, x = dY.double(), X.double()
    ref_g, abs_g = y.t() @ x, y.abs().t() @ x.abs()
    W0 = torch.randn(N_out, K_in, device="cuda", generator=g)
    ldw = K_in + 8
    results = {}
    for splits in (1, 2, 7, 0):
        for rep in range(2):
            dW = Guarded(N_out, K_in, ldw, torch.float32)
            dW.value().copy_(W0)
            assert lib.dr_cuda_gemm_dw(_p(dYw), N_out + 8, _p(Xw), K_in + 16, batch, N_out, K_in, dW.ptr(), ldw, splits, _s()) == 0
            torch.cuda.synchronize()
            dW.check_sentinels(f"dW splits={splits}")
            got = dW.value().clone()
            if rep == 0:
                tol = (2 * batch + 10) * U * abs_g + (splits if splits > 0 else 132) * U * abs_g + U * (W0.double() + ref_g).abs()
                _assert_within(got, W0.double() + ref_g, tol, f"dW splits={splits}")
                results[splits] = got
            else:
                assert torch.equal(got, results[splits]), f"dW splits={splits}: two calls differ"


# ---------------------------------------------------------------------------------------------------------------------------------------
# dr_cuda_gemm_fp8_tn: K not a multiple of 128, M = 1, N = 16, guarded outputs, per-column power-of-two scales, saturation

def _e4m3(rows, cols, pad, gen, scale):
    w = torch.zeros(rows, cols + pad, device="cuda")
    w[:, :cols] = torch.randn(rows, cols, device="cuda", generator=gen) * scale
    q = w.clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    return q, q[:, :cols].view(torch.float8_e4m3fn).double()


def _fp8_acc_bound(K, absacc):
    return (math.ceil(K / 32) + 1) * 2.0 ** -13 * absacc


@pytest.mark.parametrize("M,N,K", [(1, 16, 144), (129, 16, 272), (777, 48, 144), (300, 128, 272), (4096, 64, 272)])
@pytest.mark.parametrize("out_fp8", [0, 1])
def test_gemm_fp8_tn_edges(M, N, K, out_fp8):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(M + N + K + out_fp8)
    Aq, a = _e4m3(M, K, 16, g, 2.0)             # lda = K + 16 bytes
    Bq, b = _e4m3(N, K, 32, g, 2.0)             # ldb = K + 32 bytes
    col_scale = 2.0 ** ((torch.arange(N, device="cuda") % 11) - 5).float()      # distinct neighbours: swapped columns are caught
    bias = torch.randn(N, device="cuda", generator=g)
    acc, absacc = a @ b.t(), a.abs() @ b.abs().t()
    cs = col_scale.double()
    ref = (acc * cs + bias.double()).relu()
    eacc = _fp8_acc_bound(K, absacc) * cs + U * (absacc * cs + bias.double().abs())
    if out_fp8:
        ldc = N + 16
        out = Guarded(M, N, ldc, torch.uint8)
        inv = 448.0 / (0.25 * ref.max().item() + 1e-6)       # the largest values land far beyond +448: they must saturate to 448
        assert lib.dr_cuda_gemm_fp8_tn(_p(Aq), K + 16, _p(Bq), K + 32, M, N, K, _p(col_scale), _p(bias), 1, out.ptr(), ldc, 1, inv, _s()) == 0
        torch.cuda.synchronize()
        got = out.value().view(torch.float8_e4m3fn).double()
        assert not got.isnan().any(), "e4m3 output must saturate to +-448, not become NaN"
        want = (ref * inv).clamp(max=448.0)
        assert (want >= 448).any()
        _assert_within(got, want, 2.0 ** -4 * want.abs() + 2.0 ** -10 + eacc * inv * (1 + 2.0 ** -4), "fp8 e4m3 out")
        assert (got[(ref * inv - eacc * inv) > 464] == 448).all()
    else:
        ldc = N + 8
        out = Guarded(M, N, ldc, torch.bfloat16)
        assert lib.dr_cuda_gemm_fp8_tn(_p(Aq), K + 16, _p(Bq), K + 32, M, N, K, _p(col_scale), _p(bias), 1, out.ptr(), ldc, 0, 1.0, _s()) == 0
        torch.cuda.synchronize()
        _assert_within(out.value(), ref, 2.0 ** -8 * ref.abs() + eacc, "fp8 bf16 out")
    out.check_sentinels("fp8 out")


# ---------------------------------------------------------------------------------------------------------------------------------------
# dr_cuda_gemm_mxfp8_tn: M = 1, N = 8, Kp = 128 / 1152 (more k blocks than ring stages), max_ctas = 1 (in a child process)

def _mxfp8_cases(max_ctas_set):
    from deeprec_b200.ops.mxfp8 import dequantize_mxfp8, quantize_mxfp8_reference
    lib = _lib()
    for M, N, Kc in [(1, 8, 128), (1, 8, 1152), (300, 8, 1100), (129, 24, 128), (777, 40, 1152), (4096, 64, 1152)]:
        g = torch.Generator(device="cuda").manual_seed(M + N + Kc)
        x = torch.randn(M, Kc, device="cuda", generator=g) * torch.logspace(-3, 2, Kc, device="cuda")
        w = torch.randn(max(N, 8), Kc, device="cuda", generator=g)
        aq, sfa = quantize_mxfp8_reference(x)
        bq, sfb = quantize_mxfp8_reference(w)
        Kp = aq.shape[1]
        a, b = dequantize_mxfp8(aq, sfa).double(), dequantize_mxfp8(bq, sfb)[:N].double()
        bias = torch.randn(N, device="cuda", generator=g)
        ref = (a @ b.t() + bias.double()).relu()
        absacc = a.abs() @ b.abs().t()
        tol = 2.0 ** -8 * ref.abs() + _fp8_acc_bound(Kp, absacc) + U * (Kp / 32 + 1) * (absacc + bias.double().abs())
        outs = []
        for mc in max_ctas_set:
            ldc = N + 8
            out = Guarded(M, N, ldc, torch.bfloat16)
            assert lib.dr_cuda_gemm_mxfp8_tn(_p(aq), _p(sfa), _p(bq), _p(sfb), M, N, Kp, _p(bias), 1, out.ptr(), ldc, mc, _s()) == 0
            torch.cuda.synchronize()
            out.check_sentinels(f"mxfp8 {M, N, Kp} max_ctas={mc}")
            _assert_within(out.value(), ref, tol, f"mxfp8 {M, N, Kp} max_ctas={mc}")
            outs.append(out.value().clone())
        for o in outs[1:]:
            assert torch.equal(o, outs[0]), f"mxfp8 {M, N, Kp}: result depends on max_ctas"


def test_gemm_mxfp8_edges_and_one_cta():
    _run_child("_mxfp8_one_cta_main")
