"""The ping-pong bf16 GEMM's epilogue variants (dr_cuda_gemm_tn_ex's default kernel, at every K): the kernel picks one of twelve
epilogue bodies per tile, by aux mode (none / ReLU-backward mask / statistics partner), by whether the tile carries column statistics
and by whether it lies wholly inside M x N.  This covers each body on tiles of both kinds: M = 128 k - 1, 128 k + 1, ragged column tiles, an aux operand with a pitch
larger than N, a mask passed with aux mode 0, an fp32 output copy, and persistent grids of 1, 5, 92 and all SMs.

For each case: out, out_f32, S1 and S2 are bitwise equal to the B-resident and CTA-pair kernels (which keep the cooperative epilogue)
wherever they apply and across the grid sizes; out lies within the float64 bounds of tests/test_gpu_wgmma_edges.py; sentinel rows and
padding columns show no store past row M or column N.  Everything runs in a child process under a timeout, since a wrong barrier
protocol hangs."""
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_wgmma_edges as E  # noqa: E402

pytestmark = pytest.mark.gpu

MODES = ("fwd_s", "fwd", "aux1_s", "aux1", "aux2_s", "mask0", "plain_f32")
# (M, N, K): 128 k -/+ 1 rows; 512 / 64 / 16 columns fill their tiles, 200 leaves a ragged 128-column tile
SHAPES = [(1023, 512, 256), (1025, 200, 368), (1025, 64, 16), (1023, 16, 64), (4097, 512, 16), (1023, 368, 512)]
STEP_SHAPE = (65536, 512, 256)


def _run(lib, M, N, K, mode, max_ctas, data):
    Aw, Bw, bias, aux = data
    ldc = N + 8                                           # ldc > N: the padding columns hold sentinels
    ldm = N + 24                                          # an aux pitch larger than N
    auxw = torch.zeros(M, ldm, device="cuda", dtype=torch.bfloat16)
    auxw[:, :N] = aux
    out = E.Guarded(M, N, ldc, torch.bfloat16)
    o32 = E.Guarded(M, N, ldc, torch.float32) if mode == "plain_f32" else None
    S1 = torch.zeros(N, device="cuda") if mode.endswith("_s") else None
    S2 = torch.zeros(N, device="cuda") if mode in ("fwd_s", "aux2_s") else None
    kw = dict(max_ctas=max_ctas, S1=S1, S2=S2, o32=o32.ptr() if o32 else None)
    if mode.startswith("fwd"):
        kw.update(bias=bias, relu=1)
    elif mode.startswith("aux"):
        kw.update(aux=auxw, ldm=ldm, aux_mode=int(mode[3]))
    elif mode == "mask0":
        kw.update(aux=auxw, ldm=ldm, aux_mode=0, bias=bias)
    rc = E._gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, out.ptr(), ldc, **kw)
    assert rc == 0, (M, N, K, mode, rc)
    torch.cuda.synchronize()
    out.check_sentinels(f"{M, N, K, mode, max_ctas} out")
    if o32:
        o32.check_sentinels(f"{M, N, K, mode, max_ctas} out_f32")
    return out.value().clone(), o32.value().clone() if o32 else None, S1, S2


def _reference(mode, acc, absacc, bias, aux, K):
    if mode.startswith("fwd"):
        return (acc + bias.double()).relu(), 2 * K * E.U * (absacc + bias.double().abs())
    if mode.startswith("aux1"):
        keep = (aux.double() > 0).double()
        return acc * keep, 2 * K * E.U * absacc * keep
    if mode == "mask0":
        return acc + bias.double(), 2 * K * E.U * (absacc + bias.double().abs())
    return acc, 2 * K * E.U * absacc


def _cases_main(which):
    lib = E._lib()
    cases = [(s, m, (0, 1, 5, 92)) for s in SHAPES for m in MODES] if which == "edge" else [(STEP_SHAPE, m, (0, 92)) for m in MODES]
    for (M, N, K), mode, grids in cases:
        Aw, Bw, bias, aux, acc, absacc = E._problem(M, N, K, seed=M + 3 * N + 7 * K)
        data = (Aw, Bw, bias, aux)
        runs = {f"max_ctas={mc}": _run(lib, M, N, K, mode, mc, data) for mc in grids}
        lib.dr_cuda_set_gemm_bres(1)
        runs["bres"] = _run(lib, M, N, K, mode, 0, data)
        lib.dr_cuda_set_gemm_bres(0)
        if N > 32:
            lib.dr_cuda_set_gemm_2cta(1)
            runs["2cta"] = _run(lib, M, N, K, mode, 0, data)
            lib.dr_cuda_set_gemm_2cta(0)
        base = runs["max_ctas=0"]
        ref, e32 = _reference(mode, acc, absacc, bias, aux, K)
        E._assert_within(base[0], ref, 2.0 ** -8 * ref.abs() + e32, f"{M, N, K, mode} out")
        if base[1] is not None:
            E._assert_within(base[1], ref, e32, f"{M, N, K, mode} out_f32")
        if base[2] is not None:
            E._assert_within(base[2], ref.sum(0), E._stat_bound(ref, e32, base[2].new_zeros(N), M), f"{M, N, K, mode} S1")
        for name, r in runs.items():
            for i, what in enumerate(("out", "out_f32", "S1", "S2")):
                if base[i] is not None:
                    assert torch.equal(r[i], base[i]), (M, N, K, mode, name, what, (r[i].float() - base[i].float()).abs().max().item())
        print("ok", M, N, K, mode, sorted(runs), flush=True)
        del acc, absacc
    print("ALL_OK")


def _run_child(which, timeout=600):
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    code = f"import sys; sys.path.insert(0, {here!r}); import test_gpu_gemm_epilogue_variants as T; T._cases_main({which!r})"
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    try:
        r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired as e:
        pytest.fail(f"{which} cases timed out (kernel hang?): " + str(e.stdout)[-2000:])
    assert r.returncode == 0 and "ALL_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


def test_epilogue_variants_ragged_tiles_bitwise_and_bounds():
    _run_child("edge")


def test_epilogue_variants_step_shape_92_ctas_bitwise_and_bounds():
    _run_child("step")
