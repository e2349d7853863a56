"""The ping-pong bf16 GEMM (dr_cuda_gemm_tn_ex's default kernel for K < 512: each consumer warpgroup owns whole 128-row tiles, the aux
tile arrives by TMA and the output leaves by TMA store) at the eleven dense GEMM shapes of the DLRM training step and at ragged row
counts, in every epilogue mode the step uses.

For each case: out, S1 and S2 are bitwise equal to the B-resident and CTA-pair kernels (which keep the cooperative epilogue) wherever they
apply, and to the ping-pong kernel itself for max_ctas 1, 2, 3 and 0 (one CTA walking every tile, an odd number of tiles per CTA, a
warpgroup with no tile); out lies within the float64 bounds of tests/test_gpu_wgmma_edges.py; sentinel rows and padding columns around
out show no store past row M or column N.  Everything runs in a child process under a timeout, since a wrong barrier protocol hangs."""
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_wgmma_edges as E  # noqa: E402

pytestmark = pytest.mark.gpu

B = 65536
# (M, N, K, mode) -- the step's calls (models/dlrm_engine.py): fwd = bias + ReLU (+ S1 / S2 when "s"), aux1 = ReLU-backward mask + S1,
# aux2 = BatchNorm-backward partner + S1 / S2, plain = no epilogue
STEP_CASES = [(B, 512, 16, "fwd_s"), (B, 256, 512, "fwd_s"), (B, 64, 256, "fwd_s"), (B, 16, 64, "fwd"), (B, 512, 368, "fwd"),
              (B, 256, 512, "fwd"), (B, 512, 256, "aux1"), (B, 368, 512, "plain"), (B, 64, 16, "aux2"), (B, 256, 64, "aux2"),
              (B, 512, 256, "aux2")]
EDGE_CASES = [(M, N, K, mode) for M, (N, K) in zip((1, 127, 129, 65537), ((16, 64), (136, 72), (512, 256), (64, 16)))
              for mode in ("fwd_s", "aux1", "aux2", "plain")]


def _run(lib, M, N, K, mode, max_ctas, data):
    Aw, Bw, bias, aux = data
    ldc = N + 8                                           # ldc > N: the padding columns hold sentinels
    out = E.Guarded(M, N, ldc, torch.bfloat16)
    S1 = torch.zeros(N, device="cuda") if mode != "plain" else None
    S2 = torch.zeros(N, device="cuda") if mode in ("fwd_s", "aux2") else None
    kw = dict(max_ctas=max_ctas, S1=S1, S2=S2)
    if mode.startswith("fwd"):
        kw.update(bias=bias, relu=1)
        if mode == "fwd":
            kw.update(S1=None, S2=None)
    elif mode in ("aux1", "aux2"):
        kw.update(aux=aux, ldm=N, aux_mode=int(mode[-1]))
    rc = E._gemm_ex(lib, Aw, K + 8, Bw, K + 24, M, N, K, out.ptr(), ldc, **kw)
    assert rc == 0, (M, N, K, mode, rc)
    torch.cuda.synchronize()
    out.check_sentinels(f"{M, N, K, mode, max_ctas} out")
    return out.value().clone(), kw["S1"], kw["S2"]


def _cases_main(which):
    lib = E._lib()
    for M, N, K, mode in (STEP_CASES if which == "step" else EDGE_CASES):
        Aw, Bw, bias, aux, acc, absacc = E._problem(M, N, K, seed=M + 3 * N + 7 * K)
        data = (Aw, Bw, bias, aux)
        runs = {f"max_ctas={mc}": _run(lib, M, N, K, mode, mc, data) for mc in (0, 1, 2, 3)}
        if (K + 63) // 64 <= 8:                           # the B-resident kernel takes K <= 512
            lib.dr_cuda_set_gemm_bres(1)
            runs["bres"] = _run(lib, M, N, K, mode, 0, data)
            lib.dr_cuda_set_gemm_bres(0)
        if N > 32:                                        # the CTA-pair kernel takes the 64- and 128-column tiles
            lib.dr_cuda_set_gemm_2cta(1)
            runs["2cta"] = _run(lib, M, N, K, mode, 0, data)
            lib.dr_cuda_set_gemm_2cta(0)
        base = runs["max_ctas=0"]
        if mode.startswith("fwd"):
            ref, e32 = (acc + bias.double()).relu(), 2 * K * E.U * (absacc + bias.double().abs())
        elif mode == "aux1":
            keep = (aux.double() > 0).double()
            ref, e32 = acc * keep, 2 * K * E.U * absacc * keep
        else:
            ref, e32 = acc, 2 * K * E.U * absacc
        E._assert_within(base[0], ref, 2.0 ** -8 * ref.abs() + e32, f"{M, N, K, mode} out")
        if base[1] is not None:
            E._assert_within(base[1], ref.sum(0), E._stat_bound(ref, e32, base[1].new_zeros(N), M), f"{M, N, K, mode} S1")
        for name, r in runs.items():
            for i, what in enumerate(("out", "S1", "S2")):
                if base[i] is not None:
                    assert torch.equal(r[i], base[i]), (M, N, K, mode, name, what, (r[i].float() - base[i].float()).abs().max().item())
        print("ok", M, N, K, mode, sorted(runs), flush=True)
        del acc, absacc
    print("ALL_OK")


def _run_child(which, timeout=600):
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    code = f"import sys; sys.path.insert(0, {here!r}); import test_gpu_gemm_pingpong as T; T._cases_main({which!r})"
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    try:
        r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired as e:
        pytest.fail(f"{which} cases timed out (kernel hang?): " + str(e.stdout)[-2000:])
    assert r.returncode == 0 and "ALL_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


def test_pingpong_step_shapes_bitwise_and_bounds():
    _run_child("step")


def test_pingpong_ragged_rows_bitwise_and_bounds():
    _run_child("edge")
