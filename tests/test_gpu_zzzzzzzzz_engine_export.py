"""Engine exports on the H100: engine -> export_engine_program -> the GPU Processor against the fp32 oracle of tests/engine_export_cases.py,
the cross_linear op at MLPerf widths against float64, and a delta hot-swap under load.  Emulation twin: tests/test_cuda_emu_engine_export.py."""
import os
import threading

import numpy as np
import pytest
import torch

import engine_export_cases as K
from test_cuda_emu_engine_export import _write, cross_linear_case

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]
TOL = 3e-2
B = 1024                  # 8 row tiles of the cross GEMM per chunk of 512


def _dev():
    return torch.device("cuda", 0)


def _proc(path, **kw):
    from deeprec_b200.serving import Processor
    return Processor(path, {"session_num": 2, "max_batch": 512, "model_update_interval_ms": 0, **kw}, device="cuda")


@pytest.mark.parametrize("name,comb,D", [("deepfm", "sum", 16), ("din", "sum", 16), ("bst", "sum", 16), ("dssm", "sqrtn", 16),
                                         ("dlrm_dcnv2", None, 16), ("dlrm_dcnv2", None, 128)])
def test_engine_export_on_the_gpu_processor(tmp_path, name, comb, D):
    from deeprec_b200.serving import export_engine_program
    dev = _dev()
    eng = K.dlrm_dcn_engine(dev, B, D=D) if name == "dlrm_dcnv2" else K.make_engine(name, dev, B, combiner=comb)
    dense, ids = K.train(eng, name, B, 3, 10)
    if name in K.CRITEO or name == "dlrm_dcnv2":
        ids = ids.clone(); ids[1, :8] += 10 ** 9
    ref = K.oracle(eng, name, dense, ids, comb)
    export_engine_program(eng, str(tmp_path / "v"), root=str(tmp_path))
    p = _proc(str(tmp_path / "v"))
    try:
        req = K.request(name, dense, ids)
        assert K.max_err(p.predict(*req), ref) < TOL, K.max_err(p.predict(*req), ref)
        assert K.max_err(p.predict(req[0][:1], req[1][:, :1]), ref[:1]) < TOL
    finally:
        p.close()


@pytest.mark.parametrize("rows", [1, 127, 4099])
def test_cross_linear_at_mlperf_widths(tmp_path, rows):
    p, dense, ref = cross_linear_case(3456, 512, rows)
    _write(p, str(tmp_path / "m"), 2 * 3456 + 512, 1)
    pr = _proc(str(tmp_path / "m"), max_batch=4099)
    try:
        got = pr.predict(dense, np.zeros((1, rows), np.int64)).astype(np.float64)
    finally:
        pr.close()
    assert np.isfinite(got).all() and np.abs(got - ref).max() < TOL, np.abs(got - ref).max()


def test_delta_hot_swap_with_requests_in_flight(tmp_path):
    import time
    from deeprec_b200.serving import export_engine_delta, export_engine_program
    dev = _dev()
    eng = K.dlrm_dcn_engine(dev, B)
    dense, ids = K.train(eng, "dlrm_dcnv2", B, 3, 10)
    root = str(tmp_path)
    export_engine_program(eng, os.path.join(root, "v3"), root=root)
    req = K.request("dlrm_dcnv2", dense, ids)
    p = _proc(os.path.join(root, "v3"), checkpoint_dir=root, model_update_interval_ms=50)
    stop, errors, served = threading.Event(), [], [0]

    def load():
        try:
            while not stop.is_set():
                out = p.predict(*req)
                assert np.isfinite(out).all()
                served[0] += 1
        except Exception as e:                                       # noqa: BLE001
            errors.append(e)
    th = [threading.Thread(target=load) for _ in range(2)]
    try:
        for t in th:
            t.start()
        K.train(eng, "dlrm_dcnv2", B, 2, 40)
        export_engine_delta(eng, root, base_version=3)
        t0 = time.time()
        while p.model_info()["delta_version"] != 5 and time.time() - t0 < 60:
            time.sleep(0.05)
        n0 = served[0]
        while served[0] < n0 + 4 and time.time() - t0 < 120:
            time.sleep(0.05)
    finally:
        stop.set()
        for t in th:
            t.join()
    try:
        assert not errors, errors
        assert p.model_info()["delta_version"] == 5
        assert K.max_err(p.predict(*req), K.oracle(eng, "dlrm_dcnv2", dense, ids)) < TOL
    finally:
        p.close()


@pytest.mark.parametrize("rows", [1, 127, 4099])
def test_cross_linear_gemm_call_into_nan_prefilled_output(rows):
    """The call the GPU runtime makes for cross_linear: dr_cuda_gemm_tn_cross kind 1 without u, N = 3456, rank 512, every operand at the
    pitch of its buffer.  The output starts as NaN: every row < rows must be written, finite and within the bf16 bound of float64."""
    from test_gpu_zzzzzzzz_dlrm_dcn import _cross
    N, r = 3456, 512
    g = torch.Generator(device="cuda").manual_seed(rows)
    bf = torch.bfloat16
    t = (torch.randn(rows, r, device="cuda", generator=g) / r ** 0.5).to(bf)
    W = torch.randn(N, r, device="cuda", generator=g).to(bf)
    bias = torch.randn(N, device="cuda", generator=g)
    x0 = torch.randn(rows, N, device="cuda", generator=g).to(bf)
    xl = torch.randn(rows, N, device="cuda", generator=g).to(bf)
    out = torch.full((rows, N), float("nan"), device="cuda", dtype=bf)
    assert _cross(t, W, bias, 1, x0, xl, out, None, rows, N, r) == 0
    ref = x0.double() * (t.double() @ W.double().T + bias.double()) + xl.double()
    got = out.double()
    assert torch.isfinite(got).all()
    assert ((got - ref).abs() <= ref.abs() * 2 ** -8 + 1e-3 * (1 + x0.double().abs())).all(), (got - ref).abs().max().item()
