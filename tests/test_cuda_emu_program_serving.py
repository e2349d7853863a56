"""The GPU Processor's op-program interpreter (csrc/cuda/serving_runtime.cu::Session::RunProgram), its glue kernels (program_kernels.cu), the
device-table kernels and the fused DIN attention kernel, executed on the CUDA-on-CPU emulation (``Processor(device="cuda_emu")``: one host
thread per CUDA thread; the wgmma GEMM entry point replaced by a host loop with the same argument contract).  Same assertions as
tests/test_gpu_zzz_program_serving.py at batch sizes a CPU box can afford: a GPU-less CI catches interpreter / indexing / layout bugs before
the kernels ever reach hardware."""
import os
import time

import numpy as np
import pytest
import torch

import deeprec_b200 as dr
from deeprec_b200.data import criteo_batch
from deeprec_b200.models.zoo import build_model
from deeprec_b200.serving import Processor, export_delta_program, export_saved_model_program, predict_pb

pytestmark = [pytest.mark.timeout(900)]

CARDS = [50, 1000, 7, 300] + [97] * 22
TOL = 3e-2            # bf16 activations between the layers vs the fp32 module (probabilities)


def _train(model, opt, steps, seed, B=96):
    for s in range(steps):
        d, ids, y = criteo_batch(B, 13, CARDS, seed=seed + s)
        loss = model.loss(d, ids, y); opt.zero_grad(); loss.backward(); opt.step()
    return d, ids


def _ref(model, d, ids):
    model.eval()
    with torch.no_grad():
        p = torch.sigmoid(model(d, ids)).numpy().copy()
    model.train()
    return p


def _wait(pred, timeout=60.0):
    t0 = time.time()
    while time.time() - t0 < timeout:
        if pred():
            return True
        time.sleep(0.05)
    return False


@pytest.mark.parametrize("name", ["deepfm", "wdl", "dcn", "dcnv2", "masknet"])
def test_op_program_models_on_the_emulated_gpu_processor(tmp_path, name):
    dr.embedding_variable.clear_registry()
    torch.manual_seed(4)
    model = build_model(name, device="cpu", cardinalities=CARDS)
    opt = dr.optim.AdagradOptimizer(model, lr=0.05)
    d, ids = _train(model, opt, 4, 4)
    root = str(tmp_path)
    export_saved_model_program(model, os.path.join(root, "v1"), version=4, root=root)
    cfg = {"session_num": 2, "max_batch": 40, "checkpoint_dir": root, "model_update_interval_ms": 100}
    emu = Processor(os.path.join(root, "v1"), cfg, device="cuda_emu")
    try:
        ref = _ref(model, d, ids)
        got = emu.predict(d.numpy(), ids.numpy())                          # 96 rows > max_batch: chunked
        assert got.shape == ref.shape and np.isfinite(got).all()
        assert np.abs(got - ref).max() < TOL, np.abs(got - ref).max()
        assert np.abs(emu.predict(d.numpy()[:3], ids.numpy()[:, :3]) - ref[:3]).max() < TOL
        ids2 = ids.clone(); ids2[:, :40] += 10 ** 9                         # unseen ids read the default rows
        assert np.abs(emu.predict(d.numpy()[:40], ids2.numpy()[:, :40]) - _ref(model, d, ids2)[:40]).max() < TOL
        rc, out = emu.process(predict_pb.encode_predict_request(d.numpy()[:5], ids.numpy()[:, :5], per_feature=True))
        assert rc == 200 and np.abs(predict_pb.decode_predict_response(out)[0] - ref[:5]).max() < TOL
        # delta update: touched rows (copy-on-write) + re-folded dense tensors
        _train(model, opt, 2, 50)
        export_delta_program(model, root, base_version=4, version=6)
        assert _wait(lambda: emu.model_info()["delta_version"] == 6)
        ref2 = _ref(model, d, ids)
        assert np.abs(ref2 - ref).max() > 1e-4
        assert np.abs(emu.predict(d.numpy()[:40], ids.numpy()[:, :40]) - ref2[:40]).max() < TOL
    finally:
        emu.close()


def test_din_op_program_on_the_emulated_gpu_processor(tmp_path):
    from deeprec_b200.data import taobao_batch
    from deeprec_b200.models.rec_engine import din_ids
    dr.embedding_variable.clear_registry()
    torch.manual_seed(3)
    L, B = 20, 48
    model = build_model("din", device="cpu")
    opt = dr.optim.AdagradOptimizer(model, lr=0.05)
    for sd in range(4):
        b = taobao_batch(B, L, 500, 3000, 40, seed=sd)
        loss = model.loss(b); opt.zero_grad(); loss.backward(); opt.step()
    b["hist_item"][:5] = -1; b["hist_cat"][:5] = -1                     # five samples with an empty history
    root = str(tmp_path)
    export_saved_model_program(model, os.path.join(root, "v1"), version=2, root=root, max_len=L)
    model.eval()
    with torch.no_grad():
        ref = torch.sigmoid(model(b)).numpy().copy()
    ids = din_ids(b).numpy(); dense = np.zeros((B, 1), np.float32)
    emu = Processor(os.path.join(root, "v1"), {"session_num": 1, "max_batch": 20, "model_update_interval_ms": 0}, device="cuda_emu")
    try:
        got = emu.predict(dense, ids)                                     # 48 rows > max_batch: chunked
        assert np.isfinite(got).all() and np.abs(got - ref).max() < TOL, np.abs(got - ref).max()
        assert np.abs(emu.predict(dense[:3], ids[:, :3]) - ref[:3]).max() < TOL
    finally:
        emu.close()


@pytest.mark.parametrize("name", ["esmm", "mmoe", "ple", "dssm"])
def test_multitask_and_dssm_op_programs_on_the_emulated_gpu_processor(tmp_path, name):
    from deeprec_b200.data import taobao_batch
    from deeprec_b200.models.rec_engine import din_ids
    dr.embedding_variable.clear_registry()
    torch.manual_seed(5)
    L, B = 12, 40
    model = build_model(name, device="cpu")
    opt = dr.optim.AdagradOptimizer(model, lr=0.05)
    for sd in range(3):
        b = taobao_batch(B, L, 500, 3000, 40, seed=sd)
        loss = model.loss(b); opt.zero_grad(); loss.backward(); opt.step()
    b["hist_item"][:4] = -1; b["hist_cat"][:4] = -1
    root = str(tmp_path)
    export_saved_model_program(model, os.path.join(root, "v1"), version=1, root=root, max_len=L)
    model.eval()
    with torch.no_grad():
        out = model(b)
    ref = torch.sigmoid(out).numpy() if name == "dssm" else torch.stack([torch.sigmoid(out["ctr"]), torch.sigmoid(out["cvr"])], 1).numpy()
    ids = din_ids(b).numpy(); dense = np.zeros((B, 1), np.float32)
    emu = Processor(os.path.join(root, "v1"), {"session_num": 1, "max_batch": 25, "model_update_interval_ms": 0}, device="cuda_emu")
    try:
        got = emu.predict(dense, ids)
        assert got.shape == ref.shape and np.isfinite(got).all() and np.abs(got - ref).max() < TOL, np.abs(got - ref).max()
        rc, pb = emu.process(predict_pb.encode_predict_request(dense[:5], ids[:, :5]))
        assert rc == 200 and np.abs(predict_pb.decode_predict_response(pb)[0] - ref[:5]).max() < TOL
    finally:
        emu.close()
