"""GPU serving of op-program models (WDL / DeepFM / DCN / DCNv2 / MaskNet) -- csrc/cuda/serving_runtime.cu::Session::RunProgram: the LINEAR ops
on the wgmma GEMM, the glue ops on csrc/cuda/program_kernels.cu.  Oracle: the module's own fp32 predictions and the CPU Processor
(fp32 interpreter of the SAME exported program).  Written after the round's GPU budget was spent: this file sorts last on purpose.

Reference behaviour: any SavedModel graph runs per session on the session's device (serving/processor/serving/model_session.cc:377-386)."""
import os
import time

import numpy as np
import pytest
import torch

import deeprec_b200 as dr
from deeprec_b200.data import criteo_batch
from deeprec_b200.models.zoo import build_model
from deeprec_b200.serving import Processor, ProcessorGroup, export_delta_program, export_saved_model_program, predict_pb

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

CARDS = [50, 1000, 7, 300] + [97] * 22
TOL = 3e-2            # bf16 activations between the layers vs the fp32 module (probabilities)


def _train(model, opt, steps, seed):
    for s in range(steps):
        d, ids, y = criteo_batch(512, 13, CARDS, seed=seed + s)
        loss = model.loss(d, ids, y); opt.zero_grad(); loss.backward(); opt.step()
    return d, ids


def _ref(model, d, ids):
    model.eval()
    with torch.no_grad():
        p = torch.sigmoid(model(d, ids)).numpy().copy()
    model.train()
    return p


def _wait(pred, timeout=20.0):
    t0 = time.time()
    while time.time() - t0 < timeout:
        if pred():
            return True
        time.sleep(0.05)
    return False


@pytest.mark.parametrize("name", ["deepfm", "wdl", "dcn", "dcnv2", "masknet"])
def test_op_program_models_on_the_gpu_processor(tmp_path, name):
    dr.embedding_variable.clear_registry()
    torch.manual_seed(4)
    model = build_model(name, device="cpu", cardinalities=CARDS)
    opt = dr.optim.AdagradOptimizer(model, lr=0.05)
    d, ids = _train(model, opt, 4, 4)
    root = str(tmp_path)
    export_saved_model_program(model, os.path.join(root, "v1"), version=4, root=root)
    cfg = {"session_num": 2, "max_batch": 200, "checkpoint_dir": root, "model_update_interval_ms": 100}
    gpu = Processor(os.path.join(root, "v1"), cfg, device="cuda")
    cpu = Processor(os.path.join(root, "v1"), dict(cfg, model_update_interval_ms=0), device="cpu")
    try:
        ref = _ref(model, d, ids)
        got = gpu.predict(d.numpy(), ids.numpy())                          # 512 rows > max_batch: chunked
        host = cpu.predict(d.numpy(), ids.numpy())
        assert got.shape == ref.shape and np.isfinite(got).all()
        assert np.abs(host - ref).max() < 2e-5
        assert np.abs(got - ref).max() < TOL, np.abs(got - ref).max()
        assert np.abs(got - host).max() < TOL                              # and == the fp32 interpreter of the same program
        assert np.abs(gpu.predict(d.numpy()[:3], ids.numpy()[:, :3]) - ref[:3]).max() < TOL      # tiny batch: one partial GEMM tile
        ids2 = ids.clone(); ids2[:, :40] += 10 ** 9                         # unseen ids read the default rows
        assert np.abs(gpu.predict(d.numpy(), ids2.numpy()) - _ref(model, d, ids2)).max() < TOL
        rc, out = gpu.process(predict_pb.encode_predict_request(d.numpy()[:5], ids.numpy()[:, :5], per_feature=True))
        assert rc == 200 and np.abs(predict_pb.decode_predict_response(out)[0] - ref[:5]).max() < TOL
        # delta update: touched rows (copy-on-write) + re-folded dense tensors
        _train(model, opt, 2, 50)
        export_delta_program(model, root, base_version=4, version=6)
        assert _wait(lambda: gpu.model_info()["delta_version"] == 6)
        ref2 = _ref(model, d, ids)
        assert np.abs(ref2 - ref).max() > 1e-4
        assert np.abs(gpu.predict(d.numpy(), ids.numpy()) - ref2).max() < TOL
    finally:
        gpu.close(); cpu.close()


def test_op_program_processor_group_on_every_visible_gpu(tmp_path):
    """One replica per visible GPU in one process (config #5 shape) serving a DeepFM program."""
    dr.embedding_variable.clear_registry()
    torch.manual_seed(1)
    model = build_model("deepfm", device="cpu", cardinalities=CARDS)
    opt = dr.optim.AdagradOptimizer(model, lr=0.05)
    d, ids = _train(model, opt, 3, 9)
    root = str(tmp_path)
    export_saved_model_program(model, os.path.join(root, "v1"), version=1, root=root)
    n = torch.cuda.device_count()
    grp = ProcessorGroup(os.path.join(root, "v1"), {"session_num": 2, "max_batch": 256, "model_update_interval_ms": 0, "gpu_ids_list": list(range(n))})
    try:
        ref = _ref(model, d, ids)
        for _ in range(2 * n):                                             # round-robin over the replicas
            assert np.abs(grp.predict(d.numpy()[:128], ids.numpy()[:, :128]) - ref[:128]).max() < TOL
    finally:
        grp.close()


def test_din_op_program_on_the_gpu_processor(tmp_path):
    """DIN (lookup columns over shared tables, valid_mask / seq_zip / seq_mask / seq_sum / prelu glue kernels, the fused attention kernel of
    attention_kernels.cu behind fp32 staging) on the GPU Processor == the module == the CPU Processor."""
    from deeprec_b200.data import taobao_batch
    from deeprec_b200.models.rec_engine import din_ids
    dr.embedding_variable.clear_registry()
    torch.manual_seed(3)
    L = 20
    model = build_model("din", device="cpu")
    opt = dr.optim.AdagradOptimizer(model, lr=0.05)
    for sd in range(4):
        b = taobao_batch(256, L, 500, 3000, 40, seed=sd)
        loss = model.loss(b); opt.zero_grad(); loss.backward(); opt.step()
    b["hist_item"][:5] = -1; b["hist_cat"][:5] = -1                     # five samples with an empty history
    root = str(tmp_path)
    export_saved_model_program(model, os.path.join(root, "v1"), version=2, root=root, max_len=L)
    model.eval()
    with torch.no_grad():
        ref = torch.sigmoid(model(b)).numpy().copy()
    ids = din_ids(b).numpy(); dense = np.zeros((256, 1), np.float32)
    cfg = {"session_num": 2, "max_batch": 100, "model_update_interval_ms": 0}
    gpu = Processor(os.path.join(root, "v1"), cfg, device="cuda")
    cpu = Processor(os.path.join(root, "v1"), cfg, device="cpu")
    try:
        host = cpu.predict(dense, ids)
        got = gpu.predict(dense, ids)                                     # 256 rows > max_batch: chunked
        assert np.abs(host - ref).max() < 2e-5
        assert np.isfinite(got).all() and np.abs(got - ref).max() < TOL, np.abs(got - ref).max()
        assert np.abs(gpu.predict(dense[:3], ids[:, :3]) - ref[:3]).max() < TOL
    finally:
        gpu.close(); cpu.close()


@pytest.mark.parametrize("name", ["esmm", "mmoe", "ple", "dssm"])
def test_multitask_and_dssm_op_programs_on_the_gpu_processor(tmp_path, name):
    """Two probabilities per row (ctr, cvr) through softmax-gated expert mixtures; DSSM through the cosine kernel."""
    from deeprec_b200.data import taobao_batch
    from deeprec_b200.models.rec_engine import din_ids
    dr.embedding_variable.clear_registry()
    torch.manual_seed(5)
    L = 12
    model = build_model(name, device="cpu")
    opt = dr.optim.AdagradOptimizer(model, lr=0.05)
    for sd in range(3):
        b = taobao_batch(128, L, 500, 3000, 40, seed=sd)
        loss = model.loss(b); opt.zero_grad(); loss.backward(); opt.step()
    b["hist_item"][:4] = -1; b["hist_cat"][:4] = -1
    root = str(tmp_path)
    export_saved_model_program(model, os.path.join(root, "v1"), version=1, root=root, max_len=L)
    model.eval()
    with torch.no_grad():
        out = model(b)
    ref = torch.sigmoid(out).numpy() if name == "dssm" else torch.stack([torch.sigmoid(out["ctr"]), torch.sigmoid(out["cvr"])], 1).numpy()
    ids = din_ids(b).numpy(); dense = np.zeros((128, 1), np.float32)
    gpu = Processor(os.path.join(root, "v1"), {"session_num": 1, "max_batch": 50, "model_update_interval_ms": 0}, device="cuda")
    try:
        got = gpu.predict(dense, ids)
        assert got.shape == ref.shape and np.isfinite(got).all() and np.abs(got - ref).max() < TOL, np.abs(got - ref).max()
        rc, pb = gpu.process(predict_pb.encode_predict_request(dense[:5], ids[:, :5]))
        assert rc == 200 and np.abs(predict_pb.decode_predict_response(pb)[0] - ref[:5]).max() < TOL
    finally:
        gpu.close()
