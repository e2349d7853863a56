"""Native Processor (C ABI) end to end: export -> initialize -> process / batch_process -> full + delta hot swap."""
import os
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _engine(batch=512):
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    cards = [50, 1000, 7, 300] + [97] * 22
    return DLRMEngine(DLRMConfig(batch_size=batch, cardinalities=cards, learning_rate=0.05)), cards


def _train(eng, cards, steps, seed):
    from deeprec_b200.data import criteo_batch
    for s in range(steps):
        d, ids, y = criteo_batch(eng.B, 13, cards, seed=seed + s)
        eng.load_batch(d.cuda(), ids.cuda(), y.cuda()); eng.train_step()
    return d, ids


def test_processor_matches_engine_and_hot_swaps(tmp_path):
    from deeprec_b200.serving import Processor, decode_response, encode_request, export_delta, export_saved_model
    eng, cards = _engine()
    d, ids = _train(eng, cards, 6, 0)
    root = str(tmp_path)
    export_saved_model(eng, os.path.join(root, "v1"), version=6, root=root)
    proc = Processor(os.path.join(root, "v1"), {"session_num": 3, "select_session_policy": "RR", "max_batch": 256, "checkpoint_dir": root,
                                                "model_update_interval_ms": 100, "timeline_interval_step": 1, "timeline_start_step": 0,
                                                "timeline_trace_count": 4, "timeline_path": os.path.join(root, "trace.jsonl")})
    eng.load_batch(d.cuda(), ids.cuda(), torch.zeros(eng.B, device="cuda"))
    ref = eng.predict().cpu().numpy().copy()
    got = proc.predict(d.numpy(), ids.numpy())                  # batch 512 > max_batch 256 -> chunked inside the session
    assert got.shape == ref.shape and np.abs(got - ref).max() < 2e-2, np.abs(got - ref).max()
    rc, outs = proc.batch_process([encode_request(d.numpy()[:64], ids.numpy()[:, :64]) for _ in range(4)])
    assert rc == 200 and all(np.abs(decode_response(o)[0] - ref[:64]).max() < 2e-2 for o in outs)
    assert proc.process(b"garbage")[0] == 500
    info = proc.model_info()
    assert info["model_version"] == 6 and info["sessions"] == 3 and info["requests"] >= 5
    # ---- delta update: train more, export only dirty rows, the live model picks it up without a swap
    _train(eng, cards, 3, 100)
    export_delta(eng, root, base_version=6, version=9)
    eng.load_batch(d.cuda(), ids.cuda(), torch.zeros(eng.B, device="cuda"))
    ref2 = eng.predict().cpu().numpy().copy()
    for _ in range(100):
        time.sleep(0.1)
        if proc.model_info()["delta_updates"] >= 1:
            break
    got2 = proc.predict(d.numpy(), ids.numpy())
    assert proc.model_info()["delta_version"] == 9 and np.abs(got2 - ref2).max() < 2e-2, np.abs(got2 - ref2).max()
    assert np.abs(ref2 - ref).max() > 1e-4
    # ---- full update: new version directory, swapped after warm-up
    _train(eng, cards, 2, 200)
    export_saved_model(eng, os.path.join(root, "v2"), version=11, root=root)
    for _ in range(100):
        time.sleep(0.1)
        if proc.model_info()["model_version"] == 11:
            break
    eng.load_batch(d.cuda(), ids.cuda(), torch.zeros(eng.B, device="cuda"))
    ref3 = eng.predict().cpu().numpy().copy()
    got3 = proc.predict(d.numpy(), ids.numpy())
    assert proc.model_info()["full_updates"] == 1 and np.abs(got3 - ref3).max() < 2e-2
    assert os.path.exists(os.path.join(root, "trace.jsonl"))
    proc.close()


def test_python_session_group_round_robin():
    from deeprec_b200.serving import SessionGroup
    m = torch.nn.Linear(8, 1).cuda()
    sg = SessionGroup(m, session_num=3, select_session_policy="MOD", device="cuda")
    x = torch.randn(16, 8, device="cuda")
    outs = [sg.run(x, session_id=i) for i in range(6)]
    assert all(torch.allclose(o, outs[0]) for o in outs)
    m2 = torch.nn.Linear(8, 1).cuda()
    sg.swap_model(m2, warmup_inputs=(x,))
    assert torch.allclose(sg.run(x), m2(x))


def test_processor_fp8_mlp_close_to_bf16(tmp_path):
    """mlp_dtype=fp8: E4M3 wgmma GEMMs with calibrated static activation scales; predictions stay close to the bf16 runtime,
    and a delta update re-quantises the dense block while keeping the calibration."""
    from deeprec_b200.serving import Processor, export_delta, export_saved_model
    eng, cards = _engine()
    d, ids = _train(eng, cards, 6, 0)
    root = str(tmp_path)
    export_saved_model(eng, os.path.join(root, "v1"), version=6, root=root)
    common = {"session_num": 2, "max_batch": 512, "checkpoint_dir": root, "model_update_interval_ms": 100}
    p16 = Processor(os.path.join(root, "v1"), dict(common, model_update_interval_ms=0))
    p8 = Processor(os.path.join(root, "v1"), dict(common, mlp_dtype="fp8"))
    assert p8.model_info()["mlp_dtype"] == "fp8" and p16.model_info()["mlp_dtype"] == "bf16"
    a, b = p16.predict(d.numpy(), ids.numpy()), p8.predict(d.numpy(), ids.numpy())
    assert np.isfinite(b).all() and np.abs(a - b).max() < 0.06 and np.abs(a - b).mean() < 0.015, (np.abs(a - b).max(), np.abs(a - b).mean())
    assert np.corrcoef(a, b)[0, 1] > 0.98
    _train(eng, cards, 3, 100)
    export_delta(eng, root, base_version=6, version=9)
    eng.load_batch(d.cuda(), ids.cuda(), torch.zeros(eng.B, device="cuda"))
    ref2 = eng.predict().cpu().numpy().copy()
    for _ in range(100):
        time.sleep(0.1)
        if p8.model_info()["delta_updates"] >= 1:
            break
    b2 = p8.predict(d.numpy(), ids.numpy())
    assert p8.model_info()["delta_version"] == 9 and np.abs(b2 - ref2).max() < 0.06
    p16.close(); p8.close()
