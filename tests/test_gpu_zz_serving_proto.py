"""Native Processor: protobuf PredictRequest (reference predict.proto wire format) through ``process()`` gives the same
probabilities as the compact wire format."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_processor_accepts_protobuf_requests(tmp_path):
    from deeprec_b200.data import criteo_batch
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    from deeprec_b200.serving import Processor, export_saved_model, predict_pb
    cards = [50, 1000, 7, 300] + [97] * 22
    eng = DLRMEngine(DLRMConfig(batch_size=256, cardinalities=cards, learning_rate=0.05))
    for s in range(4):
        d, ids, y = criteo_batch(eng.B, 13, cards, seed=s)
        eng.load_batch(d.cuda(), ids.cuda(), y.cuda()); eng.train_step()
    root = str(tmp_path)
    export_saved_model(eng, os.path.join(root, "v1"), version=4, root=root)
    proc = Processor(os.path.join(root, "v1"), {"session_num": 2, "max_batch": 256, "model_update_interval_ms": 0})
    ref = proc.predict(d.numpy(), ids.numpy())
    for per_feature in (False, True):
        pb = proc.predict_proto(predict_pb.encode_predict_request(d.numpy(), ids.numpy(), per_feature=per_feature))
        probs, version = predict_pb.decode_predict_response(pb)
        assert version == 4 and np.array_equal(probs, ref)
    Req, Resp, _ = predict_pb.message_classes()
    m = Req(output_filter=["probabilities"])
    m.inputs["dense"].dtype = 1; m.inputs["dense"].float_val.extend(d.numpy().reshape(-1).tolist())
    m.inputs["ids"].dtype = 9; m.inputs["ids"].int64_val.extend(ids.numpy().reshape(-1).tolist())
    r = Resp.FromString(proc.predict_proto(m.SerializeToString()))
    assert list(r.outputs) == ["probabilities"] and np.array_equal(np.asarray(r.outputs["probabilities"].float_val, dtype=np.float32), ref)
    assert proc.process(b"garbage")[0] == 500
    proc.close()


def test_processor_group_serves_from_every_gpu(tmp_path):
    """ModelConfig gpu_ids_list: one replica per GPU, same answers from each (runs with 2 replicas on one GPU when only one is visible)."""
    from deeprec_b200.data import criteo_batch
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    from deeprec_b200.serving import ProcessorGroup, encode_request, export_saved_model, decode_response
    cards = [50, 1000, 7, 300] + [97] * 22
    eng = DLRMEngine(DLRMConfig(batch_size=256, cardinalities=cards, learning_rate=0.05))
    for s in range(3):
        d, ids, y = criteo_batch(eng.B, 13, cards, seed=s)
        eng.load_batch(d.cuda(), ids.cuda(), y.cuda()); eng.train_step()
    root = str(tmp_path)
    export_saved_model(eng, os.path.join(root, "v1"), version=3, root=root)
    gpus = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    grp = ProcessorGroup(os.path.join(root, "v1"), {"session_num": 2, "max_batch": 256, "model_update_interval_ms": 0, "gpu_ids_list": gpus})
    a = grp.predict(d.numpy(), ids.numpy()); b = grp.predict(d.numpy(), ids.numpy())          # round robin: replica 0, then replica 1
    assert np.allclose(a, b, atol=1e-6)
    rc, outs = grp.batch_process([encode_request(d.numpy()[:32], ids.numpy()[:, :32]) for _ in range(5)])
    assert rc == 200 and all(np.allclose(decode_response(o)[0], a[:32], atol=1e-6) for o in outs)
    info = grp.model_info()
    assert info["sessions"] == 4 and info["model_version"] == 3 and all(r["requests"] >= 2 for r in info["replicas"])
    grp.close()
