"""BST on FusedRecEngine on the CUDA-on-CPU emulation, where nn.fused_encoder_layer falls back to the nn.TransformerEncoderLayer module: the
fallback itself, BST.forward against the framework computation it replaced, the engine against a torch replica, micro-batches against one
batch, two ranks as threads against one rank, a checkpoint round trip, and an engine-trained dense net loaded into a fresh zoo.BST and
exported as an op program.  Cases: tests/mha_cases.py; GPU twin: test_gpu_mha.py."""
import threading

import pytest
import torch

import mha_cases as M
import pooled_bag_cases as K
from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(1500)]
DEV = torch.device("cpu")


def test_fused_encoder_layer_fallback_matches_the_module():
    from deeprec_b200.nn import fused_encoder_layer
    layer = M.encoder_layer(32, 4, DEV)
    x = torch.randn(9, 13, 32)
    valid = M.bst_valid(9, 13, 3)
    assert torch.equal(fused_encoder_layer(x, layer, valid), layer(x, src_key_padding_mask=~valid))
    with pytest.raises(ValueError, match="post-norm"):
        fused_encoder_layer(x, M.encoder_layer(32, 4, DEV, norm_first=True), valid)


def test_bst_forward_is_the_framework_computation_bit_for_bit():
    """head() took BST's dense part out of forward(); the framework path must compute exactly what the inline code did."""
    model = K.seq_model("bst", DEV)
    b = K.taobao_like(64, 5)
    u, q, k, mask = model._embed(b)
    x = torch.cat([k, q.unsqueeze(1)], 1)
    x = x + model.pos[: x.shape[1]]
    pad = torch.cat([~mask, torch.zeros(mask.shape[0], 1, dtype=torch.bool)], 1)
    h = model.enc(x, src_key_padding_mask=pad)
    valid = (~pad).unsqueeze(-1).to(h.dtype)
    pooled = (h * valid).sum(1) / valid.sum(1).clamp_min(1)
    want = model.out(model.final(torch.cat([u, q, pooled], -1))).squeeze(-1)
    assert torch.equal(model(b), want)
    with pytest.raises(ValueError, match="positional table"):
        model.head(u, q, torch.zeros(64, model.pos.shape[0], k.shape[2]), torch.ones(64, model.pos.shape[0], dtype=torch.bool))


def test_bst_engine_matches_a_torch_replica():
    with _native.cuda_emulation():
        M.run_bst_vs_replica(DEV, steps=5, B=128)


def test_micro_batches_equal_one_batch():
    from deeprec_b200.models.rec_engine import din_ids
    B, res = 128, []
    with _native.cuda_emulation():
        for mb in (1, 2):
            eng = M.bst_engine(DEV, B, learning_rate=0.05, micro_batch_num=mb)
            losses = []
            for s in range(4):
                b = K.taobao_like(B, 300 + s)
                eng.load_batch(din_ids(b), b["labels"]); eng.train_step(); losses.append(eng.loss_value())
            res.append((losses, eng.params.clone(), eng.tables[1].lookup(torch.arange(K.CARDS[1])).clone()))
    # bf16 autocast: the halves round like the whole batch sample by sample; only the order of the batch sums differs
    assert max(abs(a - b) for a, b in zip(res[0][0], res[1][0])) < 1e-3, (res[0][0], res[1][0])
    assert torch.allclose(res[0][1], res[1][1], atol=1e-3)
    assert torch.allclose(res[0][2], res[1][2], atol=1e-3)


def _rank(rank, W, shared, B, batches, out, errors):
    try:
        from deeprec_b200.models.rec_engine import din_ids
        from deeprec_b200.parallel.emu_comm import EmuComm
        with _native.cuda_emulation():
            with shared.lock:                                    # the default RNG and the variable registry are process-global
                model = K.seq_model("bst", DEV)
            comm = EmuComm(shared, rank) if W > 1 else None
            eng = M.bst_engine(DEV, B, model=model, learning_rate=0.05, rank=rank, world_size=W, comm=comm)
            losses = []
            for b in batches:
                part = {k: v[rank * B:(rank + 1) * B] for k, v in b.items()}
                eng.load_batch(din_ids(part), part["labels"]); eng.train_step(); losses.append(eng.loss_value())
            out[rank] = (losses, eng.params.clone())
            if comm is not None:
                comm.host_barrier()
    except BaseException as e:                                  # noqa: BLE001 -- surfaced by the main thread
        errors.append((rank, repr(e)))
        try:
            shared.barrier.abort()
        except Exception:
            pass
        raise


def _run_world(W, B, batches):
    from deeprec_b200.parallel.emu_comm import EmuWorld
    shared, out, errors = EmuWorld(W), {}, []
    threads = [threading.Thread(target=_rank, args=(r, W, shared, B, batches, out, errors)) for r in range(W)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=1200)
    assert not errors and len(out) == W, errors
    return out


def test_two_ranks_as_threads_equal_one_rank():
    """BST has no BatchNorm: world 2 on two halves of a batch trains like world 1 on the whole batch (global mean loss, summed gradients)."""
    with _native.cuda_emulation():
        pass
    B = 64
    batches = [K.taobao_like(2 * B, 700 + s) for s in range(4)]
    one = _run_world(1, 2 * B, batches)
    two = _run_world(2, B, batches)
    assert torch.equal(two[0][1], two[1][1]), "dense replicas diverged"
    assert max(abs(a - b) for a, b in zip(one[0][0], two[0][0])) < 2e-3, (one[0][0], two[0][0])
    assert torch.allclose(one[0][1], two[0][1], atol=2e-3)


def test_checkpoint_round_trip(tmp_path):
    from deeprec_b200.models.rec_engine import din_ids
    B = 96
    batches = [K.taobao_like(B, 400 + s) for s in range(7)]
    with _native.cuda_emulation():
        eng = M.bst_engine(DEV, B, learning_rate=0.05)
        for s in range(4):
            eng.load_batch(din_ids(batches[s]), batches[s]["labels"]); eng.train_step()
            if s == 1:
                eng.save(str(tmp_path / "ck"))
        eng.save(str(tmp_path / "ck"), incremental=True)
        fresh = M.bst_engine(DEV, B, learning_rate=0.05)
        assert fresh.restore(str(tmp_path / "ck")) == 4
        assert torch.equal(fresh.params, eng.params)
        for t in range(3):
            probe = torch.arange(K.CARDS[t])
            assert torch.equal(fresh.tables[t].lookup(probe), eng.tables[t].lookup(probe)), t
        la, lb = [], []
        for s in range(4, 7):
            for e, l in ((eng, la), (fresh, lb)):
                e.load_batch(din_ids(batches[s]), batches[s]["labels"]); e.train_step(); l.append(e.loss_value())
        assert la == lb, (la, lb)


def test_engine_trained_state_dict_loads_into_a_fresh_bst_and_exports(tmp_path):
    from deeprec_b200.models.rec_engine import din_ids
    from deeprec_b200.serving import export_saved_model_program
    B = 64
    with _native.cuda_emulation():
        eng = M.bst_engine(DEV, B, learning_rate=0.05)
        for s in range(2):
            b = K.taobao_like(B, 500 + s)
            eng.load_batch(din_ids(b), b["labels"]); eng.train_step()
    trained = eng.net.inner.state_dict()
    assert any(k.startswith("enc.self_attn.in_proj_weight") for k in trained)
    fresh = K.seq_model("bst", DEV)
    missing, unexpected = fresh.load_state_dict(trained, strict=False)
    assert not unexpected, unexpected
    assert all(k.split(".")[0] in ("user", "item", "cat") for k in missing), missing
    for k, v in trained.items():
        assert torch.equal(fresh.state_dict()[k], v), k
    export_saved_model_program(fresh, str(tmp_path / "export"), 1, max_len=K.L)
