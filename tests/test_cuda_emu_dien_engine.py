"""DIEN on FusedRecEngine on the CUDA-on-CPU emulation, where nn.fused_gru falls back to the nn.GRU module: the engine against a torch
replica, micro-batches against one batch, two ranks as threads against one rank, a checkpoint round trip, and the fallback itself.
Cases: tests/gru_cases.py; GPU twin: test_gpu_gru.py."""
import threading

import pytest
import torch

import gru_cases as G
import pooled_bag_cases as K
from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(1500)]
DEV = torch.device("cpu")


def test_fused_gru_fallback_matches_the_module():
    from deeprec_b200.nn import fused_gru
    torch.manual_seed(0)
    gru = torch.nn.GRU(12, 16, batch_first=True)
    x = torch.randn(9, 7, 12)
    lengths = torch.tensor([7, 0, 1, 3, 7, 2, 5, 6, 4])
    y = fused_gru(x, gru, lengths)
    ref, _ = gru(x)
    live = torch.arange(7)[None] < lengths[:, None]
    assert torch.equal(y[live], ref[live])
    assert bool((y[~live] == 0).all())


def test_dien_engine_matches_a_torch_replica():
    with _native.cuda_emulation():
        G.run_dien_vs_replica(DEV, steps=5, B=128)


def test_micro_batches_equal_one_batch():
    from deeprec_b200.models.rec_engine import din_ids
    B, res = 128, []
    with _native.cuda_emulation():
        for M in (1, 2):
            eng = G.dien_engine(DEV, B, learning_rate=0.05, micro_batch_num=M)
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
                model = K.seq_model("dien", DEV)
            comm = EmuComm(shared, rank) if W > 1 else None
            eng = G.dien_engine(DEV, B, model=model, learning_rate=0.05, rank=rank, world_size=W, comm=comm)
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
    """DIEN has no BatchNorm: world 2 on two halves of a batch trains like world 1 on the whole batch (global mean loss, summed gradients)."""
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
        eng = G.dien_engine(DEV, B, learning_rate=0.05)
        for s in range(4):
            eng.load_batch(din_ids(batches[s]), batches[s]["labels"]); eng.train_step()
            if s == 1:
                eng.save(str(tmp_path / "ck"))
        eng.save(str(tmp_path / "ck"), incremental=True)
        fresh = G.dien_engine(DEV, B, learning_rate=0.05)
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
