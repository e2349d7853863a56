"""The linear (wide) embedding group on the CUDA-on-CPU emulation: k_sp_linear_fwd / k_sp_linear_bwd against their numpy oracles bit for bit at
world 1 and with 2 / 3 ranks as threads, and FusedRecEngine(linear=True) -- Wide & Deep -- against a torch replica, FTRL on the linear group,
micro-batches, checkpoints and the model-parallel step.  Cases: tests/linear_group_cases.py; GPU twin: test_gpu_linear_group.py."""
import threading

import pytest
import torch

import linear_group_cases as K
from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(1500)]
DEV = torch.device("cpu")


@pytest.mark.parametrize("C", [26, 1])
def test_linear_kernels_world1_bit_for_bit(C):
    with _native.cuda_emulation():
        K.run_kernels_world1(DEV, C, 1000, owner=0x5100 + C)


@pytest.mark.parametrize("W", [2, 3])
def test_linear_kernels_ranks_as_threads(W):
    with _native.cuda_emulation():          # build + load the library on the main thread (the rank threads must not fork a compiler)
        pass
    K.run_kernels_ranks_as_threads(W, owner=0x5200 + 1000 * W)


@pytest.mark.parametrize("linear_sgd", [False, True], ids=["adagrad", "linear_sgd"])
def test_wdl_engine_matches_a_torch_replica(linear_sgd):
    with _native.cuda_emulation():
        K.run_engine_vs_replica(DEV, linear_sgd)


def test_wdl_engine_ftrl_on_the_linear_group():
    with _native.cuda_emulation():
        K.run_ftrl_one_step(DEV)


def test_wdl_engine_micro_batches_equal_one_batch():
    """micro_batch_num=4 == 1 (WDL has no batch statistics): the linear logits are sliced with the batch, their gradients land in their slices.
    The dense net runs in fp32 here so that the only difference is the order of the parameter-gradient sums."""
    from deeprec_b200.models.rec_engine import FusedRecEngine, _StripTables
    from deeprec_b200.models.zoo import build_model
    import deeprec_b200 as dr
    B, res = 128, []
    with _native.cuda_emulation():
        for M in (1, 4):
            dr.embedding_variable.clear_registry()
            torch.manual_seed(0)
            net = _StripTables(build_model("wdl", device="cpu"))
            fwd = lambda net, dense, emb, ids, linear: net.inner.wide_deep_logits(dense["dense"], emb.float(), linear[:, None])
            eng = FusedRecEngine(net, fwd, list(range(26)), K.CARDS, B, dense_inputs={"dense": ((B, 13), torch.float32)}, learning_rate=0.05,
                                 linear=True, micro_batch_num=M)
            losses = []
            for s in range(4):
                eng.load_batch(*K.engine_batch(B, 700 + s)); eng.train_step(); losses.append(eng.loss_value())
            probe = torch.arange(300)
            res.append((losses, eng.params.clone(), eng.lin_tables[3].lookup(probe).clone(), eng.tables[3].lookup(probe).clone()))
    assert max(abs(a - b) for a, b in zip(res[0][0], res[1][0])) < 1e-5, (res[0][0], res[1][0])
    assert torch.allclose(res[0][1], res[1][1], atol=1e-5)
    assert torch.allclose(res[0][2], res[1][2], atol=1e-5) and torch.allclose(res[0][3], res[1][3], atol=1e-4)


def test_wdl_engine_checkpoint_round_trip(tmp_path):
    """Full + incremental save -> restore into a fresh engine: identical parameters and linear rows, identical continuation."""
    B = 128
    batches = [K.engine_batch(B, 800 + s) for s in range(8)]
    with _native.cuda_emulation():
        eng = K.wdl_engine(DEV, B, learning_rate=0.05, linear_optimizer="ftrl", linear_learning_rate=0.2)
        for s in range(5):
            eng.load_batch(*batches[s]); eng.train_step()
            if s == 2:
                eng.save(str(tmp_path / "ck"))
        eng.save(str(tmp_path / "ck"), incremental=True)
        fresh = K.wdl_engine(DEV, B, learning_rate=0.05, linear_optimizer="ftrl", linear_learning_rate=0.2)
        assert fresh.restore(str(tmp_path / "ck")) == 5
        assert torch.equal(fresh.params, eng.params) and torch.equal(fresh.lin_hp_dev, eng.lin_hp_dev)
        for t in (0, 1, 3):
            probe = torch.arange(K.CARDS[t])
            assert torch.equal(fresh.lin_tables[t].lookup(probe), eng.lin_tables[t].lookup(probe)), t
            assert torch.equal(fresh.tables[t].lookup(probe), eng.tables[t].lookup(probe)), t
        la, lb = [], []
        for s in range(5, 8):
            for e, l in ((eng, la), (fresh, lb)):
                e.load_batch(*batches[s]); e.train_step(); l.append(e.loss_value())
        assert la == lb, (la, lb)


def _wdl_rank(rank, W, shared, B, out, errors, ckpt):
    try:
        import torch.distributed as dist
        from deeprec_b200.parallel.emu_comm import EmuComm
        with _native.cuda_emulation():
            with shared.lock:                                    # the default RNG and the variable registry are process-global
                model = K.wdl_model(DEV)
            eng = K.wdl_engine(DEV, B, model=model, learning_rate=0.05, rank=rank, world_size=W, comm=EmuComm(shared, rank))
            losses = []
            for s in range(3):
                eng.load_batch(*K.engine_batch(B, 900 + 10 * s + rank)); eng.train_step(); losses.append(eng.loss_value())
            p = eng.predict()
            assert p.shape == (B,) and bool(((p >= 0) & (p <= 1)).all())
            for s in range(3, 5):
                eng.load_batch(*K.engine_batch(B, 900 + 10 * s + rank)); eng.train_step(); losses.append(eng.loss_value())
            dist_barrier = dist.barrier
            dist.barrier = lambda *a, **k: shared.barrier.wait()      # save_engine's collective barrier, across the rank threads
            try:
                eng.save(ckpt)
            finally:
                dist.barrier = dist_barrier
            keys = [torch.arange(c) for c in K.CARDS]
            out[rank] = (losses, eng.params.clone(), [eng.lin_tables[t].get_freq(keys[t]) for t in range(26)],
                         [eng.lin_tables[t].lookup(keys[t]).clone() for t in range(26)])
            eng.comm.host_barrier()
    except BaseException as e:                                  # noqa: BLE001
        errors.append((rank, repr(e)))
        try:
            shared.barrier.abort()
        except Exception:
            pass
        raise


def test_wdl_engine_ranks_as_threads_and_world2_checkpoint_at_world1(tmp_path):
    """World 2: identical dense replicas and global loss on both ranks, every linear key on exactly one owner, train -> predict -> train keeps
    the ranks in step; the world-2 checkpoint restores into a world-1 engine."""
    from deeprec_b200.checkpoint.engine_ckpt import sp_owner
    from deeprec_b200.parallel.emu_comm import EmuWorld
    with _native.cuda_emulation():
        pass
    W, B = 2, 96
    ckpt = str(tmp_path / "ck2")
    shared, out, errors = EmuWorld(W), {}, []
    threads = [threading.Thread(target=_wdl_rank, args=(r, W, shared, B, out, errors, ckpt)) for r in range(W)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=1200)
    assert not errors and len(out) == W, errors
    assert torch.equal(out[0][1], out[1][1]), "dense replicas diverged"
    assert max(abs(a - b) for a, b in zip(out[0][0], out[1][0])) < 1e-6
    rows = []
    for t in range(26):
        freq = torch.stack([out[r][2][t] for r in range(W)])
        assert int(((freq > 0).sum(0) > 1).sum()) == 0, f"table {t}: a linear key lives on two owners"
        owner = sp_owner(torch.arange(K.CARDS[t]), W)
        assert bool((freq[1 - owner, torch.arange(K.CARDS[t])] == 0).all()), t
        rows.append(torch.stack([out[r][3][t] for r in range(W)])[owner, torch.arange(K.CARDS[t])])
    with _native.cuda_emulation():
        one = K.wdl_engine(DEV, B, learning_rate=0.05)
        assert one.restore(ckpt) == 5
        assert torch.equal(one.params, out[0][1])
        for t in range(26):
            seen = torch.stack([out[r][2][t] for r in range(W)]).sum(0) > 0
            got = one.lin_tables[t].lookup(torch.arange(K.CARDS[t]))
            assert torch.equal(got[seen], rows[t][seen]), t
