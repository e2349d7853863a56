"""Multi-hot bags on the CUDA-on-CPU emulation: k_sp_pool / k_sp_pool_segsum against their oracles for sum, mean and sqrtn at world 1 and with
2 / 3 ranks as threads; FusedRecEngine(bags=...) through pooled_seq_engine -- DSSM (sum, mean), ESMM and MMoE -- against a torch replica,
micro-batches, a checkpoint round trip and the launch count.  Cases: tests/pooled_bag_cases.py; GPU twin: test_gpu_pooled_bags.py."""
import ctypes

import pytest
import torch

import pooled_bag_cases as K
from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(1500)]
DEV = torch.device("cpu")
COMBS = ["sum", "mean", "sqrtn"]


@pytest.mark.parametrize("comb", COMBS)
def test_pool_kernels_world1(comb):
    with _native.cuda_emulation():
        K.run_kernels_world1(DEV, comb, 200, owner=0x7100 + COMBS.index(comb))


@pytest.mark.parametrize("comb", ["sum", "sqrtn"])
@pytest.mark.parametrize("W", [2, 3])
def test_pool_kernels_ranks_as_threads(W, comb):
    with _native.cuda_emulation():          # build + load the library on the main thread (the rank threads must not fork a compiler)
        pass
    K.run_kernels_ranks_as_threads(W, comb, owner=0x7200 + 1000 * W + COMBS.index(comb))


def test_bags_are_validated():
    from deeprec_b200.models.rec_engine import FusedRecEngine
    from deeprec_b200.parallel.sparse_pipeline import Bags
    with pytest.raises(ValueError, match="sum to"):
        Bags(DEV, [(2, "sum"), (2, "sum")], 5)
    with pytest.raises(ValueError, match="combiner"):
        Bags(DEV, [(5, "max")], 5)
    with pytest.raises(ValueError, match="at least one id column"):
        Bags(DEV, [(0, "sum"), (5, "sum")], 5)
    with _native.cuda_emulation():
        with pytest.raises(ValueError, match="linear"):
            FusedRecEngine(torch.nn.Linear(16, 1), lambda *a, **k: None, [0, 0], [100], 8, bags=[(2, "sum")], linear=True)


@pytest.mark.parametrize("name,comb", [("dssm", "sum"), ("dssm", "mean"), ("esmm", "sum"), ("mmoe", "sum")])
def test_engine_matches_a_torch_replica(name, comb):
    with _native.cuda_emulation():
        K.run_engine_vs_replica(name, DEV, comb)


@pytest.mark.parametrize("name", ["dbmtl", "ple", "simple_multitask"])
def test_other_multitask_models_train_on_the_engine(name):
    """One step of each remaining multi-task model: the engine's loss equals the model's own loss on a replica before any update."""
    B = 64
    with _native.cuda_emulation():
        eng = K.seq_engine(name, DEV, B, "sum", learning_rate=0.05)
        rep = K.replica_of(eng, DEV, "sum")
        b = K.taobao_like(B, 600)
        eng.load_batch(*K.engine_inputs(eng, b, DEV)); eng.train_step()
        want = rep.loss(b).item()
        assert abs(eng.loss_value() - want) < 0.03 * max(1.0, abs(want)), (eng.loss_value(), want)
        p = eng.predict()
        assert set(p) == {"ctr", "cvr"} and all(v.shape == (B,) for v in p.values())


def _fp32_dssm_engine(B, M):
    """DSSM with mean bags and its dense net in fp32, so that micro-batches differ from one batch only in the order of the gradient sums."""
    from deeprec_b200.models.rec_engine import FusedRecEngine, _StripTables
    net = _StripTables(K.seq_model("dssm", DEV))

    def fwd(net, dense, emb, ids):
        e = emb.float()
        return net.inner.head(e[:, 0], torch.cat([e[:, 1], e[:, 2]], -1), torch.cat([e[:, 3], e[:, 4]], -1))
    col_table = [0, 1, 2] + [1] * K.L + [2] * K.L
    return FusedRecEngine(net, fwd, col_table, list(K.CARDS), B, learning_rate=0.05, micro_batch_num=M,
                          bags=[(1, "mean")] * 3 + [(K.L, "mean")] * 2)


def test_micro_batches_equal_one_batch():
    from deeprec_b200.models.rec_engine import din_ids
    B, res = 128, []
    with _native.cuda_emulation():
        for M in (1, 2):
            eng = _fp32_dssm_engine(B, M)
            losses = []
            for s in range(4):
                b = K.taobao_like(B, 300 + s)
                eng.load_batch(din_ids(b), b["labels"]); eng.train_step(); losses.append(eng.loss_value())
            probe = torch.arange(K.CARDS[1])
            res.append((losses, eng.params.clone(), eng.tables[1].lookup(probe).clone()))
    assert max(abs(a - b) for a, b in zip(res[0][0], res[1][0])) < 1e-5, (res[0][0], res[1][0])
    assert torch.allclose(res[0][1], res[1][1], atol=1e-5)
    assert torch.allclose(res[0][2], res[1][2], atol=1e-4)


def test_checkpoint_round_trip(tmp_path):
    """Bags add no trained state: full + incremental save -> restore into a fresh ESMM engine, identical parameters, rows and continuation."""
    B = 96
    batches = [K.taobao_like(B, 400 + s) for s in range(7)]
    with _native.cuda_emulation():
        eng = K.seq_engine("esmm", DEV, B, "mean", learning_rate=0.05)
        for s in range(4):
            eng.load_batch(*K.engine_inputs(eng, batches[s], DEV)); eng.train_step()
            if s == 1:
                eng.save(str(tmp_path / "ck"))
        eng.save(str(tmp_path / "ck"), incremental=True)
        fresh = K.seq_engine("esmm", DEV, B, "mean", learning_rate=0.05)
        assert fresh.restore(str(tmp_path / "ck")) == 4
        assert torch.equal(fresh.params, eng.params)
        for t in range(3):
            probe = torch.arange(K.CARDS[t])
            assert torch.equal(fresh.tables[t].lookup(probe), eng.tables[t].lookup(probe)), t
        la, lb = [], []
        for s in range(4, 7):
            for e, l in ((eng, la), (fresh, lb)):
                e.load_batch(*K.engine_inputs(e, batches[s], DEV)); e.train_step(); l.append(e.loss_value())
        assert la == lb, (la, lb)


def test_launches_per_step_match_the_emulator_and_the_engine_without_bags():
    from deeprec_b200.models.rec_engine import FusedRecEngine, din_ids
    B = 64
    col_table = [0, 1, 2] + [1] * K.L + [2] * K.L
    C = len(col_table)
    counts = {}
    with _native.cuda_emulation():
        lib = _native.cuda()
        lib.dr_cuda_emu_launch_count.restype = ctypes.c_int64
        for bags in (None, [(1, "sum")] * 3 + [(K.L, "sqrtn")] * 2):
            F = C if bags is None else len(bags)
            eng = FusedRecEngine(torch.nn.Linear(F * 16, 1), lambda net, dense, emb, ids: net(emb.float().flatten(1)).squeeze(-1), col_table,
                                 list(K.CARDS), B, bags=bags)
            seen = []
            for s in range(2):
                b = K.taobao_like(B, 500 + s)
                eng.load_batch(din_ids(b), b["labels"])
                c0, n0 = lib.dr_cuda_emu_launch_count(), eng.launches
                eng.train_step()
                seen.append((eng.launches - n0, lib.dr_cuda_emu_launch_count() - c0))
            assert all(a == b for a, b in seen), seen
            counts[bags is None] = seen[-1][0]
    assert counts[True] == counts[False], counts
