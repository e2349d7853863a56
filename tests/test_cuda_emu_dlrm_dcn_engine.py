"""DLRMEngine with interaction_op="dcnv2" (DLRM-DCNv2) on the CUDA-on-CPU emulation: the cross-layer GEMM epilogues (host-loop stand-in of
dr_cuda_gemm_tn_cross), the cross backward and split kernels, the pitched gather into x0 and k_sp_segsum at dim 128, against the fp32
``DLRM(interaction_op="dcnv2")`` oracle; plus the checkpoint round trip, two ranks as threads, and the configurations the engine refuses."""
import threading

import pytest
import torch

from deeprec_b200 import _native
from dlrm_dcn_cases import CARDS, batch, bn_stats, oracle_from_engine, param_pairs, rel_err, small_config

pytestmark = [pytest.mark.timeout(1500)]


def test_dcnv2_engine_matches_the_fp32_oracle_over_three_steps(tmp_path):
    from deeprec_b200.models.dlrm_engine import DLRMEngine
    torch.manual_seed(0)
    cfg = small_config()
    with _native.cuda_emulation():
        eng = DLRMEngine(cfg)
        m = oracle_from_engine(eng)
        o_dense = torch.optim.Adagrad([p for n, p in m.named_parameters() if not n.startswith("tables")], lr=0.05, initial_accumulator_value=0.1, eps=0.0)
        o_emb = torch.optim.Adagrad(m.tables.parameters(), lr=0.05, initial_accumulator_value=0.1, eps=0.0)
        touched = []
        for s in range(3):
            dense, ids, labels = batch(cfg.batch_size, 10 + s)
            touched.append(ids)
            eng.load_batch(dense, ids, labels)
            eng.train_step()
            logits = m(dense, ids)
            loss = torch.nn.functional.binary_cross_entropy_with_logits(logits, labels)
            o_dense.zero_grad(); o_emb.zero_grad(); loss.backward()
            # bf16 activations (relative rounding 2^-9) through ~8 layers move the mean loss by ~1e-4 at most here; 5e-3 leaves room and still
            # fails when a cross term is dropped (the loss then moves by > 1e-2)
            assert abs(eng.loss_value() - loss.item()) < 5e-3, (s, eng.loss_value(), loss.item())
            assert (eng.prob - torch.sigmoid(logits)).abs().max().item() < 1e-2
            if s == 0:
                # the first step's gradients, before the two models can drift apart.  Batch sums of bf16 products with mixed signs lose up to
                # ~8 bits to cancellation, and the BatchNorm backward subtracts batch means, so the bottom layers' relative errors reach ~0.2;
                # the cross layers' stay near 0.1.  A wrong factor in a cross gradient gives an error of order 1.
                for name, e, o in param_pairs(eng, m, grads=True):
                    bound = 0.2 if name.startswith("low_rank_cross_net") else 0.02 if name.startswith("logits") else 0.35
                    assert rel_err(e, o.grad) < bound, (name, rel_err(e, o.grad))
            o_dense.step(); o_emb.step()
        # Adagrad steps of lr 0.05 on gradients of ~1e-3 move a parameter by ~1e-4 per step; the engine's parameters stay within 2e-3
        for name, e, o in param_pairs(eng, m):
            assert (e - o).abs().max().item() < 2e-3, name
        for rm_e, rm_o, rv_e, rv_o in bn_stats(eng, m):
            assert (rm_e - rm_o).abs().max().item() < 1e-3 and (rv_e - rv_o).abs().max().item() < 1e-3
        for t in (0, 1, 3):
            keys = torch.unique(torch.cat([ids[t] for ids in touched]))[:64]
            assert (eng.tables[t].lookup(keys) - m.tables[t].weight[keys]).abs().max().item() < 1e-3, t
        # checkpoint: full save -> fresh engine -> identical continuation
        eng.save(str(tmp_path / "dcn"))
        b2 = DLRMEngine(cfg)
        assert b2.restore(str(tmp_path / "dcn")) == 3
        assert torch.equal(eng.params, b2.params)
        nxt = batch(cfg.batch_size, 99)
        out = []
        for e in (eng, b2):
            e.load_batch(*nxt); e.train_step(); out.append((e.loss_value(), e.params.clone()))
        assert out[0][0] == out[1][0] and torch.equal(out[0][1], out[1][1])
        sd = eng.state_dict()
        assert "low_rank_cross_net_1_w/bias" in sd and sd["low_rank_cross_net_0_v/kernel"].numel() == 32 * 27 * 16
        p = eng.predict()
        assert p.shape == (cfg.batch_size,) and bool(((p >= 0) & (p <= 1)).all())


def _rank(rank, W, shared, steps, out, errors):
    try:
        from deeprec_b200.models.dlrm_engine import DLRMEngine
        from deeprec_b200.parallel.emu_comm import EmuComm
        with _native.cuda_emulation():
            cfg = small_config(batch_size=128 if W == 2 else 256)     # the weights come from cfg.seed, the same on every rank
            eng = DLRMEngine(cfg, None, rank, W, EmuComm(shared, rank) if W > 1 else None)
            losses = []
            for s in range(steps):
                d, ids, y = batch(256, 500 + s)                    # one global batch per step, split by rank
                lo, hi = (rank * 128, rank * 128 + 128) if W == 2 else (0, 256)
                eng.load_batch(d[lo:hi], ids[:, lo:hi], y[lo:hi]); eng.train_step(); losses.append(eng.loss_value())
            out[rank] = (losses, eng.params.clone())
            if W > 1:
                eng.comm.host_barrier()
    except BaseException as e:                                  # noqa: BLE001
        errors.append((rank, repr(e)))
        try:
            shared.barrier.abort()
        except Exception:
            pass
        raise


def test_dcnv2_two_ranks_as_threads_match_one_rank():
    """World 2 on the two halves of each global batch against world 1 on the whole batch.  The dense replicas are bit-identical; against world
    1 they differ by the order of the batch sums and by BatchNorm, which normalises with each rank's own batch statistics (as one worker of the
    reference does), so the parameters agree to 5e-3 after three steps rather than bit for bit."""
    from deeprec_b200.parallel.emu_comm import EmuWorld
    with _native.cuda_emulation():
        pass
    steps, out1, errors = 3, {}, []
    _rank(0, 1, None, steps, out1, errors)
    assert not errors, errors
    W = 2
    shared, out, errors = EmuWorld(W), {}, []
    threads = [threading.Thread(target=_rank, args=(r, W, shared, steps, out, errors)) for r in range(W)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=1200)
    assert not errors and len(out) == W, errors
    assert torch.equal(out[0][1], out[1][1]), "dense replicas diverged"
    for a, b in zip(out[0][0], out1[0][0]):
        assert abs(a - b) < 1e-3, (out[0][0], out1[0][0])
    assert (out[0][1] - out1[0][1]).abs().max().item() < 5e-3


@pytest.mark.parametrize("dim", [16, 64, 128])
def test_segsum_against_a_float64_per_key_sum(dim):
    """k_sp_segsum through the pipeline: demb rows summed per distinct key, checked against float64 (dim 128 sums a row in two 64-wide passes)."""
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
    B, C = 96, 3
    g = torch.Generator().manual_seed(dim)
    ids = torch.randint(0, 9, (C, B), generator=g)
    ids[1, ::7] = -1                                            # padding contributes nothing
    demb = (torch.randn(C, B, dim, generator=g) * 0.5).bfloat16()
    with _native.cuda_emulation():
        sp = SparsePipeline(torch.device("cpu"), 0, 1, list(range(C)), C, B, dim)
        sp.dedup(ids.contiguous())
        sp.segsum(demb)
        got = sp.ugrad.double() / float(1 << 40)                # int64 fixed point, 40 fractional bits (ugrad_fix)
        for c in range(C):
            for k in ids[c].unique().tolist():
                if k < 0:
                    continue
                rows = demb[c][ids[c] == k].double().sum(0)
                gs = int(sp.invT[c][(ids[c] == k).nonzero()[0, 0]])
                # members of a key are added in fp32 per 32-sample tile (relative 2^-24 per add), the tiles in exact fixed point
                assert (got[gs] - rows).abs().max().item() < 1e-5 * max(1.0, rows.abs().max().item()), (c, k)


def test_dcnv2_refusals():
    from deeprec_b200.models.dlrm_engine import DLRMEngine
    from deeprec_b200.serving.export import export_delta, export_saved_model
    with _native.cuda_emulation():
        for kw in (dict(fuse_interaction_gemm=True), dict(embedding_dim=8, mlp_bot=(32, 8)), dict(embedding_dim=48, mlp_bot=(32, 48)),
                   dict(mlp_bot=(32, 32)), dict(dcn_low_rank_dim=12), dict(interaction_op="cat")):
            with pytest.raises(ValueError):
                DLRMEngine(small_config(**kw))

        class _Nccl:                                            # the NCCL baseline communicator has no unique-first pipeline
            unique_first = False
        with pytest.raises(ValueError):
            DLRMEngine(small_config(), None, 0, 2, _Nccl())
        eng = DLRMEngine(small_config(batch_size=64))
        with pytest.raises(ValueError):
            export_saved_model(eng, "/nonexistent/never-written")
        with pytest.raises(ValueError):
            export_delta(eng, "/nonexistent/never-written", 0)
