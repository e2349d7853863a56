"""The flagship DLRMEngine on the CUDA-on-CPU emulation: the hand-scheduled training step that bench.py and smoke() run on an H100 -- unique-first
sparse pipeline, BatchNorm-folded bottom MLP with statistics out of the GEMM epilogue, indirect dot interaction, top MLP, fused head, backward, fused
optimizers -- executes in the CPU test tier with the SIMT kernels compiled for the host and the wgmma GEMMs replaced by host loops with the real
wrappers' argument contracts (csrc/cuda/emu/emu_stubs.cu).  Same fp32 oracle and tolerances as tests/test_gpu_table_engine.py; plus the engine's
checkpoint round trip and the model-parallel step with the ranks as threads."""
import threading

import pytest
import torch

from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(1500)]
CARDS = [50, 1000, 7, 300] + [97] * 22


def _oracle_from_engine(eng):
    from deeprec_b200.models.dlrm import DLRM
    cfg = eng.cfg
    m = DLRM(cfg.num_dense, cfg.cardinalities, cfg.embedding_dim, cfg.mlp_bot, cfg.mlp_top, use_ev=False, device="cpu", bn_eps=cfg.bn_eps, bn_momentum=cfg.bn_momentum)
    with torch.no_grad():
        for layers, mods in ((eng.bot, m.bot), (eng.top, m.top)):
            for L, lin in zip(layers, [l for l in mods if isinstance(l, torch.nn.Linear)]):
                lin.weight.copy_(eng.p(L.name + "/kernel").view(L.N, L.Kp)[:, : L.K]); lin.bias.copy_(eng.p(L.name + "/bias"))
        m.logits.weight.copy_(eng.p("logits/kernel").view(1, -1)); m.logits.bias.copy_(eng.p("logits/bias")[:1])
        for t, emb in enumerate(m.tables):
            dm = eng.tables[t].default_matrix
            emb.weight.copy_(dm[torch.arange(emb.num_embeddings) % dm.shape[0]])
    return m


def _batch(B, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, 13, generator=g) * 3, torch.stack([torch.randint(0, c, (B,), generator=g) for c in CARDS]), (torch.rand(B, generator=g) < 0.3).float())


def test_dlrm_engine_on_the_emulation_matches_the_fp32_oracle(tmp_path):
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    torch.manual_seed(0)
    cfg = DLRMConfig(batch_size=256, cardinalities=CARDS, optimizer="adagrad", learning_rate=0.05)
    with _native.cuda_emulation():
        eng = DLRMEngine(cfg)
        m = _oracle_from_engine(eng)
        o_dense = torch.optim.Adagrad([p for n, p in m.named_parameters() if not n.startswith("tables")], lr=0.05, initial_accumulator_value=0.1, eps=0.0)
        o_emb = torch.optim.Adagrad(m.tables.parameters(), lr=0.05, initial_accumulator_value=0.1, eps=0.0)
        le, lr_ = [], []
        for s in range(4):
            dense, ids, labels = _batch(cfg.batch_size, 10 + s)
            eng.load_batch(dense, ids, labels)
            if s == 0:
                eng.capture()                      # on the emulation: the eager step
            else:
                eng.train_step()
            le.append(eng.loss_value())
            loss = m.loss(dense, ids, labels)
            o_dense.zero_grad(); o_emb.zero_grad(); loss.backward(); o_dense.step(); o_emb.step()
            lr_.append(loss.item())
        for a, b in zip(le, lr_):
            assert abs(a - b) < 0.02 * max(1.0, abs(b)), (le, lr_)
        lin0 = [l for l in m.bot if isinstance(l, torch.nn.Linear)][0]
        assert (eng.p("mlp_bot_0/kernel").view(512, 16)[:, :13] - lin0.weight).abs().max().item() < 0.05
        keys = ids[1][:64]
        assert (eng.tables[1].lookup(keys) - m.tables[1].weight[keys]).abs().max().item() < 0.05
        assert eng.tables[0].overflowed() == 0
        # training-state checkpoint: full save -> fresh engine -> identical continuation
        eng.save(str(tmp_path / "dlrm"))
        b2 = DLRMEngine(cfg)
        assert b2.restore(str(tmp_path / "dlrm")) == 4
        assert torch.equal(eng.params, b2.params)
        nxt = _batch(cfg.batch_size, 99)
        out = []
        for e in (eng, b2):
            e.load_batch(*nxt); e.train_step(); out.append(e.loss_value())
        assert abs(out[0] - out[1]) < 1e-4, out
        p = eng.predict()
        assert p.shape == (cfg.batch_size,) and bool(((p >= 0) & (p <= 1)).all())


def _rank(rank, W, shared, steps, out, errors):
    try:
        from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
        from deeprec_b200.parallel.emu_comm import EmuComm
        with _native.cuda_emulation():
            with shared.lock:
                torch.manual_seed(0)
                cfg = DLRMConfig(batch_size=128, cardinalities=CARDS, optimizer="adagrad", learning_rate=0.05)
            eng = DLRMEngine(cfg, None, rank, W, EmuComm(shared, rank))
            losses = []
            for s in range(steps):
                eng.load_batch(*_batch(128, 500 + 10 * s + rank)); eng.train_step(); losses.append(eng.loss_value())
            out[rank] = (losses, eng.params.clone(), sum(t.size() for t in eng.tables.values()))
            eng.comm.host_barrier()
    except BaseException as e:                                  # noqa: BLE001
        errors.append((rank, repr(e)))
        try:
            shared.barrier.abort()
        except Exception:
            pass
        raise


def test_dlrm_engine_model_parallel_with_ranks_as_threads():
    """World 2: identical dense replicas after every fused all-reduce + optimizer step, one global loss, every key on exactly one owner."""
    from deeprec_b200.parallel.emu_comm import EmuWorld
    with _native.cuda_emulation():
        pass
    W, steps = 2, 4
    shared, out, errors = EmuWorld(W), {}, []
    threads = [threading.Thread(target=_rank, args=(r, W, shared, steps, out, errors)) for r in range(W)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=1200)
    assert not errors and len(out) == W, errors
    assert torch.equal(out[0][1], out[1][1]), "dense replicas diverged"
    assert max(abs(a - b) for a, b in zip(out[0][0], out[1][0])) < 1e-6 and all(l == l for l in out[0][0])
    distinct = sum(len(set(torch.cat([_batch(128, 500 + 10 * s + r)[1][t] for s in range(steps) for r in range(W)]).tolist())) for t in range(26))
    assert out[0][2] + out[1][2] == distinct, (out[0][2], out[1][2], distinct)
