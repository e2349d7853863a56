"""Engine exports (serving.export_engine_program / export_engine_delta) served by the CPU Processor and the GPU runtime on the CUDA-on-CPU
emulation, against the fp32 oracle of tests/engine_export_cases.py; the cross_linear op and the sqrtn mode of seq_mean against float64.
GPU twin: tests/test_gpu_zzzzzzzzz_engine_export.py."""
import json
import os
import threading
import time

import numpy as np
import pytest
import torch

import engine_export_cases as K
from deeprec_b200 import _native
from deeprec_b200.serving import Processor, export_engine_delta, export_engine_program

pytestmark = [pytest.mark.timeout(1500)]
DEV = torch.device("cpu")
TOL = 3e-2            # bf16 activations between the layers of the emulated GPU runtime (probabilities)
CPU_TOL = 1e-4        # the fp32 host interpreter
B = 64


def _cfg(**kw):
    return {"session_num": 1, "max_batch": 40, "model_update_interval_ms": 0, **kw}


def _serve_both(path, dense, ids, ref, **cfg):
    """Both Processors on one request of B > max_batch rows (chunked) and on its first 3 rows."""
    for dev, tol in (("cpu", CPU_TOL), ("cuda_emu", TOL)):
        p = Processor(path, _cfg(**cfg), device=dev)
        try:
            assert K.max_err(p.predict(dense, ids), ref) < tol, (dev, K.max_err(p.predict(dense, ids), ref))
            assert K.max_err(p.predict(dense[:3], ids[:, :3]), ref[:3]) < tol, dev
        finally:
            p.close()


def _wait(pred, timeout=60.0):
    t0 = time.time()
    while time.time() - t0 < timeout:
        if pred():
            return True
        time.sleep(0.05)
    return False


@pytest.mark.parametrize("name,comb", [(n, "sum") for n in K.CRITEO + K.DIN_FAMILY + K.POOLED] + [("dssm", "mean"), ("dssm", "sqrtn"),
                                                                                                   ("dlrm_dcnv2", None)])
def test_engine_export_matches_the_oracle(tmp_path, name, comb):
    with _native.cuda_emulation():
        eng = K.dlrm_dcn_engine(DEV, B) if name == "dlrm_dcnv2" else K.make_engine(name, DEV, B, combiner=comb)
        dense, ids = K.train(eng, name, B, 3, 10)
        if name in K.CRITEO or name == "dlrm_dcnv2":
            ids = ids.clone(); ids[1, :8] += 10 ** 9                 # unseen keys read the exported default rows
        ref = K.oracle(eng, name, dense, ids, comb)
        root = str(tmp_path)
        export_engine_program(eng, os.path.join(root, "v"), root=root)
        meta = json.load(open(os.path.join(root, "v", "saved_model.json")))
        assert meta["version"] == meta["global_step"] == 3
        if name == "wdl":                                            # the linear group: tables T .. 2T-1 read the same request rows
            assert meta["num_tables"] == 52 and meta["id_map"] == list(range(26)) * 2
        _serve_both(os.path.join(root, "v"), *K.request(name, dense, ids), ref)


def test_tiered_table_rows_come_from_the_dram_tier(tmp_path):
    """Table 1 keeps 256 rows in HBM while 1000 of its keys rotate through the batches: rows demoted to the DRAM tier are exported from there."""
    Bt = 128
    batches = []
    for s in range(7):
        ids, y, dense = K.criteo_inputs(Bt, 10 + s)
        ids[1] = torch.randint(0, 250, (Bt,), generator=torch.Generator().manual_seed(s)) + (s % 4) * 250
        batches.append((ids, y, dense))
    with _native.cuda_emulation():
        eng = K.make_engine("deepfm", DEV, Bt, tiered={1: {"cache_rows": 256, "strategy": 0}})
        eng.prefetch(batches[0][0])
        for s, (ids, y, dense) in enumerate(batches[:6]):
            eng.load_batch(ids, y, {"dense": dense})
            eng.train_step()
            eng.prefetch(batches[s + 1][0])
        mgr = eng.tiers[1][0]
        mgr.drain()
        held = mgr.host.snapshot()["keys"]
        assert held.numel() > 0 and not torch.isin(held, eng.tables[1].snapshot()["keys"]).all()
        ids, _, dense = batches[0]                                   # keys last trained in step 1, most of them demoted since
        ref = K.oracle(eng, "deepfm", dense, ids)
        root = str(tmp_path)
        export_engine_program(eng, os.path.join(root, "v"), root=root)
        _serve_both(os.path.join(root, "v"), *K.request("deepfm", dense, ids), ref)
        ids7, y7, dense7 = batches[6]                                # a delta over both tiers: exactly the keys of the step after the export
        eng.load_batch(ids7, y7, {"dense": dense7})
        eng.train_step()
        prefix = export_engine_delta(eng, root, base_version=6)
        assert _delta_keys(prefix, 1) == set(ids7[1].tolist())


def _delta_keys(prefix, t):
    from deeprec_b200.checkpoint.saver import BundleReader
    rd = BundleReader(prefix)
    try:
        return set(rd.read(f"table/{t}-sparse_incr_keys").tolist())
    finally:
        rd.close()


@pytest.mark.parametrize("name", ["deepfm", "dlrm_dcnv2"])
def test_delta_reaches_the_processors_and_leaves_the_checkpoint_chain_whole(tmp_path, name):
    with _native.cuda_emulation():
        mk = (lambda: K.dlrm_dcn_engine(DEV, B)) if name == "dlrm_dcnv2" else (lambda: K.make_engine(name, DEV, B))
        eng = mk()
        dense, ids = K.train(eng, name, B, 3, 10)
        root, ck = str(tmp_path / "serve"), str(tmp_path / "ckpt" / "model")
        eng.save(ck)
        export_engine_program(eng, os.path.join(root, "v3"), root=root)
        ref = K.oracle(eng, name, dense, ids)
        req = K.request(name, dense, ids)
        procs = [Processor(os.path.join(root, "v3"), _cfg(checkpoint_dir=root, model_update_interval_ms=100), device=d) for d in ("cpu", "cuda_emu")]
        try:
            assert K.max_err(procs[0].predict(*req), ref) < CPU_TOL
            # version boundary: rows updated by the first step after the base export are in the delta, rows untouched since are not
            K.train(eng, name, B, 1, 40)
            step4 = K.criteo_inputs(B, 40)[0]
            prefix = export_engine_delta(eng, root, base_version=3, version=4)
            for t in (0, 1, 3):
                assert _delta_keys(prefix, t) == set(step4[t].tolist()), t
            K.train(eng, name, B, 1, 41)
            prefix = export_engine_delta(eng, root, base_version=3)
            assert os.path.basename(prefix) == "delta-5"
            assert _delta_keys(prefix, 1) == set(torch.cat([step4[1], K.criteo_inputs(B, 41)[0][1]]).tolist())
            assert all(_wait(lambda p=p: p.model_info()["delta_version"] == 5) for p in procs)
            ref2 = K.oracle(eng, name, dense, ids)
            assert np.abs(ref2 - ref).max() > 1e-4
            assert K.max_err(procs[0].predict(*req), ref2) < CPU_TOL
            assert K.max_err(procs[1].predict(*req), ref2) < TOL
        finally:
            for p in procs:
                p.close()
        # the serving deltas consumed no dirty bits: the incremental checkpoint after them restores the live tables
        eng.save(ck, incremental=True)
        fresh = mk()
        assert fresh.restore(ck) == 5
        for t in range(eng.T):
            a, b = eng.tables[t].snapshot(), fresh.tables[t].snapshot()
            assert torch.equal(a["keys"], b["keys"]) and torch.equal(a["rows"], b["rows"]), t


def test_world_and_interaction_refusals(tmp_path):
    from dlrm_dcn_cases import small_config
    from deeprec_b200.models.dlrm_engine import DLRMEngine
    with _native.cuda_emulation():
        eng = DLRMEngine(small_config(batch_size=64, interaction_op="dot"))
        with pytest.raises(ValueError, match="export_saved_model"):
            export_engine_program(eng, str(tmp_path / "x"))
        eng = K.make_engine("dssm", DEV, B)
        eng.world = 2                                                 # the refusal reads only the world size
        with pytest.raises(ValueError, match="world_size 1"):
            export_engine_program(eng, str(tmp_path / "x"))
        with pytest.raises(ValueError, match="world_size 1"):
            export_engine_delta(eng, str(tmp_path), 0)
    assert not os.path.exists(tmp_path / "x")


# ---- ops against float64 ----------------------------------------------------------------------------------------------------------------
class _NoKeys:
    """A table with no trained rows: hand-made programs only need one."""
    dim = 8

    def default(self):
        return torch.zeros(4, 8)

    def full(self):
        e = torch.zeros(0, dtype=torch.int64)
        return {"keys": e, "rows": torch.zeros(0, 8), "freqs": e, "versions": e}

    def exported(self):
        pass


def _write(p, path, num_dense, C):
    from deeprec_b200.serving.export import _write_program
    p.col_table = [0] * C
    _write_program(p, [_NoKeys()], 8, None, "ops", num_dense, path, 1, None, None)


def _serve(path, dense, ids):
    out = []
    for dev in ("cpu", "cuda_emu"):
        pr = Processor(path, _cfg(max_batch=8), device=dev)
        try:
            out.append(pr.predict(dense, ids).astype(np.float64))
        finally:
            pr.close()
    return out


def cross_linear_case(N, r, rows, seed=0):
    """Program: x0, x_l, t = slices of the dense input, y = cross_linear(x0, x_l, t), 16 logits = y R^T; with the float64 probabilities.
    Inputs are bf16-representable, so the GPU runtime's cast of the dense input is exact."""
    from deeprec_b200.serving.export import _ProgramBuilder
    g = torch.Generator().manual_seed(seed)
    bf = lambda t: t.bfloat16().float()
    dense = bf(torch.randn(rows, 2 * N + r, generator=g))
    Wk, b = bf(torch.randn(N, r, generator=g) / r ** 0.5), torch.randn(N, generator=g)
    R = torch.randn(16, N, generator=g) / N ** 0.5
    p = _ProgramBuilder()
    y = p.cross_linear(p.slice("dense", 0, N), p.slice("dense", N, N), p.slice("dense", 2 * N, r), Wk, b)
    p.out = p.linear(y, R, None)
    p.num_outputs, p.output_names = 16, [str(i) for i in range(16)]
    d = dense.double()
    x0, xl, t = d[:, :N], d[:, N:2 * N], d[:, 2 * N:]
    ref = torch.sigmoid((x0 * (t @ Wk.double().t() + b.double()) + xl) @ R.double().t()).numpy()
    return p, dense.numpy(), ref


@pytest.mark.parametrize("N,r", [(432, 8), (432, 512), (3456, 8), (3456, 512)])
def test_cross_linear_against_float64(tmp_path, N, r):
    p, dense, ref = cross_linear_case(N, r, 11)
    with _native.cuda_emulation():
        _write(p, str(tmp_path / "m"), 2 * N + r, 1)
        cpu, emu = _serve(str(tmp_path / "m"), dense, np.zeros((1, 11), np.int64))
    assert np.abs(cpu - ref).max() < 1e-5, np.abs(cpu - ref).max()
    assert np.abs(emu - ref).max() < TOL, np.abs(emu - ref).max()


@pytest.mark.parametrize("sqrtn", [False, True])
def test_seq_mean_modes_against_float64(tmp_path, sqrtn):
    """seq_mean over the positions whose id is not padding: mode 1 divides by sqrt(count), and a row without a valid position gives 0."""
    from deeprec_b200.serving.export import _ProgramBuilder
    Lq, W, rows = 6, 8, 13
    g = torch.Generator().manual_seed(3)
    dense = torch.randn(rows, Lq * W, generator=g).bfloat16().float()
    ids = torch.randint(0, 5, (Lq, rows), generator=g)
    ids[torch.rand(Lq, rows, generator=g) < 0.4] = -1
    ids[:, 0] = -1                                                   # row 0: no valid position
    p = _ProgramBuilder()
    pooled = p.seq_mean(p.slice("dense", 0, Lq * W), p.valid_mask(0, Lq), Lq, sqrtn=sqrtn)
    R = torch.randn(16, W, generator=g)
    p.out = p.linear(pooled, R, None)
    p.num_outputs, p.output_names = 16, [str(i) for i in range(16)]
    v = (ids >= 0).t().double()
    n = v.sum(1, keepdim=True)
    s = (dense.double().view(rows, Lq, W) * v[..., None]).sum(1)
    pooled_ref = torch.where(n > 0, s / (n.sqrt() if sqrtn else n).clamp_min(1.0), torch.zeros_like(s))
    ref = torch.sigmoid(pooled_ref @ R.double().t()).numpy()
    with _native.cuda_emulation():
        _write(p, str(tmp_path / "m"), Lq * W, Lq)
        cpu, emu = _serve(str(tmp_path / "m"), dense.numpy(), ids.numpy())
    assert np.abs(cpu[0] - 0.5).max() == 0.0 and np.abs(emu[0] - 0.5).max() == 0.0
    assert np.abs(cpu - ref).max() < 1e-5, np.abs(cpu - ref).max()
    assert np.abs(emu - ref).max() < TOL, np.abs(emu - ref).max()


def test_cross_linear_outside_the_gemm_contract_fails_to_load(tmp_path, capfd):
    """x0 = the 12-wide embedding buffer (C = 3, D = 4): the cross GEMM would write 16 columns into a 12-column pitch.  The CPU runtime
    serves it; the GPU runtime refuses the model at load time with a message."""
    from deeprec_b200.serving.export import _ProgramBuilder, _write_program

    class _D4(_NoKeys):
        dim = 4

        def default(self):
            return torch.ones(4, 4)

        def full(self):
            e = torch.zeros(0, dtype=torch.int64)
            return {"keys": e, "rows": torch.zeros(0, 4), "freqs": e, "versions": e}
    p = _ProgramBuilder()
    y = p.cross_linear("emb", "emb", p.slice("dense", 0, 8), torch.randn(12, 8), torch.randn(12))
    p.out = p.linear(y, torch.randn(1, 12), None)
    p.col_table = [0] * 3
    path = str(tmp_path / "m")
    _write_program(p, [_D4()], 4, None, "ops", 8, path, 1, None, None)
    dense, ids = np.ones((2, 8), np.float32), np.zeros((3, 2), np.int64)
    with _native.cuda_emulation():
        cpu = Processor(path, _cfg(), device="cpu")
        try:
            assert np.isfinite(cpu.predict(dense, ids)).all()
        finally:
            cpu.close()
        with pytest.raises(Exception):
            Processor(path, _cfg(), device="cuda_emu")
    assert "cross_linear" in capfd.readouterr().err


def test_zoo_dlrm_dcn_through_the_module_export(tmp_path):
    """The framework-path DLRMDCN (EmbeddingVariable tables) exports through export_saved_model_program and serves."""
    import deeprec_b200 as dr
    from deeprec_b200.data import criteo_batch
    from deeprec_b200.serving import export_saved_model_program
    model = K.build("dlrm_dcn", DEV)
    opt = dr.optim.AdagradOptimizer(model, lr=0.05)
    for s in range(2):
        d, ids, y = criteo_batch(48, 13, K.CARDS, seed=s)
        loss = model.loss(d, ids, y); opt.zero_grad(); loss.backward(); opt.step()
    model.eval()
    with torch.no_grad():
        ref = torch.sigmoid(model(d, ids)).numpy()
    export_saved_model_program(model, str(tmp_path / "v"), version=2)
    assert any(op["op"] == "cross_linear" for op in json.load(open(tmp_path / "v" / "saved_model.json"))["program"])
    with _native.cuda_emulation():
        _serve_both(str(tmp_path / "v"), d.numpy(), ids.numpy(), ref)


# ---- world_size > 1: restore the checkpoint into a world-1 engine, export from that ------------------------------------------------------
def _world2_rank(rank, shared, name, ckpt, out, errors):
    """One of two ranks as threads: train 3 steps on this rank's half of every global batch, save, then predict() this rank's half of the
    request batch (collective)."""
    try:
        import torch.distributed as dist
        from deeprec_b200.parallel.emu_comm import EmuComm
        Bh = B // 2
        with _native.cuda_emulation():
            comm = EmuComm(shared, rank)
            model = None
            if name != "dlrm_dcnv2":
                with shared.lock:                                    # the default RNG and the variable registry are process-global
                    model = K.build(name, DEV)
            eng = _world_engine(name, Bh, rank, 2, comm, model)     # collective: outside the lock
            lo, hi = rank * Bh, (rank + 1) * Bh
            for s in range(3):
                ids, y, dense = K.criteo_inputs(B, 10 + s)
                _load(eng, name, ids[:, lo:hi], y[lo:hi], dense[lo:hi])
                eng.train_step()
            barrier = dist.barrier
            dist.barrier = lambda *a, **k: shared.barrier.wait()     # save_engine's collective barrier, across the rank threads
            try:
                eng.save(ckpt)
            finally:
                dist.barrier = barrier
            ids, y, dense = K.criteo_inputs(B, 77)
            ids[1, :8] += 10 ** 9
            _load(eng, name, ids[:, lo:hi], y[lo:hi], dense[lo:hi])
            p = eng.predict()
            out[rank] = (p.cpu().numpy().copy(), eng.params.clone())
            comm.host_barrier()
    except BaseException as e:                                      # noqa: BLE001
        errors.append((rank, repr(e)))
        try:
            shared.barrier.abort()
        except Exception:
            pass
        raise


def _world_engine(name, Bn, rank=0, world=1, comm=None, model=None):
    from deeprec_b200.models.rec_engine import criteo_engine
    if name == "dlrm_dcnv2":
        from dlrm_dcn_cases import small_config
        from deeprec_b200.models.dlrm_engine import DLRMEngine
        return DLRMEngine(small_config(batch_size=Bn), None, rank, world, comm)
    return criteo_engine(model if model is not None else K.build(name, DEV), Bn, table_rows=K.CARDS, learning_rate=0.05, rank=rank,
                         world_size=world, comm=comm)


def _load(eng, name, ids, y, dense):
    if name == "dlrm_dcnv2":
        eng.load_batch(dense, ids, y)
    else:
        eng.load_batch(ids, y, {"dense": dense})


@pytest.mark.parametrize("name", ["dcn", "dlrm_dcnv2"])
def test_two_rank_checkpoint_restored_at_world1_exports_and_serves(tmp_path, name):
    """Two ranks as threads train and save; a world-1 engine restores the checkpoint (re-sharded N -> 1) and exports; the served
    predictions match the two-rank engine's own predict().  DCN has no BatchNorm, so both ranks' halves compare.  DLRM-DCNv2's bottom
    BatchNorm keeps per-rank moving statistics and the checkpoint carries rank 0's, so rank 0's half compares."""
    from deeprec_b200.parallel.emu_comm import EmuWorld
    with _native.cuda_emulation():
        pass
    ckpt = str(tmp_path / "ck" / "model")
    shared, out, errors = EmuWorld(2), {}, []
    threads = [threading.Thread(target=_world2_rank, args=(r, shared, name, ckpt, out, errors)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=1200)
    assert not errors and len(out) == 2, errors
    assert torch.equal(out[0][1], out[1][1]), "dense replicas diverged"
    ids, _, dense = K.criteo_inputs(B, 77)
    ids[1, :8] += 10 ** 9
    with _native.cuda_emulation():
        one = _world_engine(name, B)
        assert one.restore(ckpt) == 3
        assert torch.equal(one.params, out[0][1])
        root = str(tmp_path / "serve")
        export_engine_program(one, os.path.join(root, "v"), root=root)
        assert json.load(open(os.path.join(root, "v", "saved_model.json")))["version"] == 3
        halves = 2 if name == "dcn" else 1
        want = np.concatenate([out[r][0] for r in range(halves)])
        n = want.shape[0]
        for dev in ("cpu", "cuda_emu"):
            p = Processor(os.path.join(root, "v"), _cfg(), device=dev)
            try:
                got = p.predict(*(a[..., :n] if a.ndim == 2 and a.shape[0] == 26 else a[:n] for a in K.request(name, dense, ids)))
            finally:
                p.close()
            assert K.max_err(got, want) < TOL, (dev, K.max_err(got, want))
