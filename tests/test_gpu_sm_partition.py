"""The DLRM step's SM partition (DLRMConfig.sparse_sms, csrc/cuda/sm_partition.cu): the green contexts it gets, where the captured step's
kernels run, the persistent GEMM grids inside the dense partition, and that the partition changes where kernels run but not one bit of
what they compute."""
import ctypes as C
import json
import os

import pytest
import torch

from deeprec_b200 import _native

pytestmark = pytest.mark.gpu

R = 16


def _cfg(B, sparse_sms, **kw):
    from deeprec_b200.models.dlrm_engine import DLRMConfig
    return DLRMConfig(batch_size=B, cardinalities=[5000] * 26, sparse_sms=sparse_sms, **kw)


def _batches(cfg, n, seed=5):
    from deeprec_b200.data.synthetic import criteo_batch
    return [tuple(t.cuda() for t in criteo_batch(cfg.batch_size, cfg.num_dense, cfg.cardinalities, seed=seed + i, alpha=1.05)) for i in range(n)]


def _partition(sparse_sms):
    lib = _native.cuda()
    info, h = (C.c_int * 2)(), (C.c_void_p * 5)()
    _native.check(lib.dr_cuda_sm_partition(torch.cuda.current_device(), sparse_sms, info, h), "sm_partition")
    return (info[0], info[1]), list(h)


def test_partition_reports_the_sms_it_got():
    total = torch.cuda.get_device_properties(0).multi_processor_count
    for want in (8, 12, 16, 32):
        (sp, dn), h = _partition(want)
        assert sp >= want and sp % 8 == 0 and sp - want < 8, (want, sp)       # Hopper: groups of 8 SMs, rounded up
        assert dn > 0 and sp + dn <= total, (sp, dn, total)
        assert all(h), h
    assert _partition(16) == _partition(16)                                  # created once per (device, count)
    assert _native.cuda().dr_cuda_sm_partition(0, 0, (C.c_int * 2)(), (C.c_void_p * 5)()) != 0


def _run(sparse_sms, graph, batches):
    from deeprec_b200.models.dlrm_engine import DLRMEngine
    eng = DLRMEngine(_cfg(batches[0][0].shape[0], sparse_sms))
    eng.load_batch(*batches[0])
    if graph:
        eng.capture()
    else:
        eng.train_step()
    for b in batches[1:]:
        eng.load_batch(*b)
        eng.train_step()
    torch.cuda.synchronize()
    out = {k: v.cpu() for k, v in eng.state_dict().items()}
    out["prob"], out["loss"] = eng.prob.cpu(), eng.loss.cpu()
    keys = batches[-1][1]
    for t, tb in sorted(eng.tables.items()):
        out[f"rows{t}"] = tb.lookup(keys[t].contiguous()).cpu()
    return out


def test_outputs_bitwise_equal_with_and_without_partition():
    from deeprec_b200.models.dlrm_engine import DLRMConfig
    batches = _batches(_cfg(8192, 0), 4)
    ref = _run(0, False, batches)
    for sparse_sms, graph in ((0, True), (R, False), (R, True), (DLRMConfig.sparse_sms, True)):
        got = _run(sparse_sms, graph, batches)
        assert got.keys() == ref.keys()
        bad = [k for k in ref if not torch.equal(ref[k].view(torch.uint8), got[k].view(torch.uint8))]
        assert not bad, (sparse_sms, graph, bad[:5])


def _graph_contexts(eng):
    """Kernel-node contexts of one captured step."""
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g, stream=torch.cuda.Stream()):
        eng._step_body()
    ctx = (C.c_void_p * 4096)()
    n = _native.cuda().dr_cuda_graph_kernel_contexts(C.c_void_p(g.raw_cuda_graph()), ctx, 4096)
    assert 0 < n <= 4096, n
    return [ctx[i] for i in range(n)]


def test_captured_step_keeps_the_partition():
    from deeprec_b200.models.dlrm_engine import DLRMEngine
    cfg = _cfg(8192, R)
    eng = DLRMEngine(cfg)
    eng.load_batch(*_batches(cfg, 1)[0])
    eng.train_step()
    torch.cuda.synchronize()
    _, h = _partition(R)
    sparse, dense, primary = h[2], h[3], h[4]
    ctxs = _graph_contexts(eng)
    count = {name: sum(c == v for c in ctxs) for name, v in (("sparse", sparse), ("dense", dense), ("primary", primary))}
    assert sum(count.values()) == len(ctxs), (count, len(ctxs))
    # forward: dedup + lookup; backward: segsum, reset, grad, apply + counter reset
    assert count["sparse"] >= 6, count
    # forward: cast, 4 GEMMs, 3 folds, finalize, apply, statistics sums; backward: 4 layers of statistics, BN backward, dW, dX
    assert count["dense"] >= 20, count
    assert count["primary"] >= 10, count                      # interaction, top MLP, head, dense update stay on every SM
    base = DLRMEngine(_cfg(8192, 0))
    base.load_batch(*_batches(cfg, 1)[0])
    base.train_step()
    torch.cuda.synchronize()
    assert set(_graph_contexts(base)) <= {primary, None}


def test_dense_partition_gemm_grid_follows_its_sms(tmp_path):
    from torch.profiler import ProfilerActivity, profile

    from deeprec_b200.models.dlrm_engine import DLRMEngine
    cfg = _cfg(16384, R)
    eng = DLRMEngine(cfg)
    b = _batches(cfg, 2)
    eng.load_batch(*b[0]); eng.train_step()
    torch.cuda.synchronize()
    dense_sms = eng.partition_sms[1]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.load_batch(*b[1]); eng.train_step()
        torch.cuda.synchronize()
    path = os.path.join(tmp_path, "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as fh:
        ev = sorted((e for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel" and "k_gemm_tn" in e.get("name", "")), key=lambda e: e["ts"])
    grids = [e["args"]["grid"][0] for e in ev]
    assert len(grids) == 11, grids
    # call order: bot0..3 fwd (dense partition), top0/top1 fwd, top1/top0 dX (all SMs), bot3..bot1 dX (dense partition).  B = 16384 gives
    # every call but the N <= 64 ones more tiles than SMs, so those grids equal the SMs they may use
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert grids[0] == dense_sms and grids[1] == dense_sms and grids[10] == dense_sms, (grids, dense_sms)
    assert grids[4] == sms and grids[6] == sms, (grids, sms)
    assert max(grids[i] for i in (0, 1, 2, 3, 8, 9, 10)) <= dense_sms
