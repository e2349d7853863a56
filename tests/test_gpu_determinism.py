"""The DLRM training step is deterministic: every sum over the batch goes through per-block workspaces added in block order (k_det_colsum,
csrc/cuda/common.cuh) or, for the per-key embedding gradients, through 64-bit fixed point (k_sp_segsum, csrc/cuda/sparse_pipeline.cu).
Checked bit for bit (torch.equal): each such reduction run twice on the same inputs, with a larger call on the same workspace slot in
between so that dr_workspace has to grow; and the whole engine trained twice from the same seed, eagerly and graph-captured, in one process
and in two child processes (different allocation addresses).

Not covered: the owner-side fp32 sum of the per-key gradients over ranks in multi-GPU training (k_sp_grad with world > 1) is documented
as not deterministic, and the generic (non-DLRM) engines still use fp32 atomics."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _lib():
    from deeprec_b200 import _native
    return _native.cuda()


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _twice_with_growth(run, small, large):
    """run(shape) -> tuple of result tensors.  small, then large (grows the workspace), then small again: bitwise equal."""
    r1 = [t.clone() for t in run(*small)]
    run(*large)
    r2 = [t.clone() for t in run(*small)]
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(r1, r2)):
        assert torch.equal(a, b), (small, i, (a.float() - b.float()).abs().max().item())
    return r1


def test_gemm_tn_ex_statistics_bitwise():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(0)
    A0 = torch.randn(20000, 256, device="cuda", generator=g).bfloat16()
    B0 = (torch.randn(512, 256, device="cuda", generator=g) * 0.1).bfloat16()
    bias = torch.randn(512, device="cuda", generator=g) * 0.1
    aux = torch.randn(20000, 512, device="cuda", generator=g).relu().bfloat16()

    def run(M, N, K, mode):
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        S1 = torch.zeros(N, device="cuda"); S2 = torch.zeros(N, device="cuda")
        if mode == 2:
            rc = lib.dr_cuda_gemm_tn_ex(_p(A0), 256, _p(B0), 256, M, N, K, None, 0, _p(aux), 512, 2, _p(out), N, None, _p(S1), _p(S2), 0, 0, _s())
        else:
            rc = lib.dr_cuda_gemm_tn_ex(_p(A0), 256, _p(B0), 256, M, N, K, _p(bias), 1, None, 0, 0, _p(out), N, None, _p(S1), _p(S2), 0, 0, _s())
        assert rc == 0
        return out, S1, S2

    for mode in (0, 2):
        _twice_with_growth(run, (4096, 256, 256, mode), (20000, 512, 256, mode))


def test_gemm_dw_bitwise():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(1)
    dY = (torch.randn(30000, 512, device="cuda", generator=g) * 0.1).bfloat16()
    X = torch.randn(30000, 368, device="cuda", generator=g).bfloat16()

    def run(batch, n_out, k_in, splits):
        dW = torch.full((n_out, k_in), 0.5, device="cuda")
        assert lib.dr_cuda_gemm_dw(_p(dY), 512, _p(X), 368, batch, n_out, k_in, _p(dW), k_in, splits, _s()) == 0
        return (dW,)

    for splits in (0, 3):
        _twice_with_growth(run, (4096, 256, 72, splits), (30000, 512, 368, splits))


def test_colstats_bitwise():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(2)
    a = torch.randn(70000, 512, device="cuda", generator=g).bfloat16()
    b = torch.randn(70000, 512, device="cuda", generator=g).relu().bfloat16()

    def run(Bn, N):
        S1 = torch.zeros(N, device="cuda"); S2 = torch.zeros(N, device="cuda")
        assert lib.dr_cuda_colstats(_p(a), _p(b), Bn, N, 512, 512, _p(S1), _p(S2), _s()) == 0
        return S1, S2

    S1, S2 = _twice_with_growth(run, (3000, 256), (70000, 512))
    ref1 = a[:3000, :256].double().sum(0)
    assert ((S1.double() - ref1).abs() <= 3000 * U * a[:3000, :256].double().abs().sum(0) + 1e-30).all()


def test_head_bitwise():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(3)
    Kmax, Bmax = 512, 70000
    h = torch.randn(Bmax, Kmax, device="cuda", generator=g).relu().bfloat16()
    w = torch.randn(Kmax, device="cuda", generator=g) * 0.05
    bb = torch.tensor([0.1, 0, 0, 0], device="cuda")
    y = (torch.rand(Bmax, device="cuda", generator=g) < 0.3).float()

    def run(Bn, K):
        prob = torch.empty(Bn, device="cuda"); loss = torch.zeros(1, device="cuda")
        dh = torch.empty(Bn, Kmax, device="cuda", dtype=torch.bfloat16)          # dh shares h's row pitch
        dw = torch.zeros(K, device="cuda"); db = torch.zeros(4, device="cuda"); dbh = torch.zeros(K, device="cuda")
        assert lib.dr_cuda_head(_p(h), Kmax, Bn, K, _p(w), _p(bb), _p(y), 1.0 / Bn, _p(prob), _p(loss), _p(dh), _p(dw), _p(db), 1, 1, _p(dbh), _s()) == 0
        return loss, dw, db, dbh, prob, dh[:, :K]

    _twice_with_growth(run, (3000, 256), (70000, 512))


def test_bn_bwd_apply_v2_dbias_bitwise():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(4)
    Bmax, Kmax = 70000, 512
    a = torch.randn(Bmax, Kmax, device="cuda", generator=g).relu().bfloat16()
    dy = (torch.randn(Bmax, Kmax, device="cuda", generator=g) * 0.1).bfloat16()
    scale = torch.rand(Kmax, device="cuda", generator=g) + 0.5
    mean = torch.rand(Kmax, device="cuda", generator=g); rstd = torch.rand(Kmax, device="cuda", generator=g) + 0.5
    c1 = torch.randn(Kmax, device="cuda", generator=g) * 0.01; c2 = torch.randn(Kmax, device="cuda", generator=g) * 0.01

    def run(Bn, K):
        out = torch.empty(Bn, Kmax, device="cuda", dtype=torch.bfloat16); dbias = torch.zeros(K, device="cuda")     # da shares the row pitch
        assert lib.dr_cuda_bn_bwd_apply_v2(_p(dy), _p(a), Bn, K, Kmax, _p(scale), _p(mean), _p(rstd), _p(c1), _p(c2), _p(out), 1, _p(dbias), _s()) == 0
        return out[:, :K], dbias

    _twice_with_growth(run, (3000, 256), (70000, 512))


# ---------------------------------------------------------------------------------------------------------------------------------------
# k_sp_segsum: bitwise across runs, and against an fp64 segment sum

def _segsum_setup(B, cards, D, seed):
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(seed)
    C_ = len(cards)
    sp = SparsePipeline(dev, 0, 1, list(range(C_)), C_, B, D)
    ids = torch.stack([torch.randint(0, c, (B,), generator=g) for c in cards])
    ids[0, :] = 12345                                              # one key in every sample
    mag = 10.0 ** (torch.rand(C_, B, D, generator=g) * 10 - 8)    # |g| from 1e-8 to 1e2
    sign = torch.where(torch.rand(C_, B, D, generator=g) < 0.5, -1.0, 1.0)
    grad = (mag * sign).bfloat16()
    return sp, ids.to(dev), grad.to(dev)


def _segsum_once(sp, ids, grad):
    sp.dedup(ids)
    sp.segsum(grad)
    torch.cuda.synchronize()
    inv = sp.inv[:, : ids.shape[0]].t().long().clone()
    raw = sp.ugrad.clone()
    rows = sp.ugrad_rows()
    sp.reset(); sp.step_end()
    torch.cuda.synchronize()
    return inv, raw, rows


def test_segsum_bitwise_and_fp64_accuracy():
    B, D = 4096, 16
    cards = [1, 50, 3000, 100000]
    sp, ids, grad = _segsum_setup(B, cards, D, seed=5)
    inv1, raw1, rows = _segsum_once(sp, ids, grad)
    inv2, raw2, _ = _segsum_once(sp, ids, grad)
    # a key's scratch slot is claimed by atomics (linear probing), so compare the sums by sample, i.e. by key
    assert torch.equal(raw1[inv1.reshape(-1)], raw2[inv2.reshape(-1)]), "k_sp_segsum must give the same fixed-point sums on every run"
    touched = torch.unique(inv1.reshape(-1))
    # fp64 reference and the bound: every (column, 32-row tile, key) group is one fp32 partial of n bf16 rows (n 2^-24 of its absolute
    # sum), rounded once to the fixed-point grid (2^-41); ugrad_rows rounds the exact integer sum to fp32 (2^-24 relative).
    Cn = ids.shape[0]
    g64 = grad.double().reshape(Cn * B, D)
    gs = inv1.reshape(-1)
    ref = torch.zeros(sp.Htot, D, dtype=torch.float64, device=ids.device).index_add_(0, gs, g64)
    tile = (torch.arange(Cn, device=ids.device).unsqueeze(1) * ((B + 31) // 32) + torch.arange(B, device=ids.device).unsqueeze(0) // 32).reshape(-1)
    grp, ginv = torch.unique(tile * sp.Htot + gs, return_inverse=True)
    gabs = torch.zeros(grp.numel(), D, dtype=torch.float64, device=ids.device).index_add_(0, ginv, g64.abs())
    gcnt = torch.zeros(grp.numel(), dtype=torch.float64, device=ids.device).index_add_(0, ginv, torch.ones_like(ginv, dtype=torch.float64))
    gkey = grp % sp.Htot
    bound = torch.zeros(sp.Htot, D, dtype=torch.float64, device=ids.device).index_add_(0, gkey, gcnt.unsqueeze(1) * U * gabs + 2.0 ** -41)
    bound += U * ref.abs()
    err = (rows.double() - ref)[touched].abs()
    assert (err <= bound[touched]).all(), (err - bound[touched]).max().item()
    hot = inv1[0, 0]
    assert (inv1[0] == hot).all() and (ref[hot].abs() > 1).any()


def test_segsum_fixed_point_range():
    """Inside the documented range (|sum| < 2^22) the fixed-point sum is exact for bf16 inputs; a partial beyond it saturates at 2^22
    instead of wrapping through an out-of-range conversion."""
    B, D = 64, 16
    sp, ids, _ = _segsum_setup(B, [1], D, seed=6)
    grad = torch.zeros(1, B, D, device="cuda")
    grad[0, :, 0] = 2.0 ** 15                 # 64 x 2^15 = 2^21: in range, exact
    grad[0, :, 1] = -(2.0 ** 17)              # 32-row partials of -2^22 each: at the limit
    grad[0, :32, 2] = 2.0 ** 18               # one 32-row partial of 2^23: beyond the limit, saturates at 2^22
    grad[0, :, 3] = 2.0 ** -30                # far below a bf16 gradient's resolution of interest, still counted
    inv, raw, rows = _segsum_once(sp, ids, grad.bfloat16())
    k = inv[0, 0]
    assert rows[k, 0].item() == 2.0 ** 21
    assert rows[k, 1].item() == -(2.0 ** 23)
    assert rows[k, 2].item() == 2.0 ** 22
    assert raw[k, 3].item() == 64 * 2 ** 10
    assert (rows[k, 4:] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------------------------
# the whole engine

CARDS = [50, 1000, 7, 300, 100000, 20000] + [97] * 20


def _train(graph, steps=6, batch=2048):
    from deeprec_b200.data.synthetic import criteo_batch
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    eng = DLRMEngine(DLRMConfig(batch_size=batch, cardinalities=CARDS, learning_rate=0.05))
    losses, seen = [], [set() for _ in CARDS]
    for st in range(steps):
        d, ids, y = criteo_batch(batch, 13, CARDS, seed=100 + st)          # default power-law ids: hot keys in every batch
        eng.load_batch(d.cuda(), ids.cuda(), y.cuda())
        if graph and st == 0:
            eng.capture()                                                  # step 0 runs eagerly while the graph is captured
        else:
            eng.train_step()
        losses.append(eng.loss_value())
        for t in range(len(CARDS)):
            seen[t].update(ids[t].tolist())
    torch.cuda.synchronize()
    emb = {}
    for t in range(len(CARDS)):
        keys = torch.tensor(sorted(seen[t]), dtype=torch.int64, device="cuda")
        emb[t] = eng.tables[t].lookup(keys)
    return losses, eng.prob.clone(), eng.state_dict(), emb


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_dlrm_engine_bitwise_across_runs(graph):
    la, pa, sa, ea = _train(graph)
    lb, pb, sb, eb = _train(graph)
    assert la == lb, (la, lb)
    assert torch.equal(pa, pb)
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    for t in ea:
        assert torch.equal(ea[t], eb[t]), f"embedding rows of table {t}"


_CHILD = r'''
import sys, torch
sys.path.insert(0, sys.argv[2])
import bench, test_gpu_determinism as T
from deeprec_b200.data.synthetic import criteo_batch
pad = torch.empty(int(sys.argv[3]) * 1024 * 1024, dtype=torch.uint8, device="cuda")    # shifts every later allocation
from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
eng = DLRMEngine(DLRMConfig(batch_size=2048, cardinalities=T.CARDS, learning_rate=0.05))
for st in range(6):
    d, ids, y = criteo_batch(2048, 13, T.CARDS, seed=100 + st)
    eng.load_batch(d.cuda(), ids.cuda(), y.cuda())
    eng.capture() if st == 0 else eng.train_step()
torch.cuda.synchronize()
bench.dump_outputs(eng, sys.argv[1], ids.cuda())
print("ALL_OK")
'''


def test_dlrm_engine_bitwise_across_processes(tmp_path):
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    dirs = []
    for i, pad_mb in enumerate((0, 37)):
        d = str(tmp_path / f"run{i}")
        r = subprocess.run([sys.executable, "-c", _CHILD, d, here, str(pad_mb)], cwd=root, env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0 and "ALL_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
        dirs.append(d)
    names = sorted(os.listdir(dirs[0]))
    assert names == sorted(os.listdir(dirs[1])) and any(n.startswith("emb_rows") for n in names) and "prob.npy" in names
    for n in names:
        a, b = np.load(os.path.join(dirs[0], n)), np.load(os.path.join(dirs[1], n))
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), n
