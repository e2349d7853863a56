"""DLRM-DCNv2 on DLRMEngine on the GPU: the cross / residual epilogues of the wgmma GEMM (dr_cuda_gemm_tn_cross) and the cross backward
kernel against float64, k_sp_segsum at dim 128, the whole step against the fp32 DLRM(interaction_op="dcnv2") oracle at D = 16 and 128,
bitwise determinism (two runs, eager against graph replay), two GPUs against one, and the train CLI."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

from dlrm_dcn_cases import batch, bn_stats, oracle_from_engine, param_pairs, rel_err, small_config

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from deeprec_b200 import _native
    return _native.cuda()


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _cross(A, Bw, bias, kind, x0, xl, out, u, M, N, K, lda=None, ldb=None, ld_x0=None, ld_xl=None, ldc=None, ld_u=None):
    lib = _lib()
    rc = lib.dr_cuda_gemm_tn_cross(_vp(A), lda or A.stride(0), _vp(Bw), ldb or Bw.stride(0), M, N, K, _vp(bias), kind, _vp(x0),
                                   ld_x0 or (x0.stride(0) if x0 is not None else 0), _vp(xl), ld_xl or xl.stride(0), _vp(out), ldc or out.stride(0),
                                   _vp(u), ld_u or (u.stride(0) if u is not None else 0), 0, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("kind", [1, 2])
@pytest.mark.parametrize("K", [32, 512, 3456])
@pytest.mark.parametrize("N", [8, 136, 432, 3456])
@pytest.mark.parametrize("M", [1, 127, 129, 4099])
def test_cross_epilogues_against_fp64(M, N, K, kind):
    """out (and u) against float64 from the same bf16 operands; every operand pitched 8 columns wider than it is used, outputs prefilled with
    NaN: the rows < M, columns < N are finite and right, the pad columns stay NaN."""
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K + kind)
    P = 8
    bf = torch.bfloat16
    A = (torch.randn(M, K + P, device="cuda", generator=g) / K ** 0.5).to(bf)
    Bw = torch.randn(N, K + P, device="cuda", generator=g).to(bf)
    bias = torch.randn(N, device="cuda", generator=g)
    x0 = torch.randn(M, N + P, device="cuda", generator=g).to(bf)
    xl = torch.randn(M, N + P, device="cuda", generator=g).to(bf)
    out = torch.full((M, N + P), float("nan"), device="cuda", dtype=bf)
    u = torch.full((M, N + P), float("nan"), device="cuda", dtype=bf) if kind == 1 else None
    assert _cross(A, Bw, bias if kind == 1 else None, kind, x0 if kind == 1 else None, xl, out, u, M, N, K) == 0
    acc = A[:, :K].double() @ Bw[:, :K].double().T
    if kind == 1:
        uref = acc + bias.double()
        ref = x0[:, :N].double() * uref + xl[:, :N].double()
        # u: fp32 accumulation (relative ~K 2^-24) then one bf16 rounding (2^-9 relative)
        assert ((u[:, :N].double() - uref).abs() <= uref.abs() * 2 ** -8 + 1e-3).all()
        assert torch.isnan(u[:, N:]).all()
    else:
        ref = acc + xl[:, :N].double()
    got = out[:, :N].double()
    assert torch.isfinite(got).all()
    # the epilogue runs in fp32 from the fp32 accumulator; the output is rounded once to bf16
    assert ((got - ref).abs() <= ref.abs() * 2 ** -8 + 1e-3 * (1 + x0[:, :N].double().abs())).all(), (got - ref).abs().max().item()
    assert torch.isnan(out[:, N:]).all()


def test_cross_epilogue_operand_contract():
    """Unaligned or short-pitched new operands: the documented error, nothing written."""
    M, N, K = 64, 128, 64
    bf = torch.bfloat16
    A = torch.randn(M, K, device="cuda").to(bf); Bw = torch.randn(N, K, device="cuda").to(bf)
    x0 = torch.randn(M, N + 8, device="cuda").to(bf); xl = torch.randn(M, N + 8, device="cuda").to(bf)
    out = torch.full((M, N), float("nan"), device="cuda", dtype=bf)
    assert _cross(A, Bw, None, 1, x0, xl[:, 1:], out, None, M, N, K, ld_xl=N + 8) == -3      # xl not 16-byte aligned
    assert _cross(A, Bw, None, 1, x0[:, 4:], xl, out, None, M, N, K, ld_x0=N + 8) == -3      # x0 not 16-byte aligned
    assert _cross(A, Bw, None, 2, None, xl, out, None, M, N, K, ld_xl=N + 4) == -2            # pitch not a multiple of 8
    assert _cross(A, Bw, None, 1, x0, xl, out, None, M, N, K, ld_x0=N - 8) == -5              # pitch shorter than N
    assert _cross(A, Bw, None, 1, None, xl, out, None, M, N, K) == -4                         # cross without x0
    assert _cross(A, Bw, None, 3, x0, xl, out, None, M, N, K) == -4                           # unknown kind
    assert torch.isnan(out).all()


@pytest.mark.parametrize("N", [432, 3456])
def test_cross_backward_kernel_against_fp64(N):
    B = 1000
    bf = torch.bfloat16
    gen = torch.Generator(device="cuda").manual_seed(N)
    gr, x0, u = (torch.randn(B, N, device="cuda", generator=gen).to(bf) for _ in range(3))
    gr2 = torch.randn(B, N, device="cuda", generator=gen).to(bf)
    du = torch.full((B, N), float("nan"), device="cuda", dtype=bf)
    dx0 = torch.full((B, N), float("nan"), device="cuda")
    db = torch.full((N,), 0.5, device="cuda")
    lib = _lib()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for i, g in enumerate((gr, gr2)):
        assert lib.dr_cuda_cross_bwd(_vp(g), N, _vp(x0), N, _vp(u), N, B, N, _vp(du), N, _vp(dx0), N, int(i == 0), _vp(db), s) == 0
    torch.cuda.synchronize()
    du_ref = gr2.double() * x0.double()
    assert ((du.double() - du_ref).abs() <= du_ref.abs() * 2 ** -8).all()
    dx0_ref = gr.double() * u.double() + gr2.double() * u.double()         # init on the first call (NaN overwritten), += on the second
    assert ((dx0.double() - dx0_ref).abs() <= 1e-5 * (1 + dx0_ref.abs())).all()
    db_ref = 0.5 + (gr.double() * x0.double()).sum(0) + du_ref.sum(0)
    scale = (gr.double() * x0.double()).abs().sum(0) + du_ref.abs().sum(0)
    assert ((db.double() - db_ref).abs() <= 1e-5 * (1 + scale)).all()


def test_segsum_dim128_against_fp64():
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
    B, Cn, dim = 4096, 4, 128
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 300, (Cn, B), generator=g)
    ids[2, ::5] = -1
    demb = (torch.randn(Cn, B, dim, generator=g) * 0.5).bfloat16()
    sp = SparsePipeline(torch.device("cuda"), 0, 1, list(range(Cn)), Cn, B, dim)
    sp.dedup(ids.cuda())
    sp.segsum(demb.cuda())
    torch.cuda.synchronize()
    got = sp.ugrad.cpu().double() / float(1 << 40)
    invT = sp.invT.cpu()
    for c in range(Cn):
        live = invT[c] >= 0
        ref = torch.zeros(int(invT[c][live].max()) + 1, dim, dtype=torch.float64).index_add_(0, invT[c][live].long(), demb[c][live].double())
        used = torch.unique(invT[c][live]).long()
        assert ((got[used] - ref[used]).abs() <= 1e-5 * (1 + ref[used].abs())).all(), c


@pytest.mark.parametrize("D", [16, 128])
def test_dcnv2_step_matches_the_fp32_oracle(D):
    from deeprec_b200.models.dlrm_engine import DLRMEngine
    torch.manual_seed(0)
    cfg = small_config(embedding_dim=D, mlp_bot=(32, D), batch_size=1024)
    eng = DLRMEngine(cfg)
    m = oracle_from_engine(eng, "cuda")
    o_dense = torch.optim.Adagrad([p for n, p in m.named_parameters() if not n.startswith("tables")], lr=0.05, initial_accumulator_value=0.1, eps=0.0)
    o_emb = torch.optim.Adagrad(m.tables.parameters(), lr=0.05, initial_accumulator_value=0.1, eps=0.0)
    for s in range(3):
        dense, ids, labels = (t.cuda() for t in batch(cfg.batch_size, 10 + s))
        eng.load_batch(dense, ids, labels)
        if s == 0:
            eng.capture()
        else:
            eng.train_step()
        logits = m(dense, ids)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logits, labels)
        o_dense.zero_grad(); o_emb.zero_grad(); loss.backward()
        # bounds and their reasons: tests/test_cuda_emu_dlrm_dcn_engine.py
        assert abs(eng.loss_value() - loss.item()) < 5e-3
        assert (eng.prob - torch.sigmoid(logits)).abs().max().item() < 1e-2
        if s == 0:
            for name, e, o in param_pairs(eng, m, grads=True):
                bound = 0.2 if name.startswith("low_rank_cross_net") else 0.02 if name.startswith("logits") else 0.35
                assert rel_err(e, o.grad) < bound, (name, rel_err(e, o.grad))
        o_dense.step(); o_emb.step()
    for name, e, o in param_pairs(eng, m):
        assert (e - o).abs().max().item() < 2e-3, name
    for rm_e, rm_o, rv_e, rv_o in bn_stats(eng, m):
        assert (rm_e - rm_o).abs().max().item() < 1e-3 and (rv_e - rv_o).abs().max().item() < 1e-3
    keys = ids[1][:64]
    assert (eng.tables[1].lookup(keys) - m.tables[1].weight[keys]).abs().max().item() < 1e-3


def _run(graph, steps=4, D=128):
    from deeprec_b200.models.dlrm_engine import DLRMEngine
    eng = DLRMEngine(small_config(embedding_dim=D, mlp_bot=(32, D), batch_size=2048, dcn_low_rank_dim=64, dcn_num_layers=3))
    losses = []
    for s in range(steps):
        eng.load_batch(*(t.cuda() for t in batch(2048, 40 + s)))
        if graph and s == 0:
            eng.capture()
        else:
            eng.train_step()
        losses.append(eng.loss_value())
    torch.cuda.synchronize()
    rows = eng.tables[1].lookup(torch.arange(1000, device="cuda"))
    return losses, eng.params.clone(), rows, eng.launches_per_step


def test_dcnv2_step_is_bitwise_deterministic():
    a, b, c = _run(False), _run(False), _run(True)
    for x in (b, c):
        assert x[0] == a[0] and torch.equal(x[1], a[1]) and torch.equal(x[2], a[2])
    assert c[3] == a[3] > 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_dcnv2_two_gpus_match_one():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29541",
           os.path.join(ROOT, "tests", "mp_dlrm_dcn.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "MP_DCN_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_train_cli_dcnv2_smoke():
    cmd = [sys.executable, "-m", "deeprec_b200.models.train", "--model", "dlrm", "--engine", "--interaction_op", "dcnv2", "--steps", "5",
           "--batch_size", "1024", "--log_every", "2"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "samples/s" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    losses = [float(l.split()[-1]) for l in r.stdout.splitlines() if l.startswith("global_step")]
    assert losses and all(x == x for x in losses)
