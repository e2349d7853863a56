"""GPU numerics: every hand-written sm_90a kernel against a plain PyTorch fp32 reference of the same op."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from deeprec_b200 import _native
    return _native.cuda()


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


@pytest.mark.parametrize("M,N,K,relu,use_bias", [
    (4096, 512, 16, True, True), (4096, 256, 512, True, True), (4096, 64, 256, True, True), (4096, 16, 64, True, True),
    (4096, 512, 368, True, True), (1000, 256, 512, False, True), (300, 128, 64, False, False), (8192, 32, 128, True, True),
    (65536, 512, 368, True, True),
])
def test_gemm_tn(M, N, K, relu, use_bias):
    torch.manual_seed(0)
    lib = _lib()
    A = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    B = (torch.randn(N, K, device="cuda") * 0.1).bfloat16()
    bias = torch.randn(N, device="cuda") if use_bias else None
    out = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
    rc = lib.dr_cuda_gemm_tn(_p(A), K, _p(B), K, M, N, K, _p(bias), int(relu), None, 0, _p(out), N, None, 0, _s())
    assert rc == 0
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t()
    if use_bias:
        ref = ref + bias
    if relu:
        ref = ref.relu()
    err = (out.float() - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-6
    assert err / scale < 2e-2, f"max err {err} (scale {scale})"


def test_gemm_tn_mask_and_f32_out():
    torch.manual_seed(1)
    lib = _lib()
    M, N, K = 2048, 256, 128
    A = torch.randn(M, K, device="cuda").bfloat16()
    B = (torch.randn(N, K, device="cuda") * 0.1).bfloat16()
    act = torch.randn(M, N, device="cuda").relu().bfloat16()
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    out32 = torch.empty(M, N, device="cuda", dtype=torch.float32)
    assert lib.dr_cuda_gemm_tn(_p(A), K, _p(B), K, M, N, K, None, 0, _p(act), N, _p(out), N, _p(out32), 0, _s()) == 0
    torch.cuda.synchronize()
    ref = (A.float() @ B.float().t()) * (act.float() > 0)
    assert (out32 - ref).abs().max().item() < 1e-2 * (ref.abs().max().item() + 1)
    assert (out.float() - ref).abs().max().item() < 3e-2 * (ref.abs().max().item() + 1)


@pytest.mark.parametrize("batch,N_out,K_in", [
    (4096, 512, 16), (4096, 256, 512), (8192, 64, 256), (4096, 16, 64), (4096, 512, 368), (5000, 256, 512), (65536, 512, 368),
])
def test_gemm_dw(batch, N_out, K_in):
    torch.manual_seed(2)
    lib = _lib()
    dY = (torch.randn(batch, N_out, device="cuda") * 0.1).bfloat16()
    X = (torch.randn(batch, K_in, device="cuda") * 0.5).bfloat16()
    dW = torch.zeros(N_out, K_in, device="cuda")
    assert lib.dr_cuda_gemm_dw(_p(dY), N_out, _p(X), K_in, batch, N_out, K_in, _p(dW), K_in, 0, _s()) == 0
    torch.cuda.synchronize()
    ref = dY.float().t() @ X.float()
    err = (dW - ref).abs().max().item()
    assert err < 1e-2 * (ref.abs().max().item() + 1e-3), f"err {err} ref {ref.abs().max().item()}"


def test_colstats_bn_forward_backward():
    torch.manual_seed(3)
    lib = _lib()
    B, N = 4096, 256
    a = torch.randn(B, N, device="cuda").relu().bfloat16()
    gamma = torch.rand(N, device="cuda") + 0.5
    beta = torch.randn(N, device="cuda") * 0.1
    S1 = torch.zeros(N, device="cuda"); S2 = torch.zeros(N, device="cuda")
    mean, rstd, scale, shift, c1, c2 = (torch.zeros(N, device="cuda") for _ in range(6))
    rm, rv = torch.zeros(N, device="cuda"), torch.ones(N, device="cuda")
    y = torch.empty_like(a)
    assert lib.dr_cuda_colstats(_p(a), _p(a), B, N, N, N, _p(S1), _p(S2), _s()) == 0
    assert lib.dr_cuda_bn_finalize(_p(S1), _p(S2), N, B, _p(gamma), _p(beta), 1e-3, 0.99, _p(rm), _p(rv), _p(mean), _p(rstd), _p(scale), _p(shift), 1, _s()) == 0
    assert lib.dr_cuda_bn_apply(_p(a), B, N, N, _p(scale), _p(shift), _p(y), N, _s()) == 0
    af = a.float().requires_grad_(True)
    ref = torch.nn.functional.batch_norm(af, None, None, gamma, beta, True, 0.0, 1e-3)
    torch.cuda.synchronize()
    assert (y.float() - ref).abs().max().item() < 5e-2
    assert S1.abs().max().item() == 0.0          # finalize re-zeroes the sums
    # backward
    dy = (torch.randn(B, N, device="cuda") * 0.1).bfloat16()
    dgamma, dbeta = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    da = torch.empty_like(a)
    assert lib.dr_cuda_colstats(_p(dy), _p(a), B, N, N, N, _p(S1), _p(S2), _s()) == 0
    assert lib.dr_cuda_bn_bwd_finalize(_p(S1), _p(S2), N, B, _p(mean), _p(rstd), _p(dgamma), _p(dbeta), _p(c1), _p(c2), 1.0, _s()) == 0
    assert lib.dr_cuda_bn_bwd_apply(_p(dy), _p(a), B, N, N, _p(scale), _p(mean), _p(rstd), _p(c1), _p(c2), _p(da), 0, _s()) == 0
    ref.backward(dy.float())
    torch.cuda.synchronize()
    assert (da.float() - af.grad).abs().max().item() < 2e-2
    assert (dbeta - dy.float().sum(0)).abs().max().item() < 5e-2
    xhat = (a.float() - mean) * rstd
    assert (dgamma - (dy.float() * xhat).sum(0)).abs().max().item() < 0.3


def test_head():
    torch.manual_seed(4)
    lib = _lib()
    B, K = 3000, 256
    h = torch.randn(B, K, device="cuda").relu().bfloat16()
    w = torch.randn(K, device="cuda") * 0.05
    b = torch.tensor([0.1, 0, 0, 0], device="cuda")
    y = (torch.rand(B, device="cuda") < 0.3).float()
    prob = torch.empty(B, device="cuda"); loss = torch.zeros(1, device="cuda")
    dh = torch.empty_like(h); dw = torch.zeros(K, device="cuda"); db = torch.zeros(4, device="cuda"); dbh = torch.zeros(K, device="cuda")
    assert lib.dr_cuda_head(_p(h), K, B, K, _p(w), _p(b), _p(y), 1.0 / B, _p(prob), _p(loss), _p(dh), _p(dw), _p(db), 1, 1, _p(dbh), _s()) == 0
    hf = h.float().requires_grad_(True); wf = w.clone().requires_grad_(True); bf = b[:1].clone().requires_grad_(True)
    z = hf @ wf + bf
    ref_loss = torch.nn.functional.binary_cross_entropy_with_logits(z, y)
    ref_loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - ref_loss.item()) < 1e-3
    assert (prob - torch.sigmoid(z)).abs().max().item() < 1e-4
    assert (dw - wf.grad).abs().max().item() < 1e-3
    assert abs(db[0].item() - bf.grad.item()) < 1e-4
    ref_dh = hf.grad * (h.float() > 0)
    assert (dh.float() - ref_dh).abs().max().item() < 1e-5 + 2e-2 * ref_dh.abs().max().item()
    assert (dbh - dh.float().sum(0)).abs().max().item() < 1e-4


def test_dot_interaction():
    from deeprec_b200.models.dlrm import dot_interaction
    torch.manual_seed(5)
    lib = _lib()
    B, T, D = 1537, 26, 16
    x = torch.randn(B, D, device="cuda").bfloat16()
    emb = (torch.randn(T, B, D, device="cuda") * 0.5).bfloat16()
    Zp = (D + (T + 1) * T // 2 + 7) // 8 * 8
    Z = torch.full((B, Zp), 3.0, device="cuda", dtype=torch.bfloat16)
    assert lib.dr_cuda_dot_interaction_fwd(_p(x), D, _p(emb), B * D, D, T, D, B, _p(Z), Zp, _s()) == 0
    xf = x.float().requires_grad_(True); ef = emb.float().permute(1, 0, 2).contiguous().requires_grad_(True)
    ref = dot_interaction(xf, ef)
    torch.cuda.synchronize()
    n = ref.shape[1]
    assert (Z[:, :n].float() - ref).abs().max().item() < 2e-2 * (ref.abs().max().item() + 1)
    assert Z[:, n:].abs().max().item() == 0
    dZ = torch.zeros(B, Zp, device="cuda", dtype=torch.bfloat16)
    dZ[:, :n] = (torch.randn(B, n, device="cuda") * 0.1).bfloat16()
    dx = torch.empty(B, D, device="cuda", dtype=torch.bfloat16); demb = torch.empty(T, B, D, device="cuda", dtype=torch.bfloat16)
    assert lib.dr_cuda_dot_interaction_bwd(_p(dZ), Zp, _p(x), D, _p(emb), B * D, D, T, D, B, _p(dx), D, _p(demb), B * D, D, _s()) == 0
    ref.backward(dZ[:, :n].float())
    torch.cuda.synchronize()
    assert (dx.float() - xf.grad).abs().max().item() < 3e-2 * (xf.grad.abs().max().item() + 1e-3)
    assert (demb.float().permute(1, 0, 2) - ef.grad).abs().max().item() < 3e-2 * (ef.grad.abs().max().item() + 1e-3)


def test_fm_kernels():
    torch.manual_seed(6)
    lib = _lib()
    B, T, D = 1000, 10, 16
    emb = (torch.randn(T, B, D, device="cuda") * 0.5).bfloat16()
    out = torch.empty(B, D, device="cuda", dtype=torch.bfloat16)
    ssum = torch.empty(B, D, device="cuda")
    assert lib.dr_cuda_fm_fwd(_p(emb), B * D, D, T, D, B, _p(out), D, _p(ssum), _s()) == 0
    ef = emb.float().requires_grad_(True)
    ref = 0.5 * (ef.sum(0) ** 2 - (ef ** 2).sum(0))
    torch.cuda.synchronize()
    assert (out.float() - ref).abs().max().item() < 3e-2 * (ref.abs().max().item() + 1)
    dfm = (torch.randn(B, D, device="cuda") * 0.1).bfloat16()
    demb = torch.zeros(T, B, D, device="cuda", dtype=torch.bfloat16)
    assert lib.dr_cuda_fm_bwd(_p(dfm), D, _p(emb), B * D, D, _p(ssum), T, D, B, _p(demb), B * D, D, 0, _s()) == 0
    ref.backward(dfm.float())
    torch.cuda.synchronize()
    assert (demb.float() - ef.grad).abs().max().item() < 3e-2 * (ef.grad.abs().max().item() + 1e-3)


@pytest.mark.parametrize("M,N,K", [(4096, 512, 16), (5000, 256, 512), (65536, 512, 368), (3000, 64, 256), (2048, 368, 512), (777, 128, 64)])
def test_gemm_tn_v2_epilogue_stats_and_aux(M, N, K):
    """v2 epilogue: TMA-store staging, fused column statistics, aux tile as ReLU mask / statistics partner."""
    torch.manual_seed(7)
    lib = _lib()
    A = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    B = (torch.randn(N, K, device="cuda") * 0.1).bfloat16()
    bias = torch.randn(N, device="cuda") * 0.1
    ref0 = A.float() @ B.float().t()
    # (a) forward: bias + relu + S1 = sum(out), S2 = sum(out^2)
    out = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
    S1 = torch.zeros(N, device="cuda"); S2 = torch.zeros(N, device="cuda")
    assert lib.dr_cuda_gemm_tn_ex(_p(A), K, _p(B), K, M, N, K, _p(bias), 1, None, 0, 0, _p(out), N, None, _p(S1), _p(S2), 0, 0, _s()) == 0
    torch.cuda.synchronize()
    ref = (ref0 + bias).relu()
    scale = ref.abs().max().item() + 1e-6
    assert (out.float() - ref).abs().max().item() / scale < 2e-2
    assert (S1 - ref.sum(0)).abs().max().item() < 2e-3 * M ** 0.5 * scale + 1e-2 * ref.sum(0).abs().max().item()
    assert (S2 - (ref * ref).sum(0)).abs().max().item() < 2e-2 * (ref * ref).sum(0).abs().max().item() + 1e-3
    # (b) backward dX with ReLU mask + S1 (bias gradient)
    act = torch.randn(M, N, device="cuda").relu().bfloat16()
    S1.zero_()
    assert lib.dr_cuda_gemm_tn_ex(_p(A), K, _p(B), K, M, N, K, None, 0, _p(act), N, 1, _p(out), N, None, _p(S1), None, 0, 0, _s()) == 0
    torch.cuda.synchronize()
    refm = ref0 * (act.float() > 0)
    assert (out.float() - refm).abs().max().item() < 2e-2 * (refm.abs().max().item() + 1e-6)
    assert (S1 - refm.sum(0)).abs().max().item() < 1e-2 * refm.abs().sum(0).max().item() + 1e-3
    # (c) backward dX with BatchNorm-backward statistics: S1 = sum(out), S2 = sum(out * aux), no mask
    S1.zero_(); S2.zero_()
    assert lib.dr_cuda_gemm_tn_ex(_p(A), K, _p(B), K, M, N, K, None, 0, _p(act), N, 2, _p(out), N, None, _p(S1), _p(S2), 0, 0, _s()) == 0
    torch.cuda.synchronize()
    assert (out.float() - ref0).abs().max().item() < 2e-2 * (ref0.abs().max().item() + 1e-6)
    assert (S2 - (ref0 * act.float()).sum(0)).abs().max().item() < 1e-2 * (ref0.abs() * act.float()).sum(0).max().item() + 1e-3
    assert (S1 - ref0.sum(0)).abs().max().item() < 1e-2 * ref0.abs().sum(0).max().item() + 1e-3


def test_bn_fold_fixup_and_bwd_apply_v2():
    torch.manual_seed(8)
    lib = _lib()
    B, K, Nn = 4096, 256, 64
    a = torch.randn(B, K, device="cuda").relu().bfloat16()
    gamma = torch.rand(K, device="cuda") + 0.5; beta = torch.randn(K, device="cuda") * 0.1
    Wn = torch.randn(Nn, K, device="cuda") * 0.1; bn = torch.randn(Nn, device="cuda") * 0.1
    S1 = a.float().sum(0); S2 = (a.float() ** 2).sum(0)
    mean, rstd, scale, shift = (torch.zeros(K, device="cuda") for _ in range(4))
    rm, rv = torch.zeros(K, device="cuda"), torch.ones(K, device="cuda")
    Wf = torch.empty(Nn, K, device="cuda", dtype=torch.bfloat16); bf = torch.empty(Nn, device="cuda")
    assert lib.dr_cuda_bn_fold(_p(S1), _p(S2), K, B, _p(gamma), _p(beta), 1e-3, 0.99, _p(rm), _p(rv), _p(mean), _p(rstd), _p(scale), _p(shift), 1,
                               _p(Wn), _p(bn), Nn, K, _p(Wf), _p(bf), _s()) == 0
    torch.cuda.synchronize()
    y = torch.nn.functional.batch_norm(a.float(), None, None, gamma, beta, True, 0.0, 1e-3)
    ref = y @ Wn.t() + bn
    got = a.float() @ Wf.float().t() + bf
    assert (got - ref).abs().max().item() < 3e-2 * (ref.abs().max().item() + 1)
    # dW fix-up: dW = G * s + db t^T
    da = torch.randn(B, Nn, device="cuda") * 0.1
    G = (da.t() @ a.float()).contiguous(); db = da.sum(0)
    dW = G.clone()
    assert lib.dr_cuda_dw_fixup(_p(dW), _p(db), _p(scale), _p(shift), Nn, K, K, _s()) == 0
    torch.cuda.synchronize()
    assert (dW - da.t() @ (a.float() * scale + shift)).abs().max().item() < 1e-2
    # bn backward apply v2 (+ fused bias gradient)
    dy = (torch.randn(B, K, device="cuda") * 0.1).bfloat16()
    c1 = dy.float().mean(0); xhat = (a.float() - mean) * rstd; c2 = (dy.float() * xhat).mean(0)
    out = torch.empty_like(a); dbias = torch.zeros(K, device="cuda")
    assert lib.dr_cuda_bn_bwd_apply_v2(_p(dy), _p(a), B, K, K, _p(scale), _p(mean), _p(rstd), _p(c1), _p(c2), _p(out), 1, _p(dbias), _s()) == 0
    torch.cuda.synchronize()
    refda = scale * (dy.float() - c1 - xhat * c2) * (a.float() > 0)
    assert (out.float() - refda).abs().max().item() < 2e-2 * (refda.abs().max().item() + 1e-3)
    assert (dbias - refda.sum(0)).abs().max().item() < 2e-2 * refda.abs().sum(0).max().item() + 1e-3
