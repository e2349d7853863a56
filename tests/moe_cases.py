"""Shared cases of the expert-mixture tests (tests/test_cuda_emu_moe.py on the CUDA-on-CPU emulation, device "cpu";
tests/test_gpu_zzzzzzzzzzz_moe.py on an H100, device "cuda"): the grouped GEMMs against per-group calls (bit for bit) and float64, the
mixture kernels against float64, the ops' gradients against float64 autograd, MMoE / PLE with ``moe=`` against the plain modules, and
engines.

Bounds as in masknet_cases: an output rounded once to bf16 from an fp32 computation may be off by 2^-8 |ref| plus an fp32 term scaled by
the magnitudes that were summed.  The float64 references read the same bf16 inputs the kernels read."""
from __future__ import annotations

import copy
import ctypes as C

import numpy as np
import torch

from deeprec_b200 import _native
from masknet_cases import assert_close

MAX_GROUPS = 12


def _s():
    return _native.stream_ptr()


def _sync(dev):
    if dev == "cuda":
        torch.cuda.synchronize()


def _arr(ct, vals):
    return (ct * len(vals))(*vals)


def _ptrs(vals):
    return _arr(C.c_void_p, [v if v is None or isinstance(v, int) else v.data_ptr() for v in vals])


def _i64(vals):
    return _arr(C.c_int64, vals)


def _ref(x):
    return x.detach().double().cpu()


# ---- grouped GEMMs ---------------------------------------------------------------------------------------------------------------
def _packed(rows, G, cols, ld, gen, dev, scale=1.0):
    """one [rows, G * ld] bf16 buffer: group g's [rows, cols] operand at column offset g * ld (the gap holds NaN, which must not be read)"""
    buf = torch.full((rows, G * ld), float("nan"), dtype=torch.bfloat16)
    for g in range(G):
        buf[:, g * ld: g * ld + cols] = (torch.randn(rows, cols, generator=gen) * scale).to(torch.bfloat16)
    return buf.to(dev)


def _col(buf, g, ld):
    return buf.data_ptr() + g * ld * buf.element_size()


def grouped_tn_case(dev, G, M, N, K, bias=True, relu=True, mask=False, stats=False, seed=0):
    """dr_cuda_gemm_tn_grouped over pitched, offset group operands of packed buffers against G dr_cuda_gemm_tn_ex calls (bit for bit,
    outputs and S1) and against float64."""
    lib = _native.cuda()
    gen = torch.Generator().manual_seed(seed)
    lda, ldb, ldc = K + 8, K + 16, N + 8
    A = _packed(M, G, K, lda, gen, dev)
    B = _packed(N, G, K, ldb, gen, dev, K ** -0.5)
    b = (torch.randn(G, N, generator=gen) * 0.1).to(dev) if bias else None
    aux = _packed(M, G, N, ldc, gen, dev) if mask else None
    out = torch.zeros(M, G * ldc, dtype=torch.bfloat16, device=dev)
    S1 = (torch.randn(G, N, generator=gen)).to(dev) if stats else None
    S1_ref = S1.clone() if stats else None
    rc = lib.dr_cuda_gemm_tn_grouped(G, _ptrs([_col(A, g, lda) for g in range(G)]), _i64([G * lda] * G), _ptrs([_col(B, g, ldb) for g in range(G)]),
                                     _i64([G * ldb] * G), M, N, K, _ptrs([b[g] for g in range(G)]) if bias else None, int(relu),
                                     _ptrs([_col(aux, g, ldc) for g in range(G)]) if mask else None, _i64([G * ldc] * G) if mask else None,
                                     _ptrs([_col(out, g, ldc) for g in range(G)]), _i64([G * ldc] * G),
                                     _ptrs([S1[g] for g in range(G)]) if stats else None, 0, _s())
    assert rc == 0, rc
    ref_out = torch.zeros_like(out)
    for g in range(G):
        rc = lib.dr_cuda_gemm_tn_ex(C.c_void_p(_col(A, g, lda)), G * lda, C.c_void_p(_col(B, g, ldb)), G * ldb, M, N, K,
                                    C.c_void_p(b[g].data_ptr()) if bias else None, int(relu), C.c_void_p(_col(aux, g, ldc)) if mask else None,
                                    G * ldc, 1 if mask else 0, C.c_void_p(_col(ref_out, g, ldc)), G * ldc, None,
                                    C.c_void_p(S1_ref[g].data_ptr()) if stats else None, None, 0, 0, _s())
        assert rc == 0, rc
    _sync(dev)
    for g in range(G):
        sl = slice(g * ldc, g * ldc + N)
        assert torch.equal(out[:, sl].view(torch.int16), ref_out[:, sl].view(torch.int16)), ("group", g)
        if stats:
            assert torch.equal(S1[g], S1_ref[g]), ("S1", g)
    S1_0 = S1_ref  # float64 check of the values
    for g in range(G):
        a, w = _ref(A[:, g * lda: g * lda + K]), _ref(B[:, g * ldb: g * ldb + K])
        r = a @ w.t() + (_ref(b[g]) if bias else 0)
        if relu:
            r = r.clamp_min(0)
        if mask:
            r = r * (_ref(aux[:, g * ldc: g * ldc + N]) > 0)
        assert_close(_ref(out[:, g * ldc: g * ldc + N]).numpy(), r.numpy(), (a.abs() @ w.abs().t()).numpy() + 1, ("out", g))
    return out, S1_0


def grouped_dw_case(dev, G, M, N, K, seed=0):
    """dr_cuda_gemm_dw_grouped against G dr_cuda_gemm_dw calls (bit for bit) and float64; dW is accumulated into."""
    lib = _native.cuda()
    gen = torch.Generator().manual_seed(seed)
    ldy, ldx = N + 8, K + 8
    dY = _packed(M, G, N, ldy, gen, dev)
    X = _packed(M, G, K, ldx, gen, dev)
    dW0 = torch.randn(G, N, K, generator=gen).to(dev)
    dW, dW_ref = dW0.clone(), dW0.clone()
    rc = lib.dr_cuda_gemm_dw_grouped(G, _ptrs([_col(dY, g, ldy) for g in range(G)]), _i64([G * ldy] * G), _ptrs([_col(X, g, ldx) for g in range(G)]),
                                     _i64([G * ldx] * G), M, N, K, _ptrs([dW[g] for g in range(G)]), _i64([K] * G), 0, _s())
    assert rc == 0, rc
    for g in range(G):
        rc = lib.dr_cuda_gemm_dw(C.c_void_p(_col(dY, g, ldy)), G * ldy, C.c_void_p(_col(X, g, ldx)), G * ldx, M, N, K, C.c_void_p(dW_ref[g].data_ptr()),
                                 K, 0, _s())
        assert rc == 0, rc
    _sync(dev)
    assert torch.equal(dW, dW_ref)
    for g in range(G):
        y, x = _ref(dY[:, g * ldy: g * ldy + N]), _ref(X[:, g * ldx: g * ldx + K])
        r = _ref(dW0[g]) + y.t() @ x
        err = (_ref(dW[g]) - r).abs()
        assert bool((err <= 1e-5 * (y.abs().t() @ x.abs() + _ref(dW0[g]).abs()) + 1e-6).all()), float(err.max())


def grouped_refusals(dev):
    """Every refusal code of both grouped entry points (the hardware and the emulation give the same)."""
    lib = _native.cuda()
    a = torch.zeros(64, 128, dtype=torch.bfloat16, device=dev)
    o = torch.zeros(64, 128, dtype=torch.bfloat16, device=dev)
    S = torch.zeros(128, device=dev)

    def tn(G=2, lda=128, ldb=128, ldc=128, N=64, K=64, A_off=0, S1=False, S1_null=False):
        p = a.data_ptr() + A_off
        s1 = _ptrs([S] * G) if S1 else None
        if S1_null:
            s1 = _ptrs([S] + [None] * (G - 1))
        return lib.dr_cuda_gemm_tn_grouped(G, _ptrs([p] * G), _i64([lda] * G), _ptrs([a] * G), _i64([ldb] * G), 64, N, K, None, 0, None, None,
                                           _ptrs([o] * G), _i64([ldc] * G), s1, 0, _s())

    assert tn(G=0) == -6 and tn(G=MAX_GROUPS + 1) == -6
    assert tn(lda=124) == -2 and tn(ldb=60) == -2 and tn(ldc=100) == -2 and tn(N=60) == -2
    assert tn(A_off=8) == -3
    assert tn(K=136) == -5 and tn(N=136) == -5
    assert tn(S1_null=True) == -4
    assert tn(S1=True) == 0

    def dw(G=2, ldy=128, ldx=128):
        return lib.dr_cuda_gemm_dw_grouped(G, _ptrs([a] * G), _i64([ldy] * G), _ptrs([a] * G), _i64([ldx] * G), 64, 64, 64, _ptrs([S] * G),
                                           _i64([64] * G), 0, _s())

    assert dw(G=0) == -6 and dw(G=MAX_GROUPS + 1) == -6
    assert dw(ldy=124) == -2 and dw(ldx=100) == -2
    _sync(dev)


# ---- mixture kernels ---------------------------------------------------------------------------------------------------------------
MMOE_MAP = ([0, 1, 2], [0, 1, 2])                                    # 3 experts, 2 task gates reading all of them
PLE_MAP = ([0, 1, 4], [2, 3, 4], [0, 1, 2, 3, 4])                    # 2 x 2 specific + 1 shared: the shared expert feeds 3 gates


def mix_case(dev, M, H, select, K=40, seed=0, saturate=False):
    """nn.fused_moe_mix forward and backward against float64 autograd of softmax(x W^T + b) . experts, from the same bf16 inputs; returns the
    outputs and gradients (for repeatability checks)."""
    from deeprec_b200.nn import fused_moe_mix
    gen = torch.Generator().manual_seed(seed)
    E_total = 1 + max(max(s) for s in select)
    T = len(select)
    X = torch.randn(M, E_total, H, generator=gen).to(torch.bfloat16)
    xs = [torch.randn(M, K, generator=gen).to(torch.bfloat16) for _ in range(T)]
    gates = [torch.nn.Linear(K, len(s)) for s in select]
    with torch.no_grad():
        for t, gt in enumerate(gates):
            gt.weight.copy_(torch.randn(len(select[t]), K, generator=gen) * (40.0 if saturate and t == 0 else K ** -0.5))
            gt.bias.copy_(torch.randn(len(select[t]), generator=gen) * 0.1)
    dmix = [torch.randn(M, H, generator=gen).to(torch.bfloat16) for _ in range(T)]
    Xd = X.clone().to(dev).requires_grad_(True)
    xd = [x.clone().to(dev).requires_grad_(True) for x in xs]
    gd = [copy.deepcopy(g).to(dev) for g in gates]
    out = fused_moe_mix(xd, gd, Xd, select)
    torch.autograd.backward(out, [d.to(dev) for d in dmix])
    _sync(dev)
    # float64
    X64 = X.double().requires_grad_(True)
    x64 = [x.double().requires_grad_(True) for x in xs]
    W64 = [g.weight.detach().double().requires_grad_(True) for g in gates]
    b64 = [g.bias.detach().double().requires_grad_(True) for g in gates]
    ref = [(torch.softmax(x @ W.t() + b, -1).unsqueeze(-1) * X64[:, list(s)]).sum(1) for x, W, b, s in zip(x64, W64, b64, select)]
    torch.autograd.backward(ref, [d.double() for d in dmix])
    mag_mix = 10 * X.double().abs().amax(1).numpy()                  # fp32 term: the softmax runs on fast-math exp and divide
    for t in range(T):
        assert out[t].dtype == torch.bfloat16
        assert_close(_ref(out[t]).numpy(), ref[t].detach().numpy(), mag_mix, ("mix", t))
    # expert gradient: sum over readers of g * dmix (bf16 output)
    dmag = sum(d.double().abs() for d in dmix).unsqueeze(1).expand(-1, E_total, -1).numpy()
    assert_close(_ref(Xd.grad).numpy(), X64.grad.numpy(), dmag, "dX")
    # the gate path: the logit gradients sum H products, the weight gradients M more
    hmag = float((X.double().abs().sum(2).amax() * max(d.double().abs().max() for d in dmix)).item())
    for t in range(T):
        kmag = hmag * float(gates[t].weight.detach().abs().sum(0).max()) + 1
        assert_close(_ref(xd[t].grad).numpy(), x64[t].grad.numpy(), kmag, ("dx", t))
        wmag = hmag * M * float(xs[t].float().abs().max()) + 1
        err = (_ref(gd[t].weight.grad) - W64[t].grad).abs()
        assert bool((err <= 2.0 ** -8 * W64[t].grad.abs() + 1e-5 * wmag).all()), ("dW", t, float(err.max()))
        err = (_ref(gd[t].bias.grad) - b64[t].grad).abs()
        assert bool((err <= 2.0 ** -8 * b64[t].grad.abs() + 1e-5 * hmag * M + 1e-6).all()), ("db", t, float(err.max()))
    return [o.detach().clone() for o in out], Xd.grad.clone(), [x.grad.clone() for x in xd], [g.weight.grad.clone() for g in gd]


def mix_refusals(dev):
    from deeprec_b200.nn import fused_moe_mix
    import pytest
    x = torch.randn(4, 8, device=dev)
    with pytest.raises(ValueError):                                  # H not a multiple of 8
        fused_moe_mix([x], [torch.nn.Linear(8, 2).to(dev)], torch.randn(4, 2, 12, device=dev), [[0, 1]])
    with pytest.raises(ValueError):                                  # more than 32 experts for one gate
        fused_moe_mix([x], [torch.nn.Linear(8, 33).to(dev)], torch.randn(4, 33, 8, device=dev), [list(range(33))])


# ---- ops' gradients ------------------------------------------------------------------------------------------------------------
def _mlp(dev, sizes, k):
    from deeprec_b200.models.zoo import mlp
    return mlp(sizes, k, device=dev)


def _mlp_bf16_acts(m, x):
    """float64 forward of a Linear + ReLU chain with the weights and every activation rounded to bf16 as the kernels read and store them
    (straight through for the backward), so the float64 ReLU masks are the kernels' masks"""
    from deeprec_b200.nn.layers import _mlp_layers
    ws, bs, last_act = _mlp_layers(m)
    rnd = lambda t: t + (t.detach().to(torch.bfloat16).double() - t.detach())
    h = x
    for i, (W, b) in enumerate(zip(ws, bs)):
        h = h @ rnd(W).t() + b
        if i + 1 < len(ws) or last_act:
            h = torch.relu(h)
        h = rnd(h)
    return h


def expert_grad_case(dev, M, G, K, sizes, shared=True, seed=0):
    """nn.fused_expert_mlps output and gradients against float64 autograd of the MLPs themselves, from the same bf16 input."""
    from deeprec_b200.nn import fused_expert_mlps
    torch.manual_seed(seed)
    mlps = [_mlp(dev, sizes, K) for _ in range(G)]
    m64 = [copy.deepcopy(m).double().cpu() for m in mlps]
    gen = torch.Generator().manual_seed(seed)
    xs = [torch.randn(M, K, generator=gen).to(torch.bfloat16) for _ in range(1 if shared else G)]
    gy = torch.randn(M, G * sizes[-1], generator=gen).to(torch.bfloat16)
    xd = [x.clone().to(dev).requires_grad_(True) for x in xs]
    y = fused_expert_mlps(xd[0] if shared else xd, mlps)
    y.backward(gy.to(dev))
    _sync(dev)
    x64 = [x.double().requires_grad_(True) for x in xs]
    r = torch.cat([_mlp_bf16_acts(m, x64[0] if shared else x64[i]) for i, m in enumerate(m64)], -1)
    r.backward(gy.double())
    assert y.shape == (M, G * sizes[-1]) and y.dtype == torch.bfloat16

    def close(a, b, what):
        # relative Frobenius error: the reference rounds the activations as the kernels do, and the bf16 rounding of the gradients
        # between layers stays far below 1 %; a wrongly wired group (offset, pitch, weight) moves a whole block by O(1)
        a, b = _ref(a), b.detach()
        assert float((a - b).norm()) <= 0.02 * float(b.norm()) + 1e-4, (what, float((a - b).norm()), float(b.norm()))

    close(y, r, "y")
    for i, (x, x_) in enumerate(zip(xd, x64)):
        close(x.grad, x_.grad, ("dx", i))
    for m, m_ in zip(mlps, m64):
        for p, q in zip(m.parameters(), m_.parameters()):
            close(p.grad, q.grad, tuple(p.shape))
    return y.detach().clone(), [p.grad.clone() for m in mlps for p in m.parameters()]


# ---- models and engines ----------------------------------------------------------------------------------------------------------
def model_case(name, dev, M=64, seed=0):
    """MMoE / PLE tower_logits with moe=nn.FUSED_MOE against moe=None on the same parameters: logits and every parameter's gradient."""
    import deeprec_b200 as dr
    from deeprec_b200.models.zoo import build_model
    from deeprec_b200.nn import FUSED_MOE
    dr.embedding_variable.clear_registry()
    torch.manual_seed(seed)
    m = build_model(name, device=dev)
    f = torch.randn(M, m.feat_dim, generator=torch.Generator().manual_seed(seed)).to(torch.bfloat16).float().to(dev)
    params = [p for n, p in m.named_parameters() if not n.startswith(("user", "item", "cat", "emb"))]
    out = {}
    for moe in (None, FUSED_MOE):
        for p in params:
            p.grad = None
        lg = m.tower_logits(f, moe=moe)
        sum(v.float().sum() * (i + 1) for i, v in enumerate(lg.values())).backward()
        out[moe is None] = ({k: v.detach().float() for k, v in lg.items()}, [None if p.grad is None else p.grad.clone() for p in params])
    (la, ga), (lb, gb) = out[True], out[False]
    for k in la:
        assert float((la[k] - lb[k]).abs().max()) <= 0.03 * float(la[k].abs().max()) + 2e-2, k
    for p, a, b in zip(params, ga, gb):
        if a is None or float(a.abs().max()) == 0:
            assert b is None or float(b.abs().max()) == 0
            continue
        assert float((a - b.float()).abs().max()) <= 0.06 * float(a.abs().max()) + 1e-3, tuple(p.shape)
