"""Shared cases of the MaskNet tests (tests/test_cuda_emu_masknet.py on the CUDA-on-CPU emulation, device "cpu";
tests/test_gpu_zzzzzzzzzz_masknet.py on an H100, device "cuda"): zoo.MaskBlockNet against a float64 transcription of the reference
model, the MaskBlock kernels (LayerNorm GEMM epilogue, k_ln_relu_bwd, k_bn_apply_mul, k_bn_mul_bwd) against float64, and engines.

Bounds.  Every kernel computes in fp32 and rounds its bf16 outputs once, so an output element may be off by half a bf16 ulp of itself
(2^-9 relative) plus the fp32 error of what fed it; ``bf16_bound`` allows 2^-8 |ref| plus an fp32 term scaled by the magnitudes that
were summed.  The float64 references read the same bf16 inputs the kernels read."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from deeprec_b200 import _native

CARDS = [50, 1000, 7, 300] + [97] * 22
SIMT_M = [1, 37, 300]
SIMT_N = [16, 48, 64, 128]


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _s():
    return _native.stream_ptr()


def _sync(dev):
    if dev == "cuda":
        torch.cuda.synchronize()


def bf16_bound(ref: np.ndarray, mag: np.ndarray | float) -> np.ndarray:
    return 2.0 ** -8 * np.abs(ref) + 1e-5 * np.asarray(mag) + 1e-30


def assert_close(got, ref, mag, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    err = np.abs(got - ref)
    bound = bf16_bound(ref, mag)
    assert np.isfinite(got).all(), what
    assert (err <= bound).all(), (what, float(err.max()), float((err - bound).max()))


def pitched(rows, cols, ld, dev, dtype=torch.bfloat16, fill=None):
    """[rows, cols] view of a [rows, ld] buffer (the padding columns hold NaN)."""
    buf = torch.full((rows, ld), float("nan"), dtype=dtype)
    if fill is not None:
        buf[:, :cols] = fill.to(dtype)
    return buf.to(dev)


# ---- reference model, float64 (modelzoo/masknet/train.py:150-224) ---------------------------------------------------------------------
def reference_logits(m, dense: torch.Tensor, embs: torch.Tensor) -> torch.Tensor:
    """MaskBlockNet in training mode, float64, written from the reference: _dnn with use_bn (dense + ReLU, then batch normalisation over the
    batch), the bias-free block dense, Keras LayerNormalization, ReLU; the head's logit is a plain dense (the documented deviation)."""
    f = lambda t: t.detach().double()
    x = torch.cat([dense, embs.flatten(1)], 1).double()

    def bn(t, mod):
        mu = t.mean(0)
        var = ((t - mu) ** 2).mean(0)
        return (t - mu) / torch.sqrt(var + mod.eps) * f(mod.weight) + f(mod.bias)

    def dense_relu_bn(t, lin, mod):
        return bn(torch.relu(t @ f(lin.weight).t() + f(lin.bias)), mod)

    def block(b, v_hidden):
        assert b.fc3.bias is None and b.bn1.eps == 1e-3 and b.bn2.eps == 1e-3 and b.ln.eps == 1e-3
        mask = dense_relu_bn(dense_relu_bn(x, b.fc1, b.bn1), b.fc2, b.bn2)
        h = (mask * v_hidden) @ f(b.fc3.weight).t()
        mu = h.mean(1, keepdim=True)
        var = ((h - mu) ** 2).mean(1, keepdim=True)
        return torch.relu((h - mu) / torch.sqrt(var + b.ln.eps) * f(b.ln.weight) + f(b.ln.bias))

    if m.model_type == "parallel":
        h = torch.cat([block(b, x) for b in m.blocks], 1)
        lins = [l for l in m.head if isinstance(l, torch.nn.Linear)]
        bns = [l for l in m.head if isinstance(l, torch.nn.BatchNorm1d)]
        assert [l.out_features for l in lins] == [64, 16] and len(bns) == 2
        for lin, mod in zip(lins, bns):
            h = dense_relu_bn(h, lin, mod)
    else:
        h = x
        for b in m.blocks:
            h = block(b, h)
    return (h @ f(m.out.weight).t() + f(m.out.bias)).squeeze(-1)


# ---- SIMT kernels -----------------------------------------------------------------------------------------------------------------------
def ln_relu_bwd_case(dev, M, N, seed=0):
    """k_ln_relu_bwd on pitched operands against float64; row 0 is a constant row (x^ = 0), row 1 has y <= 0 everywhere (ReLU-dead)."""
    g_ = torch.Generator().manual_seed(seed)
    ld = N + 8
    g = torch.randn(M, N, generator=g_)
    xh = torch.randn(M, N, generator=g_)
    gamma = torch.randn(N, generator=g_)
    beta = torch.randn(N, generator=g_) * 0.1
    rstd = torch.rand(M, generator=g_) * 2 + 0.1
    xh[0] = 0.0
    y = torch.relu(gamma * xh + beta)
    if M > 1:
        y[1] = 0.0
    gb, yb, xb = (pitched(M, N, ld, dev, fill=t) for t in (g, y, xh))
    rs, gm = rstd.to(dev), gamma.to(dev)
    outs = []
    for _ in range(2):
        dh = pitched(M, N, ld, dev)
        dg, db = torch.zeros(N, device=dev), torch.zeros(N, device=dev)
        rc = _native.cuda().dr_cuda_ln_relu_bwd(_p(gb), ld, _p(yb), ld, _p(xb), ld, _p(rs), _p(gm), M, N, _p(dh), ld, _p(dg), _p(db), _s())
        assert rc == 0, rc
        _sync(dev)
        outs.append((dh.cpu(), dg.cpu(), db.cpu()))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                           b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))
    dh, dg, db = outs[0]
    G, Y, X = (t.cpu()[:, :N].double() for t in (gb, yb, xb))
    d = G * (Y > 0)
    dgm = d * gamma.double()
    ref = rstd.double()[:, None] * (dgm - dgm.mean(1, keepdim=True) - X * (dgm * X).mean(1, keepdim=True))
    mag = rstd.double()[:, None] * (dgm.abs().max(1, keepdim=True).values * (1 + X.abs()))
    assert_close(dh[:, :N].double().numpy(), ref.numpy(), mag.numpy(), "dh")
    assert torch.isnan(dh[:, N:].float()).all(), "dh padding written"
    if M > 1:
        assert (dh[1, :N].float() == 0).all(), "ReLU-dead row"
    assert_close(dg.numpy(), (d * X).sum(0).numpy(), (d * X).abs().sum(0).numpy(), "dgamma")
    assert_close(db.numpy(), d.sum(0).numpy(), d.abs().sum(0).numpy(), "dbeta")


def bn_mul_case(dev, M, N, seed=0):
    """k_bn_apply_mul and k_bn_mul_bwd on pitched operands against float64; two backward calls bit-identical."""
    g_ = torch.Generator().manual_seed(seed)
    ld = N + 16
    a = torch.relu(torch.randn(M, N, generator=g_))
    v = torch.randn(M, N, generator=g_)
    dp = torch.randn(M, N, generator=g_)
    scale, shift = torch.randn(N, generator=g_), torch.randn(N, generator=g_)
    ab, vb, dpb = (pitched(M, N, ld, dev, fill=t) for t in (a, v, dp))
    sc, sf = scale.to(dev), shift.to(dev)
    lib = _native.cuda()
    p = pitched(M, N, ld, dev)
    assert lib.dr_cuda_bn_apply_mul(_p(ab), ld, _p(sc), _p(sf), _p(vb), ld, M, N, _p(p), ld, _s()) == 0
    _sync(dev)
    A, V, DP = (t.cpu()[:, :N].double() for t in (ab, vb, dpb))
    bnv = A * scale.double() + shift.double()
    assert_close(p.cpu()[:, :N].double().numpy(), (bnv * V).numpy(), (bnv.abs() * V.abs()).numpy(), "p")
    assert torch.isnan(p.cpu()[:, N:].float()).all()
    outs = []
    for _ in range(2):
        dv, dm = pitched(M, N, ld, dev), pitched(M, N, ld, dev)
        S1, S2 = torch.zeros(N, device=dev), torch.zeros(N, device=dev)
        rc = lib.dr_cuda_bn_mul_bwd(_p(dpb), ld, _p(ab), ld, _p(vb), ld, _p(sc), _p(sf), M, N, _p(dv), ld, _p(dm), ld, _p(S1), _p(S2), _s())
        assert rc == 0, rc
        _sync(dev)
        outs.append((dv.cpu(), dm.cpu(), S1.cpu(), S2.cpu()))
    for x, y in zip(outs[0], outs[1]):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))
    dv, dm, S1, S2 = outs[0]
    assert_close(dv[:, :N].double().numpy(), (DP * bnv).numpy(), (DP.abs() * bnv.abs()).numpy(), "dv")
    assert_close(dm[:, :N].double().numpy(), (DP * V).numpy(), (DP * V).abs().numpy(), "dm")
    DM = dm[:, :N].double()                                           # the sums are of the bf16 dm the BatchNorm backward reads
    assert_close(S1.numpy(), DM.sum(0).numpy(), DM.abs().sum(0).numpy(), "sum dm")
    assert_close(S2.numpy(), (DM * A).sum(0).numpy(), (DM * A).abs().sum(0).numpy(), "sum dm a")


# ---- LayerNorm GEMM epilogue ------------------------------------------------------------------------------------------------------------
def gemm_ln_case(dev, M, N, K, bias: bool, relu: bool, ldc_pad: int = 0, seed=0):
    """dr_cuda_gemm_tn_ln against float64 of the same bf16 operands.  Row 0 is constant (zero variance: B's rows equal, no bias), row 1 has
    |mean| >> std.  Bound: y and x^ are rounded once to bf16; the fp32 accumulation of K products and the fp32 statistics add at most
    ~K 2^-24 sum|a b| to h, which enters x^ multiplied by rstd."""
    g_ = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g_)
    Bw = torch.randn(N, K, generator=g_) / K ** 0.5
    if M > 1:
        A[1] = A[1] * 0.01 + 3.0                                        # h = A Bw^T: large common offset across columns
        Bw[:, 0] += 20.0
    b = torch.randn(N, generator=g_) if bias else None
    gamma, beta = torch.randn(N, generator=g_), torch.randn(N, generator=g_)
    Ab, Bb = A.to(torch.bfloat16), Bw.to(torch.bfloat16)
    if M > 0:
        Ab[0] = 0.0                                                      # h = bias: constant only without bias
    ldc = N + ldc_pad
    Ad, Bd = Ab.to(dev), Bb.to(dev)
    out = pitched(M, N, ldc, dev)
    xh = pitched(M, N, N, dev)
    rstd = torch.full((M,), float("nan"), device=dev)
    bd = b.to(dev) if b is not None else None
    gd, bed = gamma.to(dev), beta.to(dev)
    rc = _native.cuda().dr_cuda_gemm_tn_ln(_p(Ad), K, _p(Bd), K, M, N, K, _p(bd), _p(gd), _p(bed), 1e-3, int(relu), _p(out), ldc, _p(xh), N,
                                           _p(rstd), 0, _s())
    assert rc == 0, rc
    _sync(dev)
    h = Ab.double() @ Bb.double().t() + (b.double() if b is not None else 0)
    mu = h.mean(1, keepdim=True)
    var = ((h - mu) ** 2).mean(1, keepdim=True)
    rs = 1 / torch.sqrt(var + 1e-3)
    x = (h - mu) * rs
    y = gamma.double() * x + beta.double()
    if relu:
        y = torch.relu(y)
    acc_mag = (Ab.double().abs() @ Bb.double().abs().t()).max(1, keepdim=True).values + (b.double().abs().max() if b is not None else 0)
    mag_x = acc_mag * rs * 2                                          # bf16_bound takes 1e-5 of it: the fp32 error of h, times rstd
    mag_y = mag_x * gamma.double().abs()
    o = out.cpu()
    assert_close(o[:, :N].double().numpy(), y.numpy(), (mag_y + 1e-6).numpy(), "y")
    if ldc_pad:
        assert torch.isnan(o[:, N:].float()).all(), "columns past N written"
    assert_close(xh.cpu().double().numpy(), x.numpy(), (mag_x + 1e-6).numpy(), "xhat")
    r = rstd.cpu().double()
    assert ((r - rs[:, 0]).abs() <= 1e-5 * rs[:, 0] * (1 + mag_x[:, 0])).all(), "rstd"
    if M > 0 and not bias:
        assert (xh.cpu()[0].float() == 0).all(), "constant row"


def gemm_ln_refusals(dev):
    """Operand contract: -2 N > 128, N not a multiple of 8 (odd N included), a pitch not a multiple of 8; -3 misaligned; -5 short pitch; -4 no
    gamma.  Nothing is launched: the output keeps its NaN fill."""
    lib = _native.cuda()
    A = torch.zeros(4, 64, dtype=torch.bfloat16, device=dev)
    B = torch.zeros(256, 64, dtype=torch.bfloat16, device=dev)
    out = torch.full((4, 256), float("nan"), dtype=torch.bfloat16, device=dev)
    g = torch.ones(256, device=dev)

    def call(N, lda=64, ldc=256, a_off=0, gamma=True):
        return lib.dr_cuda_gemm_tn_ln(C.c_void_p(A.data_ptr() + a_off), lda, _p(B), 64, 4, N, 64 if not a_off else 56, None, _p(g) if gamma else None,
                                      _p(g), 1e-3, 1, _p(out), ldc, None, 0, None, 0, _s())
    assert call(136) == -2
    assert call(63) == -2
    assert call(60) == -2
    assert call(64, ldc=100) == -2
    assert call(64, a_off=2) == -3
    assert call(64, ldc=56) == -5
    assert call(64, gamma=False) == -4
    _sync(dev)
    assert torch.isnan(out.float()).all()


# ---- the op against float64 autograd ----------------------------------------------------------------------------------------------------
def op_grad_case(dev, M, E, H, O=64, seed=0, same_input=False):
    """FusedMaskBlock (kernels) against float64 autograd of its torch expression on the same bf16-rounded inputs and parameters; returns the
    kernel path's (out, grads) so a caller can check repeatability."""
    from deeprec_b200.nn import FusedMaskBlock
    torch.manual_seed(seed)
    blk = FusedMaskBlock(H, E, O)
    with torch.no_grad():
        for prm in blk.parameters():
            prm.copy_((prm + 0.1 * torch.randn_like(prm)).to(torch.bfloat16).float())
        # a row's |x^| is at most sqrt(O - 1); beta = 6 keeps the output ReLU away from its kink, where bf16 rounding upstream would flip an
        # element's mask and move its gradient by O(1) (k_ln_relu_bwd's masking is checked on its own in ln_relu_bwd_case)
        blk.ln.bias.fill_(6.0)
    ref = FusedMaskBlock(H, E, O).double()
    ref.load_state_dict(blk.state_dict())
    g_ = torch.Generator().manual_seed(seed + 1)
    ve = torch.randn(M, E, generator=g_).to(torch.bfloat16).float()
    vh = ve if same_input else torch.randn(M, H, generator=g_).to(torch.bfloat16).float()
    gy = torch.randn(M, O, generator=g_).to(torch.bfloat16).float()
    # float64 reference on the CPU path
    re = ve.double().requires_grad_()
    rh = re if same_input else vh.double().requires_grad_()
    ry = ref.expression(re, rh)
    ry.backward(gy.double())
    # kernel path
    blk = blk.to(dev)
    ke = ve.to(dev).requires_grad_()
    kh = ke if same_input else vh.to(dev).requires_grad_()
    ky = blk(ke, kh)
    ky.backward(gy.to(dev))
    _sync(dev)
    out = ky.detach().float().cpu()
    # every stage stores bf16 activations (2^-9 each), and the LayerNorm divides by a batch of 40 rows' spread: 2 % of the largest output
    assert (out.double() - ry.detach()).abs().max().item() < 0.02 * ry.detach().abs().max().item()
    grads = {"v_emb": ke.grad.float().cpu()}
    refs = {"v_emb": re.grad}
    if not same_input:
        grads["v_hidden"] = kh.grad.float().cpu(); refs["v_hidden"] = rh.grad
    for (n, p), (_, rp) in zip(blk.named_parameters(), ref.named_parameters()):
        grads[n] = p.grad.float().cpu(); refs[n] = rp.grad
    rels = {}
    for n, r in refs.items():
        got, r = grads[n].double(), r.double()
        rels[n] = ((got - r).norm() / (r.norm() + 1e-12)).item()
    # relative Frobenius error.  Every stage keeps bf16 activations (2^-9 each), and a ReLU ahead of a BatchNorm whose pre-activation lies
    # within that rounding of 0 flips its mask; a BatchNorm's bias gradient is made of the masked elements alone, so it shows flips most.
    assert max(rels.values()) < 0.25, rels
    for a, b in ((blk.bn1, ref.bn1), (blk.bn2, ref.bn2)):           # the moving averages were updated in the step
        assert torch.allclose(a.running_mean.cpu().double(), b.running_mean, rtol=2e-2, atol=2e-3)
        assert torch.allclose(a.running_var.cpu().double(), b.running_var, rtol=2e-2, atol=2e-3)
    return out, grads


# ---- engines ------------------------------------------------------------------------------------------------------------------------------
def build(name, dev=None, num_blocks=None):
    """Zoo model ``name``; ``num_blocks`` builds ``masknet_<mode>`` with fewer MaskBlocks (the emulation tier keeps its host-loop GEMMs short)."""
    import deeprec_b200 as dr
    from deeprec_b200.models.zoo import MaskBlockNet, build_model
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    if num_blocks is not None:
        return MaskBlockNet(model_type=name.split("_", 1)[1], num_blocks=num_blocks, device=dev or "cpu")
    return build_model(name, device=dev or "cpu")


def make_engine(name, B, dev=None, num_blocks=None, **kw):
    from deeprec_b200.models.rec_engine import criteo_engine
    kw.setdefault("learning_rate", 0.05)
    return criteo_engine(build(name, dev, num_blocks), B, table_rows=CARDS, device=dev, **kw)


def batch(B, seed, learnable=False):
    g = torch.Generator().manual_seed(seed)
    ids = torch.stack([torch.randint(0, c, (B,), generator=g) for c in CARDS])
    dense = torch.rand(B, 13, generator=g) * 3
    if learnable:                                                     # label = a function of two dense features and table 2's id
        y = ((dense[:, 0] - dense[:, 1] + (ids[2] % 2).float()) > 1.0).float()
    else:
        y = (torch.rand(B, generator=g) < 0.3).float()
    return ids, y, {"dense": dense}


def replica_step_losses(eng_net, tables, batches, lr=0.05):
    """The torch replica of a criteo_engine step (Adagrad, initial accumulator 0.1, fp32): one loss per batch."""
    import copy
    net = copy.deepcopy(eng_net)
    opt = torch.optim.Adagrad(list(net.parameters()) + list(tables.parameters()), lr=lr, initial_accumulator_value=0.1, eps=0.0)
    out = []
    for ids, y, dense in batches:
        embs = torch.stack([tables[t](ids[t]) for t in range(26)], 1)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(net.logits(dense["dense"], embs).float(), y)
        opt.zero_grad(); loss.backward(); opt.step()
        out.append(loss.item())
    return out, net


def replica_tables(eng):
    tables = torch.nn.ModuleList([torch.nn.Embedding(c, 16) for c in CARDS])
    with torch.no_grad():
        for t, emb in enumerate(tables):
            dm = eng.tables[t].default_matrix.cpu()
            emb.weight.copy_(dm[torch.arange(CARDS[t]) % dm.shape[0]])
    return tables
