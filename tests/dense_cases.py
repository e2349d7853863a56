"""Cases for the dense-path kernels of the DLRM step (csrc/cuda/dense_kernels.cu), written once and run on an H100
(tests/test_gpu_dense_edges.py, device "cuda") and on the CUDA-on-CPU emulation (tests/test_cuda_emu_dense_edges.py, device "cpu" inside
``_native.cuda_emulation()``).  Every result is compared with the float64 oracle of tests/dense_ref.py under its bound.

Kernel cases go through the exported dr_cuda_* wrappers.  Every output lives inside a buffer filled with a NaN sentinel the kernels never
store (guard elements before and after it, and the padding columns of a strided output): every sentinel must survive.  Each batch sum is run
once on "exact" inputs, bf16 values k / 8 with |k| <= 8, on which every fp32 partial sum is exact, so the kernel must return the float64 sum
bit for bit and a dropped or doubled row, column, row-group or block partial cannot hide inside a bound; and once on random inputs under the
derived bound.

The engine case runs one eager DLRMEngine step and checks every stage against float64 computed from the engine's own inputs to that stage
(its stored bf16 activations and upstream gradients), so each bound covers one kernel and a failure points at it."""
from __future__ import annotations

import ctypes as C

import torch

import dense_ref as D
from deeprec_b200 import _native
from optim_ref import E, U

BF16_SENT = 0x7FA5                  # NaN payloads no store of the kernels produces
F32_SENT = 0x7FC0DEAD


def _lib():
    return _native.cuda()


def _s():
    return _native.stream_ptr()


def _sync():
    _native.stream_sync()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def on(dev, *ts):
    """Device copies of the inputs, held by the caller until the kernel has run: a temporary ``t.to(dev)`` passed as a raw pointer can be
    freed, and its memory handed to the next copy, before the launch."""
    return tuple(t.to(dev) for t in ts)


def num_sms(dev) -> int:
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count if dev == "cuda" else 2


class Guarded:
    """An output [rows, cols] at row pitch ld inside a sentinel-filled buffer with ``guard`` sentinel elements before and after it.  The
    guard keeps the output 16-byte aligned, as the kernels' vector accesses require."""

    def __init__(self, dev, rows, cols, ld, dtype, guard=64, init=None):
        self.rows, self.cols, self.ld, self.guard = rows, cols, ld, guard
        ity, self.sent = (torch.int16, BF16_SENT) if dtype == torch.bfloat16 else (torch.int32, F32_SENT)
        self.raw = torch.full((rows * ld + 2 * guard,), self.sent, dtype=ity, device=dev)
        self.t = self.raw[guard: guard + rows * ld].view(dtype).view(rows, ld)
        if init is not None:
            self.value()[:] = init.view(rows, cols).to(dev)

    @staticmethod
    def vec(dev, n, dtype=torch.float32, init=None):
        return Guarded(dev, 1, n, n, dtype, init=init)

    def ptr(self):
        return _p(self.t)

    def value(self):
        return self.t[:, : self.cols]

    def flat(self):
        return self.value().reshape(-1)

    def check_sentinels(self, what):
        r = self.raw.cpu()
        g = self.guard
        assert (r[:g] == self.sent).all() and (r[g + self.rows * self.ld:] == self.sent).all(), f"{what}: store outside the output"
        body = r[g: g + self.rows * self.ld].view(self.rows, self.ld)
        assert (body[:, self.cols:] == self.sent).all(), f"{what}: store into the padding columns"


def check(name: str, got, ref: E) -> None:
    got = got.detach().double().cpu().reshape(ref.v.shape)
    err = (got - ref.v).abs()
    tol = ref.tol()
    bad = ~(err <= tol)
    if bad.any():
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements beyond the bound; first at flat index {i}: "
                             f"got {got.reshape(-1)[i].item()!r}, oracle {ref.v.reshape(-1)[i].item()!r}, bound {tol.reshape(-1)[i].item():.3g}")


def check_exact(name: str, got, ref) -> None:
    got = got.detach().cpu()
    ref = ref.detach().cpu().to(got.dtype).reshape(got.shape)
    same = (got == ref) | (got.isnan() & ref.isnan())
    if not bool(same.all()):
        i = int((~same).reshape(-1).nonzero()[0])
        raise AssertionError(f"{name}: {int((~same).sum())} of {same.numel()} elements differ; first at flat index {i}: "
                             f"got {got.reshape(-1)[i].item()!r}, expected {ref.reshape(-1)[i].item()!r}")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def exact_bf16(shape, gen, k=8):
    """bf16 values j / 8, |j| <= k: every fp32 sum of up to 2^17 of them (and of their products) is exact."""
    return (torch.randint(-k, k + 1, shape, generator=gen).double() / 8).bfloat16()


def rand_bf16(shape, gen, scale=1.0, relu=False):
    x = torch.randn(shape, generator=gen) * scale
    return (x.relu() if relu else x).bfloat16()


def strided(dev, x: torch.Tensor, pad: int):
    """x [rows, cols] copied into a [rows, cols + pad] buffer whose padding is NaN: (buffer, row pitch)."""
    rows, cols = x.shape
    buf = torch.full((rows, cols + pad), float("nan"), dtype=x.dtype)
    buf[:, :cols] = x
    return buf.to(dev), cols + pad


# ---------------------------------------------------------------------------------------------------------------------------------------
# colstats:  S1[n] += sum_b u[b, n],  S2[n] += sum_b u[b, n] v[b, n]

COLSTATS_N = [8, 16, 24, 40, 64, 504, 512, 1024, 2048]


def rows_par(N):
    return 256 // (N // 8)


def colstats_batches(N, big=True):
    rp = rows_par(N)
    out = [1, rp - 1, rp + 1, 4097] + ([65537] if big else [])
    return sorted({b for b in out if b >= 1})


def _colstats(lib, dev, u, v, B, N, ldu, ldv, S1, S2):
    rc = lib.dr_cuda_colstats(_p(u), _p(v), B, N, ldu, ldv, S1.ptr(), S2.ptr() if S2 is not None else None, _s())
    assert rc == 0, rc
    _sync()


def colstats_case(dev, N, B, seed=0):
    lib = _lib()
    g = _gen(seed * 1000 + N * 7 + B)
    depth = D.colsum_depth(B, N)
    # (1) exact inputs, v != u, both strided, accumulating into non-zero sums: the float64 sum exactly
    u, v = exact_bf16((B, N), g), exact_bf16((B, N), g)
    S10, S20 = exact_bf16((N,), g).float() * 4, exact_bf16((N,), g).float()
    ub, ldu = strided(dev, u, 8)
    vb, ldv = strided(dev, v, 24)
    S1, S2 = Guarded.vec(dev, N, init=S10), Guarded.vec(dev, N, init=S20)
    _colstats(lib, dev, ub, vb, B, N, ldu, ldv, S1, S2)
    check_exact(f"colstats exact N={N} B={B} S1", S1.flat(), S10.double() + u.double().sum(0))
    check_exact(f"colstats exact N={N} B={B} S2", S2.flat(), S20.double() + (u.double() * v.double()).sum(0))
    S1.check_sentinels("colstats S1"); S2.check_sentinels("colstats S2")
    # (2) random inputs, v = u (the BatchNorm forward sums), strided: the depth bound
    a = rand_bf16((B, N), g, 2.0, relu=True)
    ab, lda = strided(dev, a, 16)
    S10 = torch.randn(N, generator=g)
    S20 = torch.rand(N, generator=g) * 3
    S1, S2 = Guarded.vec(dev, N, init=S10), Guarded.vec(dev, N, init=S20)
    _colstats(lib, dev, ab, ab, B, N, lda, lda, S1, S2)
    A = D.exact(a)
    check(f"colstats N={N} B={B} S1", S1.flat(), D.tree_sum(A, depth, init=D.exact(S10)))
    check(f"colstats N={N} B={B} S2", S2.flat(), D.tree_sum(D.mul_exact(A, A), depth, init=D.exact(S20)))
    S1.check_sentinels("colstats S1"); S2.check_sentinels("colstats S2")
    # (3) S2 = null (the bias-gradient sums): S1 only, exact
    S10 = exact_bf16((N,), g).float()
    S1 = Guarded.vec(dev, N, init=S10)
    _colstats(lib, dev, ub, None, B, N, ldu, 0, S1, None)
    check_exact(f"colstats S2=null N={N} B={B} S1", S1.flat(), S10.double() + u.double().sum(0))
    S1.check_sentinels("colstats S1 (S2 null)")


def colstats_rejects_case(dev):
    lib = _lib()
    buf = torch.zeros(64, 4096, dtype=torch.bfloat16, device=dev)
    S = torch.zeros(4096, device=dev)
    for N in (12, 2056, 4):
        assert lib.dr_cuda_colstats(_p(buf), _p(buf), 64, N, N, N, _p(S), _p(S), _s()) == -2, N
        assert lib.dr_cuda_bn_bwd_apply_v2(_p(buf), _p(buf), 64, N, N, _p(S), _p(S), _p(S), _p(S), _p(S), _p(buf), 1, _p(S), _s()) == -2, N
    _sync()
    assert bool((S == 0).all())


# ---------------------------------------------------------------------------------------------------------------------------------------
# BatchNorm forward: finalize (last bottom layer) and fold (into the next Linear), training and eval

EPS, MOM = 1e-3, 0.99


def bn_activation(B, K, gen):
    """[B, K] bf16 activations: a dead ReLU column (all 0), a constant non-zero column, a column with mean / std = 64, the rest ReLU'd
    random values."""
    a = rand_bf16((B, K), gen, 1.5, relu=True)
    a[:, 0] = 0
    if K > 1:
        a[:, 1] = 0.75
    if K > 2:
        a[:, 2] = torch.where(torch.arange(B) % 2 == 0, 63.0, 65.0).bfloat16() if B > 1 else 64.0
    return a


def _sums(a):
    """fp32 S1, S2 of the bf16 activations, as the kernel receives them."""
    x = a.double()
    return x.sum(0).float(), (x * x).sum(0).float()


def _bn_params(K, gen):
    return (torch.rand(K, generator=gen) + 0.5), torch.randn(K, generator=gen) * 0.2


def _check_bn_out(tag, outs, ref, K):
    for nm in ("mean", "rstd", "scale", "shift"):
        check(f"{tag} {nm}", outs[nm].flat(), ref[nm])
        outs[nm].check_sentinels(f"{tag} {nm}")


def bn_forward_case(dev, kind, K, B, Nn=1, Kp=None, seed=0):
    """kind "finalize" or "fold": three training calls (each against the oracle restarted from the kernel's running statistics), then
    two eval calls that must read the running statistics, not the batch sums they are given."""
    lib = _lib()
    g = _gen(seed + 31 * K + B)
    Kp = Kp or K
    gamma, beta = _bn_params(K, g)
    gd, bd = gamma.to(dev), beta.to(dev)
    rm = Guarded.vec(dev, K, init=torch.randn(K, generator=g) * 0.1)
    rv = Guarded.vec(dev, K, init=torch.rand(K, generator=g) + 0.5)
    Wn = torch.randn(Nn, Kp, generator=g) * 0.2
    Wn[:, K:] = 5.0                                       # padding columns: must neither reach W' nor b'
    bn = torch.randn(Nn, generator=g) * 0.1
    Wnd, bnd = Wn.to(dev), bn.to(dev)
    for step, training in enumerate((True, True, True, False, False)):
        a = bn_activation(B, K, g) if step % 2 == 0 else rand_bf16((B, K), g, 3.0, relu=True)
        S1v, S2v = _sums(a)
        S1, S2 = Guarded.vec(dev, K, init=S1v), Guarded.vec(dev, K, init=S2v)
        outs = {nm: Guarded.vec(dev, K) for nm in ("mean", "rstd", "scale", "shift")}
        rm0, rv0 = rm.flat().clone(), rv.flat().clone()
        ref = D.bn_forward(D.exact(S1v), D.exact(S2v), B, D.exact(gamma.double()), D.exact(beta.double()), EPS, MOM, D.exact(rm0),
                           D.exact(rv0), training)
        tag = f"bn_{kind} {'train' if training else 'eval'} call {step + 1} K={K} B={B}"
        if kind == "finalize":
            rc = lib.dr_cuda_bn_finalize(S1.ptr(), S2.ptr(), K, B, _p(gd), _p(bd), EPS, MOM, rm.ptr(), rv.ptr(), outs["mean"].ptr(),
                                         outs["rstd"].ptr(), outs["scale"].ptr(), outs["shift"].ptr(), int(training), _s())
        else:
            Wf = Guarded(dev, Nn, Kp, Kp, torch.bfloat16)
            bf = Guarded.vec(dev, Nn)
            rc = lib.dr_cuda_bn_fold(S1.ptr(), S2.ptr(), K, B, _p(gd), _p(bd), EPS, MOM, rm.ptr(), rv.ptr(), outs["mean"].ptr(), outs["rstd"].ptr(),
                                     outs["scale"].ptr(), outs["shift"].ptr(), int(training), _p(Wnd), _p(bnd), Nn, Kp, Wf.ptr(), bf.ptr(), _s())
        assert rc == 0
        _sync()
        _check_bn_out(tag, outs, ref, K)
        if training:
            check(f"{tag} running_mean", rm.flat(), ref["running_mean"])
            check(f"{tag} running_var", rv.flat(), ref["running_var"])
        else:
            check_exact(f"{tag} running_mean untouched", rm.flat(), rm0)
            check_exact(f"{tag} running_var untouched", rv.flat(), rv0)
        rm.check_sentinels(f"{tag} running_mean"); rv.check_sentinels(f"{tag} running_var")
        if kind == "finalize":           # the sums are re-zeroed for the next step in training, left alone in eval
            check_exact(f"{tag} S1", S1.flat(), torch.zeros(K) if training else S1v)
            check_exact(f"{tag} S2", S2.flat(), torch.zeros(K) if training else S2v)
        else:                            # the fold never writes the sums
            check_exact(f"{tag} S1", S1.flat(), S1v)
            check_exact(f"{tag} S2", S2.flat(), S2v)
            rWf, rbf = D.bn_fold(D.exact(Wn), D.exact(bn), ref["scale"], ref["shift"], K, Kp)
            check(f"{tag} W'", Wf.value(), rWf)
            assert bool((Wf.value()[:, K:].float() == 0).all()), f"{tag}: W' padding columns not 0"
            check(f"{tag} b'", bf.flat(), rbf)
            Wf.check_sentinels(f"{tag} W'"); bf.check_sentinels(f"{tag} b'")
        if training and step % 2 == 0:   # the dead ReLU column: mean exactly 0 (the constant and mean/std = 64 columns are inside the bounds)
            check_exact(f"{tag} dead column mean", outs["mean"].flat()[:1], torch.zeros(1))


# ---------------------------------------------------------------------------------------------------------------------------------------
# BatchNorm apply (the last bottom layer's normalised output)

def bn_apply_case(dev, N, B, seed=0):
    lib = _lib()
    g = _gen(seed + 17 * N + B)
    a = rand_bf16((B, N), g, 2.0, relu=True)
    scale, shift = torch.rand(N, generator=g) * 3 + 0.1, torch.randn(N, generator=g)
    ab, lda = strided(dev, a, 8)
    y = Guarded(dev, B, N, N + 24, torch.bfloat16)
    scd, shd = on(dev, scale, shift)
    assert lib.dr_cuda_bn_apply(_p(ab), B, N, lda, _p(scd), _p(shd), y.ptr(), N + 24, _s()) == 0
    _sync()
    check(f"bn_apply N={N} B={B}", y.value(), D.bn_apply(D.exact(a), D.exact(scale), D.exact(shift)))
    y.check_sentinels(f"bn_apply N={N} B={B}")


# ---------------------------------------------------------------------------------------------------------------------------------------
# BatchNorm backward: finalize (dgamma, dbeta, c1, c2 from the sums) and apply (v1, and v2 with the fused bias gradient)

def bn_bwd_finalize_case(dev, N, B, gas, seed=0):
    lib = _lib()
    g = _gen(seed + 13 * N + B)
    dy, a = rand_bf16((B, N), g, 0.1), rand_bf16((B, N), g, 2.0, relu=True)
    S1v = dy.double().sum(0).float()
    S2v = (dy.double() * a.double()).sum(0).float()
    mean, rstd = a.double().mean(0).float(), (a.double().var(0, unbiased=False) + EPS).rsqrt().float()
    dg0, db0 = torch.randn(N, generator=g), torch.randn(N, generator=g)
    S1, S2 = Guarded.vec(dev, N, init=S1v), Guarded.vec(dev, N, init=S2v)
    dgamma, dbeta = Guarded.vec(dev, N, init=dg0), Guarded.vec(dev, N, init=db0)
    c1, c2 = Guarded.vec(dev, N), Guarded.vec(dev, N)
    md, rd = on(dev, mean, rstd)
    assert lib.dr_cuda_bn_bwd_finalize(S1.ptr(), S2.ptr(), N, B, _p(md), _p(rd), dgamma.ptr(), dbeta.ptr(), c1.ptr(), c2.ptr(),
                                       gas, _s()) == 0
    _sync()
    ref = D.bn_bwd_finalize(D.exact(S1v), D.exact(S2v), B, D.exact(mean), D.exact(rstd), D.exact(dg0), D.exact(db0), gas)
    tag = f"bn_bwd_finalize N={N} B={B} scale={gas}"
    for nm, buf in (("dgamma", dgamma), ("dbeta", dbeta), ("c1", c1), ("c2", c2)):
        check(f"{tag} {nm}", buf.flat(), ref[nm])
        buf.check_sentinels(f"{tag} {nm}")
    check_exact(f"{tag} S1 re-zeroed", S1.flat(), torch.zeros(N))
    check_exact(f"{tag} S2 re-zeroed", S2.flat(), torch.zeros(N))


def bn_bwd_batches(N, big=True):
    rp = rows_par(N)
    out = [1, rp - 1 if rp % 2 == 0 else rp - 2, rp + 1, 2 * rp + 3, 4097] + ([65537] if big and N <= 64 else [])
    return sorted({b for b in out if b >= 1})


def bn_bwd_apply_case(dev, N, B, version, relu_mask, with_dbias, seed=0):
    """version 1 (k_bn_bwd_apply) or 2 (k_bn_bwd_apply_v2, dbias null or not).  a holds exact zeros (the ReLU tie a == 0)."""
    lib = _lib()
    g = _gen(seed + 11 * N + B + 5 * version + relu_mask)
    tag = f"bn_bwd_apply_v{version} N={N} B={B} relu_mask={relu_mask} dbias={'on' if with_dbias else 'null'}"
    ld = N + 8

    def run(dy, a, scale, mean, rstd, c1, c2, db0):
        dyb, _ = strided(dev, dy, 8)
        ab, _ = strided(dev, a, 8)
        da = Guarded(dev, B, N, ld, torch.bfloat16)
        dbias = Guarded.vec(dev, N, init=db0) if with_dbias else None
        params = on(dev, scale, mean, rstd, c1, c2)
        args = [_p(dyb), _p(ab), B, N, ld] + [_p(t) for t in params] + [da.ptr(), relu_mask]
        if version == 1:
            rc = lib.dr_cuda_bn_bwd_apply(*args, _s())
        else:
            rc = lib.dr_cuda_bn_bwd_apply_v2(*args, dbias.ptr() if dbias is not None else None, _s())
        assert rc == 0
        _sync()
        da.check_sentinels(f"{tag} da")
        if dbias is not None:
            dbias.check_sentinels(f"{tag} dbias")
        return da, dbias

    a = rand_bf16((B, N), g, 1.0, relu=True)               # about half the entries are exactly 0
    # (1) exact: scale 1, c1 = c2 = 0 make da = dy (masked), so dbias is an exact sum and da equals dy bit for bit
    dy = exact_bf16((B, N), g)
    one, zero = torch.ones(N), torch.zeros(N)
    db0 = exact_bf16((N,), g).float()
    da, dbias = run(dy, a, one, torch.randn(N, generator=g), torch.rand(N, generator=g) + 0.5, zero, zero, db0)
    keep = (a.float() > 0) if relu_mask else torch.ones(B, N, dtype=torch.bool)
    ref = torch.where(keep, dy.float(), torch.zeros(()))
    check_exact(f"{tag} exact da", da.value().float(), ref)
    if dbias is not None:
        check_exact(f"{tag} exact dbias", dbias.flat(), db0.double() + ref.double().sum(0))
    # (2) random: the bound of the transcription
    dy = rand_bf16((B, N), g, 0.1)
    scale, mean, rstd = torch.rand(N, generator=g) + 0.5, torch.rand(N, generator=g), torch.rand(N, generator=g) * 2 + 0.5
    c1, c2 = torch.randn(N, generator=g) * 0.05, torch.randn(N, generator=g) * 0.05
    db0 = torch.randn(N, generator=g)
    da, dbias = run(dy, a, scale, mean, rstd, c1, c2, db0)
    gref, _ = D.bn_bwd_apply(D.exact(dy), D.exact(a), D.exact(scale), D.exact(mean), D.exact(rstd), D.exact(c1), D.exact(c2), bool(relu_mask))
    check(f"{tag} da", da.value(), D.bf16(gref))
    if dbias is not None:
        check(f"{tag} dbias", dbias.flat(), D.tree_sum(gref, D.colsum_depth(B, N), init=D.exact(db0)))


# ---------------------------------------------------------------------------------------------------------------------------------------
# dW fix-up of a Linear whose input is a folded BatchNorm

def dw_fixup_case(dev, N, K, Kp, seed=0):
    lib = _lib()
    g = _gen(seed + N + 3 * Kp)
    G = torch.randn(N, Kp, generator=g)
    db, s, t = torch.randn(N, generator=g), torch.rand(K, generator=g) + 0.5, torch.randn(K, generator=g)
    dW = Guarded(dev, N, Kp, Kp, torch.float32, init=G)
    dbd, sd, td = on(dev, db, s, t)
    assert lib.dr_cuda_dw_fixup(dW.ptr(), _p(dbd), _p(sd), _p(td), N, K, Kp, _s()) == 0
    _sync()
    check(f"dw_fixup N={N} K={K} Kp={Kp}", dW.value(), D.dw_fixup(D.exact(G), D.exact(db), D.exact(s), D.exact(t), K, Kp))
    assert bool((dW.value()[:, K:] == 0).all()), "dw_fixup: padding columns not 0"
    dW.check_sentinels("dw_fixup")


# ---------------------------------------------------------------------------------------------------------------------------------------
# logit head

HEAD_K = [256, 512, 1024]


GRID_TAIL = "8grid+1"
HEAD_B = [1, 7, 9, GRID_TAIL]       # GRID_TAIL: one row more than 8 warps x the head's largest grid, resolved when the case runs


def head_batch(dev, B) -> int:
    """B of a head case; GRID_TAIL is 8 * grid + 1 with grid = 4 num_sms() blocks, so one warp gets a second row.  Resolved at run time,
    not at collection, so that collecting the GPU file needs no GPU."""
    return 8 * 4 * num_sms(dev) + 1 if B == GRID_TAIL else B


def _head_inputs(B, K, g, variant):
    h = rand_bf16((B, K), g, 1.0, relu=(variant != "saturated"))
    w = torch.randn(K, generator=g) * 0.08
    b0 = 0.1
    if variant == "scaled":
        y = torch.rand(B, generator=g)
    else:
        y = (torch.rand(B, generator=g) < 0.4).float()
    if variant == "saturated":       # rows with |z| up to 90, on the right and on the wrong side of their label
        zs = torch.tensor([90.0, -90.0, 40.0, -40.0, 17.5, -17.5, 88.0, -88.0])
        w[0], w[1] = 1.0, -1.0
        for r in range(B):
            zi = float(zs[r % len(zs)])
            h[r] = 0
            h[r, 0 if zi > 0 else 1] = abs(zi) - b0 if r % 3 else abs(zi)
            y[r] = float((r // len(zs)) % 2)
    return h, w, b0, y


def head_case(dev, K, B, variant, seed=0):
    """variant "train" (relu mask, dbias_h, inv = 1 / B, accumulating loss / dw / db), "scaled" (no relu mask, dbias_h null,
    inv = 1 / (3 B), soft labels), "saturated" (|z| up to 90) or "eval" (train = 0: dh, dw, db, dbias_h untouched)."""
    lib = _lib()
    B = head_batch(dev, B)
    g = _gen(seed + K + 7 * B + len(variant))
    h, w, b0, y = _head_inputs(B, K, g, variant)
    relu_mask = variant in ("train", "eval")
    train = variant != "eval"
    inv = 1.0 / B if variant in ("train", "eval") else 1.0 / (3 * B)
    with_dbh = variant in ("train", "eval")
    ldh = K + 8
    hb, _ = strided(dev, h, 8)
    bias = torch.tensor([b0, 0.0, 0.0, 0.0])
    loss0, dw0, db0, dbh0 = torch.tensor([0.25]), torch.randn(K, generator=g) * 0.1, torch.tensor([0.5, 0, 0, 0]), torch.randn(K, generator=g)
    prob = Guarded.vec(dev, B)
    loss = Guarded.vec(dev, 1, init=loss0)
    dh = Guarded(dev, B, K, ldh, torch.bfloat16)
    dw, db = Guarded.vec(dev, K, init=dw0), Guarded.vec(dev, 4, init=db0)
    dbh = Guarded.vec(dev, K, init=dbh0) if with_dbh else None
    wd, biasd, yd = on(dev, w, bias, y)
    rc = lib.dr_cuda_head(_p(hb), ldh, B, K, _p(wd), _p(biasd), _p(yd), inv, prob.ptr(), loss.ptr(), dh.ptr(), dw.ptr(),
                          db.ptr(), int(relu_mask), int(train), dbh.ptr() if dbh is not None else None, _s())
    assert rc == 0
    _sync()
    tag = f"head K={K} B={B} {variant}"
    ref = D.head(D.exact(h), D.exact(w.double()), b0, y, inv, relu_mask)
    depth = D.head_depth(B)
    check(f"{tag} prob", prob.flat(), ref["p"])
    check(f"{tag} loss", loss.flat(), _sum1(ref["loss"], depth, loss0))
    for buf, nm in ((prob, "prob"), (loss, "loss"), (dh, "dh"), (dw, "dw"), (db, "db")):
        buf.check_sentinels(f"{tag} {nm}")
    if not train:
        assert bool((dh.raw == dh.sent).all()), f"{tag}: dh written with train = 0"
        check_exact(f"{tag} dw untouched", dw.flat(), dw0)
        check_exact(f"{tag} db untouched", db.flat(), db0)
        check_exact(f"{tag} dbias_h untouched", dbh.flat(), dbh0)
        return
    check(f"{tag} dh", dh.value(), D.bf16(ref["dh"]))
    check(f"{tag} dw", dw.flat(), D.tree_sum(ref["dw"], depth, init=D.exact(dw0)))
    check(f"{tag} db", db.flat()[:1], _sum1(ref["dz"], depth, db0[:1]))
    check_exact(f"{tag} db[1:]", db.flat()[1:], db0[1:])
    if dbh is not None:
        check(f"{tag} dbias_h", dbh.flat(), D.tree_sum(ref["dh"], depth, init=D.exact(dbh0)))
        dbh.check_sentinels(f"{tag} dbias_h")


def _sum1(terms: E, depth: int, init: torch.Tensor) -> E:
    s = D.tree_sum(terms, depth, init=D.exact(init[0].double()))
    return E(s.v.reshape(1), s.e.reshape(1))


def head_rejects_case(dev):
    lib = _lib()
    z = torch.zeros(64, 128, dtype=torch.bfloat16, device=dev)
    f = torch.zeros(256, device=dev)
    assert lib.dr_cuda_head(_p(z), 128, 64, 128, _p(f), _p(f), _p(f), 1.0 / 64, _p(f), _p(f), _p(z), _p(f), _p(f), 1, 1, _p(f), _s()) == -2
    _sync()


# ---------------------------------------------------------------------------------------------------------------------------------------
# weight packing and input cast: round to nearest even, bit for bit

def _rne_values(shape, g):
    """Random fp32 values plus exact bf16 ties (1 + 2^-8 rounds down to even, 1 + 3 2^-8 up) and a spread of magnitudes."""
    x = torch.randn(shape, generator=g) * torch.exp2(torch.randint(-20, 20, shape, generator=g).float())
    flat = x.view(-1)
    ties = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 3 * 2 ** -9 + 2 ** -17, 65504.0, -0.0, 0.0, 2.0 ** 100])
    n = min(flat.numel(), ties.numel())
    flat[:n] = ties[:n]
    return x


PACK_SHAPES = [(1, 13), (13, 367), (367, 16), (16, 1), (367, 367), (1, 1)]


def pack_weights_case(dev, N, Kp, ldt_pad, with_t=True, seed=0):
    lib = _lib()
    g = _gen(seed + N * 5 + Kp)
    w = _rne_values((N, Kp), g)
    ldt = N + ldt_pad
    wb = Guarded(dev, N, Kp, Kp, torch.bfloat16)
    wt = Guarded(dev, Kp, ldt, ldt, torch.bfloat16) if with_t else None
    wd, = on(dev, w)
    assert lib.dr_cuda_pack_weights(_p(wd), N, Kp, wb.ptr(), wt.ptr() if wt is not None else None, ldt, _s()) == 0
    _sync()
    tag = f"pack_weights N={N} Kp={Kp} ldt={ldt if with_t else 'null'}"
    check_exact(f"{tag} W bits", wb.value().view(torch.int16), w.bfloat16().view(torch.int16))
    wb.check_sentinels(f"{tag} W")
    if wt is not None:
        ref = torch.zeros(Kp, ldt, dtype=torch.bfloat16)
        ref[:, :N] = w.t().bfloat16()
        check_exact(f"{tag} W^T bits", wt.value().view(torch.int16), ref.view(torch.int16))
        wt.check_sentinels(f"{tag} W^T")


CAST_SHAPES = [(1, 13, 16), (13, 1, 8), (367, 13, 32), (1, 16, 16), (367, 16, 35)]


def cast_pad_case(dev, B, Cdim, Cp, seed=0):
    lib = _lib()
    g = _gen(seed + B + Cdim + Cp)
    x = _rne_values((B, Cdim), g)
    y = Guarded(dev, B, Cp, Cp, torch.bfloat16)
    xd, = on(dev, x)
    assert lib.dr_cuda_cast_pad(_p(xd), B, Cdim, y.ptr(), Cp, _s()) == 0
    _sync()
    check_exact(f"cast_pad B={B} C={Cdim} Cp={Cp}", y.value().view(torch.int16), D.cast_pad(x, Cp).view(torch.int16))
    y.check_sentinels("cast_pad")


# ---------------------------------------------------------------------------------------------------------------------------------------
# the DLRM step, stage by stage

CARDS = [50, 1000, 7, 300] + [97] * 22


def gemm_ref(A: torch.Tensor, W: torch.Tensor, bias=None, relu=False, mask=None) -> E:
    """fp32-accumulated A [M, K] W [N, K]^T (+ bias)(ReLU)(* relu'(mask)) of bf16 operands: the bound of tests/test_gpu_wgmma_edges.py,
    |v - ref| <= 2 K u (|A| |W|^T + |bias|), before any bf16 store."""
    a, w = A.double().cpu(), W.double().cpu()
    v, av = a @ w.t(), a.abs() @ w.abs().t()
    if bias is not None:
        b = bias.double().cpu()
        v, av = v + b, av + b.abs()
    r = E(v, a.shape[1] * U * av)
    if relu:
        r = r.maximum(0.0)
    if mask is not None:
        r = r.where(mask.cpu() > 0, E(torch.zeros_like(r.v)))
    return r


def gemm_dw_ref(dY: torch.Tensor, X: torch.Tensor) -> E:
    """dW = dY^T X accumulated in fp32 over the batch."""
    d, x = dY.double().cpu(), X.double().cpu()
    return E(d.t() @ x, d.shape[0] * U * (d.abs().t() @ x.abs()))


def epilogue_sum(rounded: torch.Tensor, weights=None, nround=1) -> E:
    """A column sum the GEMM epilogue takes of its fp32 values before their bf16 store, compared against the stored bf16 values
    ``rounded`` (times ``weights``): each term may differ by ``nround`` bf16 roundings (2 for a square), plus the epilogue's reduction
    depth (tests/test_gpu_wgmma_edges.py)."""
    x = rounded.double().cpu()
    t = x if weights is None else x * weights.double().cpu()
    m_tiles = -(-x.shape[0] // 128)
    return E(t.sum(0), (nround * D.UB + (m_tiles + 14) * U) * t.abs().sum(0))


def _pairs(f):
    F = f.shape[1]
    i, j = torch.tril_indices(F, F, -1)
    return (f[:, i] * f[:, j]).sum(-1), (f[:, i].abs() * f[:, j].abs()).sum(-1), i, j


class Snapshot:
    """What a step reads before it changes it: parameters, BatchNorm running statistics, the batch's bf16 embedding rows."""

    def __init__(self, eng):
        self.params = eng.params.detach().clone().cpu()
        self.views = eng.views
        self.running = [(L.running_mean.detach().clone().cpu(), L.running_var.detach().clone().cpu()) for L in eng.bot]
        ids = eng.ids.detach()
        self.emb = torch.stack([eng.tables[t].lookup(ids[t], out_dtype=torch.bfloat16).cpu() for t in range(eng.T)])   # [T, B, D]

    def p(self, name):
        o, n = self.views[name]
        return self.params[o:o + n]


def _cpu(t):
    return t.detach().cpu()


def check_forward(eng, snap: Snapshot, train: bool, tag: str) -> None:
    cfg, B = eng.cfg, eng.B
    t = f"{tag} forward"
    x0 = _cpu(eng.x0)
    check_exact(f"{t} x0", x0.view(torch.int16), D.cast_pad(_cpu(eng.dense_in), x0.shape[1]).view(torch.int16))
    nb = len(eng.bot)
    x = x0
    for i, L in enumerate(eng.bot):
        W = snap.p(L.name + "/kernel").view(L.N, L.Kp)
        if i == 0:
            w, bias = W.bfloat16(), snap.p(L.name + "/bias")
        else:
            w, bias = _cpu(L.wf_bf16), _cpu(L.bf)
        a = _cpu(L.a)
        check(f"{t} bot[{i}].a", a, D.bf16(gemm_ref(x, w, bias, relu=True)))
        gamma, beta = D.exact(snap.p(L.name + "/bn_gamma").double()), D.exact(snap.p(L.name + "/bn_beta").double())
        rm0, rv0 = snap.running[i]
        A = D.exact(a)
        fused = train and L.N > 32 and not cfg.gemm_v1
        if train:
            if i + 1 < nb:           # the fold leaves the sums in place: check them, then use them as the fold's input
                if fused:
                    check(f"{t} bot[{i}].S1 (epilogue)", _cpu(L.S1), epilogue_sum(a))
                    check(f"{t} bot[{i}].S2 (epilogue)", _cpu(L.S2), epilogue_sum(a, weights=a, nround=2))
                else:
                    d = D.colsum_depth(B, L.N)
                    check(f"{t} bot[{i}].S1", _cpu(L.S1), D.tree_sum(A, d))
                    check(f"{t} bot[{i}].S2", _cpu(L.S2), D.tree_sum(D.mul_exact(A, A), d))
                S1, S2 = D.exact(_cpu(L.S1)), D.exact(_cpu(L.S2))
            else:                    # k_bn_finalize re-zeroes them: the oracle sums the stored activations itself
                assert bool((_cpu(L.S1) == 0).all() and (_cpu(L.S2) == 0).all()), f"{t} bot[{i}]: sums not re-zeroed"
                d = D.colsum_depth(B, L.N)
                S1, S2 = D.tree_sum(A, d), D.tree_sum(D.mul_exact(A, A), d)
        else:
            S1 = S2 = None
        ref = D.bn_forward(S1, S2, B, gamma, beta, cfg.bn_eps, cfg.bn_momentum, D.exact(rm0), D.exact(rv0), train)
        for nm in ("mean", "rstd", "scale", "shift"):
            check(f"{t} bot[{i}].{nm}", _cpu(getattr(L, nm)), ref[nm])
        if train:
            check(f"{t} bot[{i}].running_mean", _cpu(L.running_mean), ref["running_mean"])
            check(f"{t} bot[{i}].running_var", _cpu(L.running_var), ref["running_var"])
        else:
            check_exact(f"{t} bot[{i}].running_mean untouched", _cpu(L.running_mean), rm0)
            check_exact(f"{t} bot[{i}].running_var untouched", _cpu(L.running_var), rv0)
        if i + 1 < nb:
            Ln = eng.bot[i + 1]
            Wn = snap.p(Ln.name + "/kernel").view(Ln.N, Ln.Kp)
            rWf, rbf = D.bn_fold(D.exact(Wn.double()), D.exact(snap.p(Ln.name + "/bias").double()), ref["scale"], ref["shift"], L.N, Ln.Kp)
            check(f"{t} bot[{i + 1}].wf_bf16", _cpu(Ln.wf_bf16), rWf)
            check(f"{t} bot[{i + 1}].bf", _cpu(Ln.bf), rbf)
            x = a
        else:
            y = _cpu(L.y)
            check(f"{t} bot[{i}].y", y, D.bn_apply(A, D.exact(_cpu(L.scale)), D.exact(_cpu(L.shift))))
            x = y
    # interaction: Z = [y | strict lower triangle of the Gram matrix of (y, emb_0 .. emb_T-1)], zero padded
    f = torch.cat([x.double()[:, None, :], snap.emb.double().permute(1, 0, 2)], 1)
    pv, pa, _, _ = _pairs(f)
    Z = _cpu(eng.Z)
    Dm = eng.D
    check_exact(f"{t} Z[:, :D]", Z[:, :Dm].view(torch.int16), x.view(torch.int16))
    check(f"{t} Z pairs", Z[:, Dm: Dm + pv.shape[1]], D.bf16(E(pv, Dm * U * pa)))
    assert bool((Z[:, eng.inter_dim:].float() == 0).all()), f"{t}: Z padding not 0"
    x = Z
    for i, L in enumerate(eng.top):
        W = snap.p(L.name + "/kernel").view(L.N, L.Kp).bfloat16()
        a = _cpu(L.a)
        check(f"{t} top[{i}].a", a, D.bf16(gemm_ref(x, W, snap.p(L.name + "/bias"), relu=True)))
        x = a
    inv = 1.0 / (B * eng.world)
    href = D.head(D.exact(x), D.exact(snap.p("logits/kernel").double()), float(snap.p("logits/bias")[0]), _cpu(eng.labels), inv)
    check(f"{t} prob", _cpu(eng.prob), href["p"])
    check(f"{t} loss", _cpu(eng.loss), _sum1(href["loss"], D.head_depth(B), torch.zeros(1)))
    return href


def check_backward(eng, snap: Snapshot, href, tag: str) -> None:
    cfg, B = eng.cfg, eng.B
    v2 = not cfg.gemm_v1
    t = f"{tag} backward"
    depth = D.head_depth(B)
    grads = _cpu(eng.grads)

    def g(name):
        o, n = eng.views[name]
        return grads[o:o + n]

    hL = eng.top[-1]
    check(f"{t} top[-1].da (head dh)", _cpu(hL.da), D.bf16(href["dh"]))
    check(f"{t} logits/kernel grad", g("logits/kernel"), D.tree_sum(href["dw"], depth))
    check(f"{t} logits/bias grad", g("logits/bias")[:1], _sum1(href["dz"], depth, torch.zeros(1)))
    check_exact(f"{t} logits/bias grad padding", g("logits/bias")[1:], torch.zeros(3))
    check(f"{t} {hL.name}/bias grad (head dbias_h)", g(hL.name + "/bias"), D.tree_sum(href["dh"], depth))
    for i in range(len(eng.top) - 1, -1, -1):
        L = eng.top[i]
        da = _cpu(L.da)
        x = _cpu(eng.top[i - 1].a) if i > 0 else _cpu(eng.Z)
        check(f"{t} {L.name}/kernel grad", g(L.name + "/kernel").view(L.N, L.Kp), gemm_dw_ref(da, x))
        Wt = snap.p(L.name + "/kernel").view(L.N, L.Kp).bfloat16().t()              # W^T [Kp, N]
        if i > 0:
            P = eng.top[i - 1]
            pa = _cpu(P.a)
            vals = gemm_ref(da, Wt[: P.N], mask=pa)
            pda = _cpu(P.da)
            check(f"{t} top[{i - 1}].da", pda, D.bf16(vals))
            check(f"{t} {P.name}/bias grad", g(P.name + "/bias"), epilogue_sum(pda) if v2 else D.tree_sum(D.exact(pda), D.colsum_depth(B, P.N)))
        else:
            check(f"{t} dZ", _cpu(eng.dZ), D.bf16(gemm_ref(da, Wt)))
    # interaction backward: dy of the last bottom layer and demb [T, B, D]
    last = eng.bot[-1]
    dZ = _cpu(eng.dZ).double()
    f = torch.cat([_cpu(last.y).double()[:, None, :], snap.emb.double().permute(1, 0, 2)], 1)
    F, Dm = f.shape[1], eng.D
    _, _, ii, jj = _pairs(f)
    Gm = torch.zeros(B, F, F, dtype=torch.float64)
    gp = dZ[:, Dm: Dm + ii.numel()]
    Gm[:, ii, jj] = gp
    Gm[:, jj, ii] = gp
    gv, ga = Gm @ f, Gm.abs() @ f.abs()
    gv[:, 0] += dZ[:, :Dm]
    ga[:, 0] += dZ[:, :Dm].abs()
    gref = E(gv, (F + 1) * U * ga)
    check(f"{t} bot[-1].dy (interaction dx)", _cpu(last.dy), D.bf16(E(gref.v[:, 0], gref.e[:, 0])))
    check(f"{t} demb", _cpu(eng.demb).permute(1, 0, 2), D.bf16(E(gref.v[:, 1:], gref.e[:, 1:])))
    # bottom MLP backward
    nb = len(eng.bot)
    for i in range(nb - 1, -1, -1):
        L = eng.bot[i]
        dy, a = _cpu(L.dy), _cpu(L.a)
        DY, A = D.exact(dy), D.exact(a)
        from_epilogue = v2 and i < nb - 1 and L.N > 32
        if from_epilogue:    # sums of the fp32 epilogue dy; the bf16 dy is what is stored (and what k_bn_bwd_apply_v2 reads)
            S1 = epilogue_sum(dy)
            S2 = epilogue_sum(dy, weights=a)
        else:
            d = D.colsum_depth(B, L.N)
            S1, S2 = D.tree_sum(DY, d), D.tree_sum(D.mul_exact(DY, A), d)
        mean, rstd = D.exact(_cpu(L.mean)), D.exact(_cpu(L.rstd))
        zero = D.exact(torch.zeros(L.N))
        fin = D.bn_bwd_finalize(S1, S2, B, mean, rstd, zero, zero)
        check(f"{t} {L.name}/bn_gamma grad", g(L.name + "/bn_gamma"), fin["dgamma"])
        check(f"{t} {L.name}/bn_beta grad", g(L.name + "/bn_beta"), fin["dbeta"])
        check(f"{t} bot[{i}].c1", _cpu(L.c1), fin["c1"])
        check(f"{t} bot[{i}].c2", _cpu(L.c2), fin["c2"])
        graw, _ = D.bn_bwd_apply(DY, A, D.exact(_cpu(L.scale)), mean, rstd, D.exact(_cpu(L.c1)), D.exact(_cpu(L.c2)), True)
        da = _cpu(L.da)
        check(f"{t} bot[{i}].da", da, D.bf16(graw))
        check(f"{t} {L.name}/bias grad", g(L.name + "/bias"), D.tree_sum(graw, D.colsum_depth(B, L.N)))
        if i > 0:
            P = eng.bot[i - 1]
            G = gemm_dw_ref(da, _cpu(P.a))
            ref = D.dw_fixup(G, D.exact(g(L.name + "/bias")), D.exact(_cpu(P.scale)), D.exact(_cpu(P.shift)), L.K, L.Kp)
            check(f"{t} {L.name}/kernel grad (fix-up)", g(L.name + "/kernel").view(L.N, L.Kp), ref)
            Wt = snap.p(L.name + "/kernel").view(L.N, L.Kp).bfloat16().t()
            check(f"{t} bot[{i - 1}].dy", _cpu(P.dy), D.bf16(gemm_ref(da, Wt[: P.N])))
        else:
            check(f"{t} {L.name}/kernel grad", g(L.name + "/kernel").view(L.N, L.Kp), gemm_dw_ref(da, _cpu(eng.x0)))


def _batch(B, seed, dev):
    g = torch.Generator().manual_seed(seed)
    dense = torch.rand(B, 13, generator=g) * 3
    ids = torch.stack([torch.randint(0, c, (B,), generator=g) for c in CARDS])
    labels = (torch.rand(B, generator=g) < 0.3).float()
    return dense.to(dev), ids.to(dev), labels.to(dev)


def engine_step_case(dev, B, steps=3, **cfg_over):
    """One eager step checked stage by stage; the BatchNorm state after 1 and after ``steps`` steps; predict() after them in eval mode."""
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    torch.manual_seed(0)
    cfg = DLRMConfig(batch_size=B, cardinalities=CARDS, optimizer="adagrad", learning_rate=0.05, **cfg_over)
    eng = DLRMEngine(cfg)
    tag = f"B={B} {cfg_over}"
    for s in range(steps):
        eng.load_batch(*_batch(B, 40 + s, dev))
        snap = Snapshot(eng)
        eng.train_step_eager()
        _native.device_sync(eng.dev)
        if s == 0:
            href = check_forward(eng, snap, True, f"{tag} step 1")
            check_backward(eng, snap, href, f"{tag} step 1")
        elif s == steps - 1:         # BatchNorm state after the last step, from the state before it
            for i, L in enumerate(eng.bot):
                rm0, rv0 = snap.running[i]
                a = D.exact(_cpu(L.a))
                d = D.colsum_depth(B, L.N)
                S1 = D.exact(_cpu(L.S1)) if i + 1 < len(eng.bot) else D.tree_sum(a, d)
                S2 = D.exact(_cpu(L.S2)) if i + 1 < len(eng.bot) else D.tree_sum(D.mul_exact(a, a), d)
                m, var = D.bn_stats(S1, S2, B)
                check(f"{tag} step {steps} bot[{i}].running_mean", _cpu(L.running_mean), D.moving_average(D.exact(rm0), m, cfg.bn_momentum))
                check(f"{tag} step {steps} bot[{i}].running_var", _cpu(L.running_var), D.moving_average(D.exact(rv0), var, cfg.bn_momentum))
    eng.load_batch(*_batch(B, 90, dev))
    snap = Snapshot(eng)
    eng.predict()
    _native.device_sync(eng.dev)
    check_forward(eng, snap, False, f"{tag} predict after {steps} steps")


def engine_bad_head_width_case(dev):
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    cfg = DLRMConfig(batch_size=64, cardinalities=CARDS, mlp_top=(512, 384))
    eng = DLRMEngine(cfg)
    eng.load_batch(*_batch(64, 7, dev))
    try:
        eng.train_step_eager()
    except RuntimeError as e:
        assert "dr_cuda_head" in str(e), e
    else:
        raise AssertionError("a head width of 384 trained without an error")
    _native.device_sync(eng.dev)
