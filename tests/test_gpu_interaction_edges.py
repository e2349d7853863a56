"""DLRM dot interaction and FM kernels (csrc/cuda/interaction_kernels.cu) at their edges against float64 references with per-element bounds.

The operands are bf16; the reference upcasts them to float64, so the only error left is fp32 accumulation plus the bf16 output rounding:
- a pair of the dot interaction is a D-term dot product:  |Z - ref| <= 2^-8 |ref| + 2 D 2^-24 sum_d |f_i f_j|;
- a backward row sums F = T + 1 products per element (plus the x passthrough for dx):  |g - ref| <= 2^-8 |ref| + 2 (F + 1) 2^-24 (the same
  backward over |dZ| and |f|);
- FM: s = sum_t f and q = sum_t f^2 accumulate T terms, out = (s^2 - q) / 2:  |out - ref| <= 2^-8 |ref| + (2 T + 4) 2^-24 ((sum |f|)^2 + q);
  backward: demb_t (+)= dfm (s - f_t):  |g - ref| <= 2^-8 |ref| + 4 (T + 2) 2^-24 (|dfm| (sum |f| + |f_t|) + |demb_0|).
The embedding rows are a strided sample-major layout (row pitch D + 8), x has pitch D + 8, and Z is wider than its used width: its padding
columns must be exactly zero.  D = 16 runs on the tensor cores (mma.sync) unless dr_cuda_dot_set_simt(1) selects the SIMT kernels, which
also serve D = 8 and D = 32."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _lib():
    from deeprec_b200 import _native
    lib = _native.cuda()
    lib.dr_cuda_dot_set_simt.argtypes, lib.dr_cuda_dot_set_simt.restype = [C.c_int], C.c_int
    return lib


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr())


def _within(got, ref, tol, what):
    err = (got.double() - ref).abs()
    bad = err > tol
    assert not bad.any(), f"{what}: {int(bad.sum())} elements outside the bound, worst excess {(err - tol).max().item()}"


def _pairs(f):
    """f [B, F, D] float64 -> the strictly lower triangle of f f^T per sample, row-major (i > j): [B, F (F - 1) / 2]."""
    F = f.shape[1]
    i, j = torch.tril_indices(F, F, -1, device=f.device)
    return (f[:, i] * f[:, j]).sum(-1)


def _dot_case(lib, B, T, D, simt, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    F = T + 1
    n = D + F * (F - 1) // 2
    ldz = min(512, (n + 7) // 8 * 8 + 16)
    xw = torch.randn(B, D + 8, device="cuda", generator=g).bfloat16()
    ew = (torch.randn(B, T, D + 8, device="cuda", generator=g) * 0.5).bfloat16()        # sample-major, row pitch D + 8
    x, emb = xw[:, :D], ew[:, :, :D]
    Z = torch.full((B, ldz), 3.0, device="cuda", dtype=torch.bfloat16)
    lib.dr_cuda_dot_set_simt(int(simt))
    try:
        assert lib.dr_cuda_dot_interaction_fwd(_p(xw), D + 8, _p(ew), D + 8, T * (D + 8), T, D, B, _p(Z), ldz, _s()) == 0
        torch.cuda.synchronize()
        f = torch.cat([x.double().unsqueeze(1), emb.double()], 1)
        ref = torch.cat([x.double(), _pairs(f)], 1)
        absref = torch.cat([x.double().abs(), _pairs(f.abs())], 1)
        tz = 2.0 ** -8 * ref.abs() + 2 * D * U * absref
        _within(Z[:, :n], ref, tz, f"Z B={B} T={T} D={D} simt={simt}")
        assert torch.equal(Z[:, :D], x), "the x columns of Z are a copy"
        assert (Z[:, n:] == 0).all(), "padding columns of Z must be exactly zero"
        # backward
        dZ = torch.zeros(B, ldz, device="cuda", dtype=torch.bfloat16)
        dZ[:, :n] = (torch.randn(B, n, device="cuda", generator=g) * 0.1).bfloat16()
        dxw = torch.full((B, D + 8), 5.0, device="cuda", dtype=torch.bfloat16)
        demw = torch.full((B, T, D + 8), 5.0, device="cuda", dtype=torch.bfloat16)
        assert lib.dr_cuda_dot_interaction_bwd(_p(dZ), ldz, _p(xw), D + 8, _p(ew), D + 8, T * (D + 8), T, D, B, _p(dxw), D + 8, _p(demw),
                                               D + 8, T * (D + 8), _s()) == 0
        torch.cuda.synchronize()
    finally:
        lib.dr_cuda_dot_set_simt(0)
    grads = []
    for absolute in (False, True):
        fx = (x.double().abs() if absolute else x.double()).requires_grad_(True)
        fe = (emb.double().abs() if absolute else emb.double()).requires_grad_(True)
        out = torch.cat([fx, _pairs(torch.cat([fx.unsqueeze(1), fe], 1))], 1)
        dz = dZ[:, :n].double()
        out.backward(dz.abs() if absolute else dz)
        grads.append((fx.grad, fe.grad))
    (rdx, rde), (adx, ade) = grads
    tx = 2.0 ** -8 * rdx.abs() + 2 * (F + 1) * U * adx
    te = 2.0 ** -8 * rde.abs() + 2 * (F + 1) * U * ade
    _within(dxw[:, :D], rdx, tx, f"dx B={B} T={T} D={D} simt={simt}")
    _within(demw[:, :, :D], rde, te, f"demb B={B} T={T} D={D} simt={simt}")
    assert (dxw[:, D:] == 5.0).all() and (demw[:, :, D:] == 5.0).all(), "stores into the row padding"
    return (Z[:, :n], dxw[:, :D], demw[:, :, :D]), (tz, tx, te)


DOT_CASES = [(1, 1), (3, 2), (4, 15), (5, 26), (1537, 31), (1, 31), (4, 1), (1537, 2), (5, 15), (3, 26), (1537, 26)]


@pytest.mark.parametrize("B,T", DOT_CASES)
def test_dot_interaction_tensor_core_and_simt_d16(B, T):
    lib = _lib()
    tc, tol = _dot_case(lib, B, T, 16, False, seed=B * 31 + T)
    si, _ = _dot_case(lib, B, T, 16, True, seed=B * 31 + T)
    # each path is within the bound of the fp64 reference, so they differ by at most twice the bound; the forward pairs are D = 16 term
    # dot products rounded once from fp32 on both paths
    for a, b, t, what in zip(tc, si, tol, ("Z", "dx", "demb")):
        assert ((a.double() - b.double()).abs() <= 2 * t).all(), what


@pytest.mark.parametrize("D", [8, 32])
@pytest.mark.parametrize("B,T", [(1, 1), (5, 15), (1537, 26), (4, 31)])
def test_dot_interaction_simt_d8_d32(B, T, D):
    if D + (T + 1) * T // 2 > 512:
        pytest.skip("Z wider than the kernels' 512-column limit")
    _dot_case(_lib(), B, T, D, True, seed=B + T + D)


@pytest.mark.parametrize("D", [8, 16, 32])
@pytest.mark.parametrize("B,T", [(1, 1), (5, 2), (1537, 26), (4, 31)])
def test_fm_forward_backward_accumulate(B, T, D):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(B + T + D)
    ew = (torch.randn(B, T, D + 8, device="cuda", generator=g) * 0.5).bfloat16()
    emb = ew[:, :, :D].double()
    ldo = D + 8
    out = torch.full((B, ldo), 5.0, device="cuda", dtype=torch.bfloat16)
    ssum = torch.empty(B, D, device="cuda")
    assert lib.dr_cuda_fm_fwd(_p(ew), D + 8, T * (D + 8), T, D, B, _p(out), ldo, _p(ssum), _s()) == 0
    torch.cuda.synchronize()
    s, q, sa = emb.sum(1), (emb * emb).sum(1), emb.abs().sum(1)
    ref = 0.5 * (s * s - q)
    _within(out[:, :D], ref, 2.0 ** -8 * ref.abs() + (2 * T + 4) * U * (sa * sa + q), f"fm out B={B} T={T} D={D}")
    assert (out[:, D:] == 5.0).all()
    assert ((ssum.double() - s).abs() <= T * U * sa).all()
    dfm = (torch.randn(B, D, device="cuda", generator=g) * 0.1).bfloat16()
    dw = (torch.randn(B, T, D + 8, device="cuda", generator=g) * 0.01).bfloat16()
    d0 = dw[:, :, :D].double().clone()
    assert lib.dr_cuda_fm_bwd(_p(dfm), D, _p(ew), D + 8, T * (D + 8), _p(ssum), T, D, B, _p(dw), D + 8, T * (D + 8), 1, _s()) == 0
    torch.cuda.synchronize()
    df = dfm.double().unsqueeze(1)
    refg = d0 + df * (s.unsqueeze(1) - emb)
    tol = 2.0 ** -8 * refg.abs() + 4 * (T + 2) * U * (df.abs() * (sa.unsqueeze(1) + emb.abs()) + d0.abs())
    _within(dw[:, :, :D], refg, tol, f"fm demb (accumulate) B={B} T={T} D={D}")
