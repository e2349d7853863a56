"""dr_cuda_det_colsum (k_det_colsum, csrc/cuda/common.cuh): the ordered reduction of per-block partials that ends every batch sum of the DLRM
step, bit for bit against the sequential fp32 oracle s = 0; s = s + ws[r] for r = 0 .. rows-1; dst + s.  Every elementwise add of the oracle
rounds once, exactly as each step of the kernel's add chain does, and the inputs mix signs and magnitudes (2^-12 .. 2^13), so a sum in any
other order (a tree, rows split between threads) gives other bits.  The workspace starts at an offset that is not 16-byte aligned and has an
odd row pitch larger than the columns it sums; dst starts non-zero, and NaN guards around it must survive.  Runs on the CUDA-on-CPU emulation
in the default tier and on an H100 under the gpu mark."""
import ctypes as C

import pytest
import torch

from deeprec_b200 import _native

ROWS = [1, 7, 256, 512, 528, 1056, 4099]
NS = [1, 16, 17, 512, 1026]
GUARD = 16
OFF = 5                                 # workspace base = buffer + 5 floats: no vector alignment


def _mixed(g, *shape):
    mag = torch.exp2(torch.randint(-12, 13, shape, generator=g).float())
    sign = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    return sign * mag * (1 + torch.rand(shape, generator=g))


def _oracle(ws, n, col, dst):
    s = torch.zeros(n)
    for r in range(ws.shape[0]):
        s = s + ws[r, col: col + n]
    return dst + s


def _case(dev, rows, n, with_dst1):
    g = torch.Generator().manual_seed(rows * 10007 + n * 2 + int(with_dst1))
    ld = 2 * n + 3                                        # odd pitch > the 2n columns summed
    ws = _mixed(g, rows, ld)
    buf = torch.cat([_mixed(g, OFF), ws.reshape(-1), _mixed(g, 7)]).to(dev)
    dsts, init = [], []
    for _ in range(2 if with_dst1 else 1):
        d0 = _mixed(g, n)
        d = torch.full((GUARD + n + GUARD,), float("nan"))
        d[GUARD: GUARD + n] = d0
        dsts.append(d.to(dev)); init.append(d0)
    p = lambda t, o: C.c_void_p(t.data_ptr() + 4 * o)
    rc = _native.cuda().dr_cuda_det_colsum(p(buf, OFF), rows, ld, n, p(dsts[0], GUARD), p(dsts[1], GUARD) if with_dst1 else None,
                                           _native.stream_ptr())
    assert rc == 0
    _native.stream_sync()
    for k, (d, d0) in enumerate(zip(dsts, init)):
        got = d.cpu()
        assert torch.equal(got[GUARD: GUARD + n], _oracle(ws, n, k * n, d0)), f"dst{k}"
        assert torch.isnan(got[:GUARD]).all() and torch.isnan(got[GUARD + n:]).all(), f"dst{k} guard written"


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("rows", ROWS)
def test_det_colsum_on_the_emulation(rows, n):
    with _native.cuda_emulation():
        _case("cpu", rows, n, with_dst1=(rows + n) % 2 == 1)


@pytest.mark.gpu
@pytest.mark.parametrize("with_dst1", [False, True])
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("rows", ROWS)
def test_det_colsum_on_the_gpu(rows, n, with_dst1):
    torch.cuda.set_device(0)
    _case("cuda", rows, n, with_dst1)
