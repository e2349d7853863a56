"""FP8 (E4M3) wgmma GEMM + quantisation kernels against fp32 references."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from deeprec_b200 import _native
    return _native.cuda()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("M,N,K", [(1, 512, 368), (256, 256, 512), (2048, 512, 479), (777, 64, 256), (4096, 1024, 1024), (33, 16, 128)])
@pytest.mark.parametrize("out_fp8", [0, 1])
def test_fp8_gemm_matches_dequantised_reference(M, N, K, out_fp8):
    torch.manual_seed(0)
    lib = _lib()
    Kp = (K + 15) // 16 * 16
    x = torch.randn(M, K, device="cuda").relu()
    w = torch.randn(N, K, device="cuda") / K ** 0.5
    bias = torch.randn(N, device="cuda") * 0.1
    a_scale = float(x.abs().max()) / 448.0
    xq = torch.empty(M, Kp, dtype=torch.uint8, device="cuda")
    assert lib.dr_cuda_quantize_e4m3(_p(x), 0, M, K, K, _p(xq), Kp, 1.0 / a_scale, _s()) == 0
    wq = torch.empty(N, Kp, dtype=torch.uint8, device="cuda"); w_scale = torch.empty(N, device="cuda")
    assert lib.dr_cuda_quantize_weights_e4m3(_p(w), N, K, K, _p(wq), Kp, _p(w_scale), _s()) == 0
    # the quantisers agree with torch's e4m3 cast
    xd = xq.view(torch.float8_e4m3fn).float()[:, :K] * a_scale
    wd = wq.view(torch.float8_e4m3fn).float()[:, :K] * w_scale[:, None]
    assert (xd - x).abs().max() <= 0.07 * x.abs().max() and (wd - w).abs().max() <= 0.07 * w.abs().max()
    assert torch.equal(xq.view(torch.float8_e4m3fn)[:, :K].float(), (x / a_scale).to(torch.float8_e4m3fn).float())
    col_scale = (w_scale * a_scale).contiguous()
    ref = torch.relu(xd @ wd.t() + bias)
    out_scale = float(ref.abs().max()) / 448.0 if out_fp8 else 1.0
    out = torch.empty(M, N, dtype=torch.uint8 if out_fp8 else torch.bfloat16, device="cuda")
    assert lib.dr_cuda_gemm_fp8_tn(_p(xq), Kp, _p(wq), Kp, M, N, Kp, _p(col_scale), _p(bias), 1, _p(out), N, out_fp8, 1.0 / out_scale, _s()) == 0
    torch.cuda.synchronize()
    got = out.view(torch.float8_e4m3fn).float() * out_scale if out_fp8 else out.float()
    tol = (0.07 if out_fp8 else 1e-2) * (ref.abs().max().item() + 1e-6)
    assert (got - ref).abs().max().item() <= tol
    # and stays close to the un-quantised fp32 layer
    full = torch.relu(x @ w.t() + bias)
    assert ((got - full).norm() / (full.norm() + 1e-9)).item() < 0.08


def test_absmax():
    lib = _lib()
    x = (torch.randn(100000, device="cuda") * 3).bfloat16()
    out = torch.zeros(1, device="cuda")
    assert lib.dr_cuda_absmax_bf16(_p(x), x.numel(), _p(out), _s()) == 0
    assert out.item() == x.float().abs().max().item()
