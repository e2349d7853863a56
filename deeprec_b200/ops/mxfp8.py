"""MXFP8 (block-scaled fp8) for the MLP path: E4M3 elements with one UE8M0 power-of-two scale per 32 elements along K.  On H100 the
GEMM (dr_cuda_gemm_mxfp8_tn, csrc/cuda/gemm_wgmma.cu) issues one m64nNk32 e4m3 wgmma per 32-element scale block and promotes its product
into the fp32 accumulator with the two scales, so there is no calibration pass and no per-tensor scale to go stale when a model is
hot-swapped.

`quantize_mxfp8_reference` / `dequantize_mxfp8` are plain torch (run anywhere; the CPU tests pin the format and the scale-word layout
with them); `quantize_mxfp8` and `mxfp8_gemm` call the CUDA kernels; `MXFP8Linear` is the inference layer built from them.

Scale-word layout: rows are grouped in blocks of 128, K in blocks of 128; the uint32 of row r and k block kb sits at
``((r // 128) * num_kb + kb) * 128 + (r % 32) * 4 + (r % 128) // 32`` and its byte j is the scale of elements ``kb * 128 + 32 j .. + 31``.

Reference parity: DeepRec quantises models offline with tools/low_precision_optimize (BF16 / FP16 / INT8, SURVEY §2.9).
"""
from __future__ import annotations

import ctypes as C

import torch

E4M3_MAX = 448.0


def padded_k(k: int) -> int:
    return (k + 127) // 128 * 128


def sf_words(rows: int, kp: int) -> int:
    return (rows + 127) // 128 * (kp // 128) * 128


def _sf_index(rows: int, num_kb: int, device) -> torch.Tensor:
    """[rows, num_kb] -> flat scale-word index."""
    r = torch.arange(rows, device=device).unsqueeze(1)
    kb = torch.arange(num_kb, device=device).unsqueeze(0)
    return ((r // 128) * num_kb + kb) * 128 + (r % 32) * 4 + (r % 128) // 32


def block_exponents(x: torch.Tensor) -> torch.Tensor:
    """x [R, Kp] fp32 (Kp % 32 == 0) -> e [R, Kp / 32] int32 with 2^e >= amax / 448 (smallest such power of two, clamped to >= 2^-126)."""
    R, Kp = x.shape
    amax = x.abs().reshape(R, Kp // 32, 32).amax(dim=2)
    m, ex = torch.frexp(amax * (1.0 / E4M3_MAX))        # value = m * 2^ex, m in [0.5, 1)
    e = torch.where(m == 0.5, ex - 1, ex).to(torch.int32)
    e = torch.where(amax == 0, torch.full_like(e, -126), e)
    return e.clamp(-126, 127)


def quantize_mxfp8_reference(x: torch.Tensor):
    """x [R, C] -> (q uint8 [R, Kp] holding E4M3 bits, sf int32 [sf_words] in the scale-word layout above).  Bit-exact model of k_quantize_mxfp8."""
    R, Cc = x.shape
    Kp = padded_k(Cc)
    xf = torch.zeros(R, Kp, dtype=torch.float32, device=x.device)
    xf[:, :Cc] = x.float()
    e = block_exponents(xf)                                                  # [R, Kp / 32]
    inv = torch.ldexp(torch.ones_like(e, dtype=torch.float32), -e)           # 2^-e
    scaled = (xf.reshape(R, Kp // 32, 32) * inv.unsqueeze(2)).reshape(R, Kp)
    q = scaled.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)
    byte = (e + 127).to(torch.int64).reshape(R, Kp // 128, 4)
    word = byte[..., 0] | (byte[..., 1] << 8) | (byte[..., 2] << 16) | (byte[..., 3] << 24)
    word = torch.where(word >= 2 ** 31, word - 2 ** 32, word).to(torch.int32)
    sf = torch.zeros(sf_words(R, Kp), dtype=torch.int32, device=x.device)
    sf[_sf_index(R, Kp // 128, x.device).reshape(-1)] = word.reshape(-1)
    return q, sf


def dequantize_mxfp8(q: torch.Tensor, sf: torch.Tensor) -> torch.Tensor:
    """(q uint8 [R, Kp], sf) -> fp32 [R, Kp]: exactly the operand values the block-scaled MMA multiplies."""
    R, Kp = q.shape
    word = sf[_sf_index(R, Kp // 128, q.device)].to(torch.int64) & 0xFFFFFFFF             # [R, num_kb]
    byte = torch.stack([(word >> (8 * j)) & 0xFF for j in range(4)], dim=2).reshape(R, Kp // 32)
    scale = torch.ldexp(torch.ones(R, Kp // 32, dtype=torch.float32, device=q.device), (byte - 127).to(torch.int32))
    return (q.view(torch.float8_e4m3fn).float().reshape(R, Kp // 32, 32) * scale.unsqueeze(2)).reshape(R, Kp)


def _lib():
    from .. import _native
    return _native.cuda()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def quantize_mxfp8(x: torch.Tensor):
    """CUDA quantiser (k_quantize_mxfp8): x [R, C] fp32 / bf16 on the device -> (q uint8 [R, Kp], sf int32 [sf_words])."""
    assert x.is_cuda and x.dim() == 2 and x.stride(1) == 1 and x.dtype in (torch.float32, torch.bfloat16)
    R, Cc = x.shape
    Kp = padded_k(Cc)
    q = torch.empty(R, Kp, dtype=torch.uint8, device=x.device)
    sf = torch.zeros(sf_words(R, Kp), dtype=torch.int32, device=x.device)
    rc = _lib().dr_cuda_quantize_mxfp8(C.c_void_p(x.data_ptr()), int(x.dtype == torch.bfloat16), R, Cc, x.stride(0), C.c_void_p(q.data_ptr()), Kp,
                                       C.c_void_p(sf.data_ptr()), _stream())
    if rc != 0:
        raise RuntimeError(f"dr_cuda_quantize_mxfp8 failed: {rc}")
    return q, sf


def mxfp8_gemm(aq, sfa, bq, sfb, n: int, bias=None, relu: bool = False, max_ctas: int = 0) -> torch.Tensor:
    """out [M, N] bf16 = blockscaled(aq [M, Kp]) @ blockscaled(bq [>= N, Kp])^T (+bias)(ReLU) on the block-scaled wgmma path."""
    M, Kp = aq.shape
    assert bq.shape[1] == Kp and bq.shape[0] >= n and n % 8 == 0
    out = torch.empty(M, n, dtype=torch.bfloat16, device=aq.device)
    rc = _lib().dr_cuda_gemm_mxfp8_tn(C.c_void_p(aq.data_ptr()), C.c_void_p(sfa.data_ptr()), C.c_void_p(bq.data_ptr()), C.c_void_p(sfb.data_ptr()), M, n, Kp,
                                      C.c_void_p(bias.data_ptr()) if bias is not None else None, int(relu), C.c_void_p(out.data_ptr()), n, max_ctas,
                                      _stream())
    if rc != 0:
        raise RuntimeError(f"dr_cuda_gemm_mxfp8_tn failed: {rc}")
    return out


class MXFP8Linear(torch.nn.Module):
    """Inference Linear (+ReLU) with MXFP8 weights: the weight is quantised once, activations per call; the kernel stores bf16 (N padded to 8), returned in the input's dtype."""

    def __init__(self, linear: torch.nn.Linear, relu: bool = False):
        super().__init__()
        w = linear.weight.detach()
        self.out_features, self.in_features = w.shape
        self.np = (self.out_features + 7) // 8 * 8
        self.relu = relu
        wp = torch.zeros(self.np, self.in_features, dtype=torch.float32, device=w.device)      # the tensor map spans np rows: they must exist
        wp[: self.out_features] = w.float()
        wq, sfb = (quantize_mxfp8 if w.is_cuda else quantize_mxfp8_reference)(wp)
        self.register_buffer("wq", wq)
        self.register_buffer("sfb", sfb)
        b = torch.zeros(self.np, dtype=torch.float32, device=w.device)
        if linear.bias is not None:
            b[: self.out_features] = linear.bias.detach().float()
        self.register_buffer("bias", b)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not x.is_cuda:                 # host fallback for tests / export checks: the same arithmetic in fp32
            xq, sfa = quantize_mxfp8_reference(x.float())
            y = dequantize_mxfp8(xq, sfa) @ dequantize_mxfp8(self.wq, self.sfb)[: self.out_features].t() + self.bias[: self.out_features]
            return (y.relu() if self.relu else y).bfloat16().to(x.dtype)      # same rounding point as the kernel's bf16 store
        xq, sfa = quantize_mxfp8(x.contiguous() if x.dtype in (torch.float32, torch.bfloat16) else x.float().contiguous())
        return mxfp8_gemm(xq, sfa, self.wq, self.sfb, self.np, self.bias, self.relu)[:, : self.out_features].to(x.dtype)
