"""Fused LayerNorm / L2-normalize / GELU / Dice (kernels/fused_layer_norm, fused_l2_normalize, gelu_op*, dice_fusion in the reference).
CUDA tensors run the sm_90a kernels (csrc/cuda/fused_ops.cu); CPU tensors use the equivalent torch expression."""
from __future__ import annotations

import ctypes as C

import torch

from .. import _native
from .._native import ptr, stream_ptr

_BOUND = False


def _lib():
    global _BOUND
    lib = _native.cuda()
    if not _BOUND:
        i64, INT, f32, P = C.c_int64, C.c_int, C.c_float, C.c_void_p
        for name, args in {"dr_cuda_layer_norm_fwd": [P, i64, INT, P, P, f32, P, P, P, P], "dr_cuda_layer_norm_bwd": [P, P, i64, INT, P, P, P, P, P, P, P],
                           "dr_cuda_l2_normalize_fwd": [P, i64, INT, f32, P, P, P], "dr_cuda_l2_normalize_bwd": [P, P, P, i64, INT, P, P],
                           "dr_cuda_gelu_fwd": [P, i64, INT, P, P], "dr_cuda_gelu_bwd": [P, P, i64, INT, P, P],
                           "dr_cuda_dice_fwd": [P, i64, INT, P, P, P, P, P]}.items():
            fn = getattr(lib, name); fn.argtypes, fn.restype = args, INT
        _BOUND = True
    return lib


class _LayerNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        x2 = x.contiguous().float().view(-1, x.shape[-1])
        rows, cols = x2.shape
        y = torch.empty_like(x2); mean = torch.empty(rows, device=x.device); rstd = torch.empty(rows, device=x.device)
        _lib().dr_cuda_layer_norm_fwd(ptr(x2), rows, cols, ptr(gamma), ptr(beta), float(eps), ptr(y), ptr(mean), ptr(rstd), stream_ptr())
        ctx.save_for_backward(x2, gamma, mean, rstd); ctx.shape = x.shape
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, g):
        x2, gamma, mean, rstd = ctx.saved_tensors
        rows, cols = x2.shape
        g2 = g.contiguous().float().view(rows, cols)
        dx = torch.empty_like(x2); dg = torch.zeros(cols, device=g.device); db = torch.zeros(cols, device=g.device)
        _lib().dr_cuda_layer_norm_bwd(ptr(g2), ptr(x2), rows, cols, ptr(gamma), ptr(mean), ptr(rstd), ptr(dx), ptr(dg), ptr(db), stream_ptr())
        return dx.view(ctx.shape), dg, db, None


def fused_layer_norm(x, gamma, beta, eps: float = 1e-5):
    if x.is_cuda:
        return _LayerNorm.apply(x, gamma.contiguous().float(), beta.contiguous().float(), eps)
    return torch.nn.functional.layer_norm(x, x.shape[-1:], gamma, beta, eps)


class _L2Norm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, eps):
        x2 = x.contiguous().float().view(-1, x.shape[-1])
        rows, cols = x2.shape
        y = torch.empty_like(x2); rn = torch.empty(rows, device=x.device)
        _lib().dr_cuda_l2_normalize_fwd(ptr(x2), rows, cols, float(eps), ptr(y), ptr(rn), stream_ptr())
        ctx.save_for_backward(y, rn); ctx.shape = x.shape
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, g):
        y, rn = ctx.saved_tensors
        rows, cols = y.shape
        g2 = g.contiguous().float().view(rows, cols)
        dx = torch.empty_like(y)
        _lib().dr_cuda_l2_normalize_bwd(ptr(g2), ptr(y), ptr(rn), rows, cols, ptr(dx), stream_ptr())
        return dx.view(ctx.shape), None


def fused_l2_normalize(x, eps: float = 1e-12):
    """``tf.nn.l2_normalize`` over the last axis (fused_l2_normalize op)."""
    if x.is_cuda:
        return _L2Norm.apply(x, eps)
    return x * torch.rsqrt(torch.clamp((x * x).sum(-1, keepdim=True), min=eps))


class _Gelu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, approximate):
        x2 = x.contiguous().float()
        y = torch.empty_like(x2)
        _lib().dr_cuda_gelu_fwd(ptr(x2), x2.numel(), int(approximate), ptr(y), stream_ptr())
        ctx.save_for_backward(x2); ctx.approx = approximate
        return y

    @staticmethod
    def backward(ctx, g):
        (x2,) = ctx.saved_tensors
        dx = torch.empty_like(x2)
        _lib().dr_cuda_gelu_bwd(ptr(g.contiguous().float()), ptr(x2), x2.numel(), int(ctx.approx), ptr(dx), stream_ptr())
        return dx, None


def gelu(x, approximate: bool = True):
    if x.is_cuda:
        return _Gelu.apply(x, approximate)
    return torch.nn.functional.gelu(x, approximate="tanh" if approximate else "none")


def dice(x, alpha, mean, var, eps: float = 1e-9):
    """Dice activation (DIN): p = sigmoid(BN(x)); y = p x + (1 - p) alpha x.  Inference-time fusion (dice_fusion.cc)."""
    rstd = torch.rsqrt(var + eps)
    if x.is_cuda and not x.requires_grad:
        x2 = x.contiguous().float().view(-1, x.shape[-1])
        y = torch.empty_like(x2)
        _lib().dr_cuda_dice_fwd(ptr(x2), x2.shape[0], x2.shape[1], ptr(mean.contiguous().float()), ptr(rstd.contiguous().float()),
                                ptr(alpha.contiguous().float()), ptr(y), stream_ptr())
        return y.view(x.shape)
    p = torch.sigmoid((x - mean) * rstd)
    return p * x + (1 - p) * alpha * x
