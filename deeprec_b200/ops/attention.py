"""DIN attention unit (modelzoo/din/train.py:143-188): ``concat[q, k, q-k, q*k] -> H1 -> H2 -> 1`` (sigmoid activations), masked
softmax over the behaviour history, weighted sum of the keys.

* training (autograd needed) -> the composite PyTorch implementation below, or (``DEEPREC_DIN_FUSED_TRAIN=1``) the fused forward + backward
  kernels: the backward recomputes the activations in shared memory, so neither they nor their gradients touch HBM;
* inference on CUDA          -> ONE fused kernel (csrc/cuda/attention_kernels.cu): weights resident in shared memory, the
  ``[B, L, 4D]`` concat never materialised, half the first-layer FLOPs via ``W1 f = (W1q+W1d) q + (W1k-W1d) k + W1p (q*k)``.
"""
from __future__ import annotations

import os

import torch
import torch.nn as nn

from .. import _native
from .._native import check, ptr, stream_ptr


def din_attention_reference(q: torch.Tensor, k: torch.Tensor, mask: torch.Tensor, att: nn.Module) -> torch.Tensor:
    """Composite implementation (any device, differentiable).  q [B, D], k [B, L, D], mask [B, L] bool -> [B, D]."""
    qe = q.unsqueeze(1).expand_as(k)
    s = att(torch.cat([qe, k, qe - k, qe * k], -1)).squeeze(-1)
    s = s.masked_fill(~mask, -2 ** 31)
    w = torch.softmax(s, -1) * mask.any(-1, keepdim=True)
    return (w.unsqueeze(-1) * k).sum(1)


def din_attention_composite(q: torch.Tensor, k: torch.Tensor, mask: torch.Tensor, att: nn.Module) -> torch.Tensor:
    """Differentiable training path: same math as ``din_attention_reference`` with the first layer split
    (``W1 [q, k, q-k, q*k] = (Wq + Wd) q + (Wk - Wd) k + Wp (q*k)``): the q term is computed once per sample, the ``[B, L, 4D]``
    concat is never built and the first layer costs half the FLOPs.  Falls back to the reference for other ``att`` shapes."""
    if not _fusable(att) or att[0].in_features != 4 * q.shape[-1]:
        return din_attention_reference(q, k, mask, att)
    import torch.nn.functional as F
    D = q.shape[-1]
    Wq, Wk, Wp = split_first_layer(att[0].weight, D)
    hq = F.linear(q, Wq, att[0].bias)                                        # [B, H1], once per sample
    h1 = torch.sigmoid(hq.unsqueeze(1) + F.linear(k, Wk) + F.linear(q.unsqueeze(1) * k, Wp))
    s = att[4](torch.sigmoid(att[2](h1))).squeeze(-1)
    s = s.masked_fill(~mask, -2 ** 31)
    w = torch.softmax(s, -1) * mask.any(-1, keepdim=True)
    return torch.bmm(w.unsqueeze(1), k).squeeze(1)                            # weighted sum of the keys


def split_first_layer(W1: torch.Tensor, D: int):
    """The algebra the kernel uses: W1 [H1, 4D] -> (Wq, Wk, Wp) with  W1 @ [q, k, q-k, q*k] = Wq q + Wk k + Wp (q*k)."""
    Wa, Wb, Wc, Wd = W1[:, :D], W1[:, D:2 * D], W1[:, 2 * D:3 * D], W1[:, 3 * D:]
    return Wa + Wc, Wb - Wc, Wd


def _fusable(att: nn.Module) -> bool:
    mods = list(att.children()) if isinstance(att, nn.Sequential) else []
    return (len(mods) == 5 and all(isinstance(mods[i], nn.Linear) for i in (0, 2, 4)) and all(isinstance(mods[i], nn.Sigmoid) for i in (1, 3))
            and mods[4].out_features == 1 and all(m.bias is not None for m in (mods[0], mods[2], mods[4])))


class _DinAttentionFused(torch.autograd.Function):
    """Fused forward AND backward (csrc/cuda/attention_kernels.cu): nothing but q, k, mask, the output and the gradients touches HBM --
    the ``[B, L, 4D]`` concat, the two ``[B * L, H]`` activations and their gradients live in shared memory (the backward recomputes them)."""

    @staticmethod
    def forward(ctx, q, k, mask, W1, b1, W2, b2, W3, b3):
        B, L, D = k.shape
        qf, kf = q.detach().float().contiguous(), k.detach().float().contiguous()
        mk = mask.to(torch.bool).contiguous()
        ws = [t.detach().float().contiguous() for t in (W1, b1, W2, b2, W3.reshape(-1))]
        b3f = float(b3.detach().float().item())
        out = torch.empty(B, D, device=q.device, dtype=torch.float32)
        check(_native.cuda().dr_cuda_din_attention_fwd(ptr(qf), ptr(kf), ptr(mk), B, L, D, ptr(ws[0]), ptr(ws[1]), W1.shape[0], ptr(ws[2]), ptr(ws[3]),
                                                       W2.shape[0], ptr(ws[4]), b3f, ptr(out), stream_ptr()), "din_attention_fwd")
        ctx.save_for_backward(qf, kf, mk, *ws)
        ctx.b3, ctx.dtypes = b3f, (q.dtype, k.dtype, W1.dtype, b1.dtype, W2.dtype, b2.dtype, W3.dtype, b3.dtype)
        ctx.w3_shape = W3.shape
        return out.to(q.dtype)

    @staticmethod
    def backward(ctx, g):
        qf, kf, mk, W1, b1, W2, b2, w3 = ctx.saved_tensors
        B, L, D = kf.shape
        H1, H2 = W1.shape[0], W2.shape[0]
        dev = qf.device
        gf = g.detach().float().contiguous()
        dq, dk = torch.empty_like(qf), torch.empty_like(kf)
        dW1, db1, dW2, db2 = torch.zeros_like(W1), torch.zeros_like(b1), torch.zeros_like(W2), torch.zeros_like(b2)
        dw3, db3 = torch.zeros_like(w3), torch.zeros(1, device=dev)
        check(_native.cuda().dr_cuda_din_attention_bwd(ptr(qf), ptr(kf), ptr(mk), ptr(gf), B, L, D, ptr(W1), ptr(b1), H1, ptr(W2), ptr(b2), H2, ptr(w3),
                                                       ctx.b3, ptr(dq), ptr(dk), ptr(dW1), ptr(db1), ptr(dW2), ptr(db2), ptr(dw3), ptr(db3), stream_ptr()),
              "din_attention_bwd")
        t = ctx.dtypes
        return (dq.to(t[0]), dk.to(t[1]), None, dW1.to(t[2]), db1.to(t[3]), dW2.to(t[4]), db2.to(t[5]), dw3.view(ctx.w3_shape).to(t[6]), db3.to(t[7]))


def din_attention_fused_train(q: torch.Tensor, k: torch.Tensor, mask: torch.Tensor, att: nn.Module) -> torch.Tensor:
    """Differentiable fused path (CUDA, the Linear-Sigmoid-Linear-Sigmoid-Linear(1) unit): ``k`` is masked inside the kernels, so masked
    positions receive zero gradient.  Selected by ``din_attention`` when ``DEEPREC_DIN_FUSED_TRAIN=1``; outside CUDA-graph capture only (the
    forward reads the scalar output bias on the host)."""
    l1, l2, l3 = att[0], att[2], att[4]
    return _DinAttentionFused.apply(q, k, mask, l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias)


def din_attention(q: torch.Tensor, k: torch.Tensor, mask: torch.Tensor, att: nn.Module) -> torch.Tensor:
    """Dispatch: fused kernel when on CUDA, no gradient is required and ``att`` is the Linear-Sigmoid-Linear-Sigmoid-Linear(1) unit."""
    needs_grad = torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or any(p.requires_grad for p in att.parameters()))
    if needs_grad and _native.on_device(q) and _fusable(att) and att[0].in_features == 4 * q.shape[-1] and os.environ.get("DEEPREC_DIN_FUSED_TRAIN", "0") == "1" \
            and not torch.cuda.is_current_stream_capturing():
        return din_attention_fused_train(q, k, mask, att)
    if not _native.on_device(q) or needs_grad or not _fusable(att) or att[0].in_features != 4 * q.shape[-1]:
        return din_attention_composite(q, k, mask, att)
    B, L, D = k.shape
    l1, l2, l3 = att[0], att[2], att[4]
    qf, kf = q.detach().float().contiguous(), k.detach().float().contiguous()
    mk = mask.to(torch.bool).contiguous()
    out = torch.empty(B, D, device=q.device, dtype=torch.float32)
    rc = _native.cuda().dr_cuda_din_attention_fwd(ptr(qf), ptr(kf), ptr(mk), B, L, D, ptr(l1.weight.detach().float().contiguous()),
                                                  ptr(l1.bias.detach().float().contiguous()), l1.out_features,
                                                  ptr(l2.weight.detach().float().contiguous()), ptr(l2.bias.detach().float().contiguous()), l2.out_features,
                                                  ptr(l3.weight.detach().float().contiguous().view(-1)), _b3(l3),
                                                  ptr(out), stream_ptr())
    if rc == -1:                                   # shape does not fit the kernel's shared-memory budget
        return din_attention_reference(q, k, mask, att)
    check(rc, "din_attention_fwd")
    return out.to(q.dtype)


_B3_CACHE: dict = {}


def _b3(l3: nn.Linear) -> float:
    """Scalar bias of the last layer as a host float, cached per parameter version (avoids a device sync on every call)."""
    key = (id(l3.bias), l3.bias._version)
    v = _B3_CACHE.get(key)
    if v is None:
        _B3_CACHE.clear()
        v = _B3_CACHE[key] = float(l3.bias.detach().float().item())
    return v
