"""torch.nn layers on the hand-written sm_90a kernels -- the building blocks the model zoo uses on a GPU.

  * ``FusedMLP`` / ``FusedLinear``: a chain of Linear(+ReLU) layers as ONE autograd node.  Forward = wgmma/TMA GEMM with
    bias + ReLU in the epilogue (csrc/cuda/gemm_wgmma.cu); backward = split-K wgmma weight-gradient GEMMs reading both
    operands MN-major, and dX GEMMs whose epilogue applies the previous layer's ReLU mask and reduces its bias gradient,
    i.e. the same dataflow as models/dlrm_engine.py but usable from any nn.Module.  Master weights stay fp32; bf16 shadows
    are re-packed every forward by one small kernel per layer.
  * ``dot_interaction`` (DLRM) and ``fm_interaction`` (DeepFM second order) autograd functions on
    csrc/cuda/interaction_kernels.cu.

The reference runs these through cuBLAS (stream_executor/cuda/cuda_blas.cc) and ~10 TF ops per interaction
(modelzoo/dlrm/train.py:163-236, modelzoo/deepfm/train.py:178-187).  CPU tensors fall back to the equivalent torch expression.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
from torch import nn
from torch.nn import functional as F

from .. import _native
from .._native import ptr, stream_ptr


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


def _chk(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"deeprec_cuda: {what} failed with code {rc}")


_CONST = {}


def _const_vec(dev: torch.device, n: int, value: float) -> torch.Tensor:
    key = (dev, value)
    t = _CONST.get(key)
    if t is None or t.numel() < n:
        t = torch.full((max(n, 2048),), value, dtype=torch.float32, device=dev)
        _CONST[key] = t
    return t


def _to_bf16_padded(x: torch.Tensor, Kp: int) -> torch.Tensor:
    """[M, K] any float dtype -> contiguous bf16 [M, Kp] (zero padded columns)."""
    M, K = x.shape
    if x.dtype == torch.float32 and x.is_contiguous():
        y = torch.empty(M, Kp, dtype=torch.bfloat16, device=x.device)
        _chk(_native.cuda().dr_cuda_cast_pad(ptr(x), M, K, ptr(y), Kp, stream_ptr()), "cast_pad")
        return y
    y = x.to(torch.bfloat16)
    if Kp != K:
        y = F.pad(y, (0, Kp - K))
    return y.contiguous()


class _FusedMLPFn(torch.autograd.Function):
    """y = L_n(...relu(L_1(x))) ; ``params`` = W_1, b_1, ..., W_n, b_n (fp32 masters, W_i [N_i, K_i])."""

    @staticmethod
    def forward(ctx, x, last_act: bool, *params):
        lib = _native.cuda()
        s = stream_ptr()
        dev = x.device
        nl = len(params) // 2
        M, K0 = x.shape
        h = _to_bf16_padded(x, _pad8(K0))
        acts: List[torch.Tensor] = [h]
        wts: List[torch.Tensor] = []
        dims = []
        for i in range(nl):
            W, b = params[2 * i], params[2 * i + 1]
            N, K = W.shape
            Np, Kp = _pad8(N), _pad8(K)
            assert Kp == acts[-1].shape[1], f"layer {i}: expected input width {K}, got {acts[-1].shape[1]}"
            Wp = W.detach().float()
            if (Np, Kp) != (N, K):
                Wp = F.pad(Wp, (0, Kp - K, 0, Np - N))
            Wp = Wp.contiguous()
            wb = torch.empty(Np, Kp, dtype=torch.bfloat16, device=dev)
            wt = torch.empty(Kp, Np, dtype=torch.bfloat16, device=dev)
            _chk(lib.dr_cuda_pack_weights(ptr(Wp), Np, Kp, ptr(wb), ptr(wt), Np, s), "pack_weights")
            bias = b.detach().float() if b is not None else None
            if bias is not None and Np != N:
                bias = F.pad(bias, (0, Np - N))
            relu = int(i + 1 < nl or last_act)
            out = torch.empty(M, Np, dtype=torch.bfloat16, device=dev)
            _chk(lib.dr_cuda_gemm_tn_ex(ptr(acts[-1]), Kp, ptr(wb), Kp, M, Np, Kp, ptr(bias) if bias is not None else None, relu, None, 0, 0,
                                        ptr(out), Np, None, None, None, 0, 0, s), "gemm_tn")
            acts.append(out); wts.append(wt); dims.append((N, K, Np, Kp, b is not None))
        ctx.save_for_backward(*acts, *wts)
        ctx.meta = (nl, last_act, dims, x.dtype, x.requires_grad, K0)
        N_last = dims[-1][0]
        y = acts[-1][:, :N_last] if dims[-1][2] != N_last else acts[-1]
        return y.to(x.dtype) if x.dtype != torch.bfloat16 else y

    @staticmethod
    def backward(ctx, gy):
        lib = _native.cuda()
        s = stream_ptr()
        nl, last_act, dims, xdtype, need_dx, K0 = ctx.meta
        saved = ctx.saved_tensors
        acts, wts = saved[: nl + 1], saved[nl + 1:]
        dev = gy.device
        M = gy.shape[0]
        N, K, Np, Kp, _ = dims[-1]
        g = _to_bf16_padded(gy.contiguous() if gy.dtype == torch.float32 else gy, Np)
        grads: List[Optional[torch.Tensor]] = [None] * (2 * nl)
        # gradient w.r.t. the last pre-activation (+ its bias gradient)
        db = torch.zeros(Np, dtype=torch.float32, device=dev)
        if last_act:
            one, zero = _const_vec(dev, Np, 1.0), _const_vec(dev, Np, 0.0)
            da = torch.empty(M, Np, dtype=torch.bfloat16, device=dev)
            _chk(lib.dr_cuda_bn_bwd_apply_v2(ptr(g), ptr(acts[-1]), M, Np, Np, ptr(one), ptr(zero), ptr(zero), ptr(zero), ptr(zero), ptr(da), 1, ptr(db), s),
                 "relu_bwd")
        else:
            da = g
            _chk(lib.dr_cuda_colstats(ptr(da), None, M, Np, Np, Np, ptr(db), None, s), "colstats")
        for i in range(nl - 1, -1, -1):
            N, K, Np, Kp, has_bias = dims[i]
            dW = torch.zeros(Np, Kp, dtype=torch.float32, device=dev)
            _chk(lib.dr_cuda_gemm_dw(ptr(da), Np, ptr(acts[i]), Kp, M, Np, Kp, ptr(dW), Kp, 0, s), "gemm_dw")
            grads[2 * i] = dW[:N, :K] if (Np, Kp) != (N, K) else dW
            if has_bias:
                grads[2 * i + 1] = db[:N] if Np != N else db
            if i == 0 and not need_dx:
                break
            prev = torch.empty(M, Kp, dtype=torch.bfloat16, device=dev)
            if i > 0:
                # dX epilogue: * relu'(a_{i-1}); the bias gradient of layer i-1 (column sums) is fused for wide layers
                db = torch.zeros(Kp, dtype=torch.float32, device=dev)
                fused = Kp > 32
                _chk(lib.dr_cuda_gemm_tn_ex(ptr(da), Np, ptr(wts[i]), Np, M, Kp, Np, None, 0, ptr(acts[i]), Kp, 1, ptr(prev), Kp, None,
                                            ptr(db) if fused else None, None, 0, 0, s), "gemm_dx")
                if not fused:
                    _chk(lib.dr_cuda_colstats(ptr(prev), None, M, Kp, Kp, Kp, ptr(db), None, s), "colstats")
            else:
                _chk(lib.dr_cuda_gemm_tn_ex(ptr(da), Np, ptr(wts[i]), Np, M, Kp, Np, None, 0, None, 0, 0, ptr(prev), Kp, None, None, None, 0, 0, s), "gemm_dx")
            da = prev
        dx = None
        if need_dx:
            dx = da[:, :K0] if da.shape[1] != K0 else da
            dx = dx.to(xdtype)
        return (dx, None, *grads)


class FusedMLP(nn.Module):
    """Linear+ReLU chain on the wgmma GEMM kernels (CUDA) with an identical-math torch fallback (CPU).

    ``sizes`` are the layer widths; ``last_act`` says whether the last layer is followed by ReLU."""

    def __init__(self, in_dim: int, sizes: Sequence[int], last_act: bool = True, bias: bool = True, device=None):
        super().__init__()
        self.in_dim, self.sizes, self.last_act = in_dim, list(sizes), last_act
        self.weights = nn.ParameterList()
        self.biases = nn.ParameterList() if bias else None
        k = in_dim
        for n in sizes:
            w = torch.empty(n, k, device=device)
            nn.init.xavier_uniform_(w)                      # tf.layers.dense default (glorot_uniform)
            self.weights.append(nn.Parameter(w))
            if bias:
                self.biases.append(nn.Parameter(torch.zeros(n, device=device)))
            k = n

    def _params(self):
        out = []
        for i, w in enumerate(self.weights):
            out += [w, self.biases[i] if self.biases is not None else None]
        return out

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        lead = x.shape[:-1]
        x2 = x.reshape(-1, x.shape[-1])
        if x2.is_cuda:
            y = _FusedMLPFn.apply(x2, self.last_act, *self._params())
        else:
            y = x2
            n = len(self.weights)
            for i, w in enumerate(self.weights):
                y = F.linear(y, w, self.biases[i] if self.biases is not None else None)
                if i + 1 < n or self.last_act:
                    y = torch.relu(y)
        return y.reshape(*lead, y.shape[-1])


class FusedLinear(FusedMLP):
    """One Linear (optionally + ReLU) on the wgmma GEMM."""

    def __init__(self, in_features: int, out_features: int, relu: bool = False, bias: bool = True, device=None):
        super().__init__(in_features, [out_features], last_act=relu, bias=bias, device=device)


# ---- interactions ----------------------------------------------------------------------------------------------------------
class _DotInteraction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, emb):
        """x [B, D], emb [B, T, D] -> [B, D + (T+1)T/2]: x followed by the strict lower triangle of the Gram matrix of [x; emb]."""
        lib = _native.cuda()
        B, T, D = emb.shape
        xb, eb = x.to(torch.bfloat16).contiguous(), emb.to(torch.bfloat16).contiguous()
        nz = D + (T + 1) * T // 2
        Zp = _pad8(nz)
        Z = torch.zeros(B, Zp, dtype=torch.bfloat16, device=x.device)
        _chk(lib.dr_cuda_dot_interaction_fwd(ptr(xb), D, ptr(eb), D, T * D, T, D, B, ptr(Z), Zp, stream_ptr()), "dot_interaction_fwd")
        ctx.save_for_backward(xb, eb)
        ctx.meta = (nz, Zp, x.dtype, emb.dtype)
        return Z[:, :nz].to(x.dtype)

    @staticmethod
    def backward(ctx, gz):
        lib = _native.cuda()
        xb, eb = ctx.saved_tensors
        nz, Zp, xdt, edt = ctx.meta
        B, T, D = eb.shape
        g = _to_bf16_padded(gz.contiguous() if gz.dtype == torch.float32 else gz, Zp)
        dx = torch.empty(B, D, dtype=torch.bfloat16, device=gz.device)
        de = torch.empty(B, T, D, dtype=torch.bfloat16, device=gz.device)
        _chk(lib.dr_cuda_dot_interaction_bwd(ptr(g), Zp, ptr(xb), D, ptr(eb), D, T * D, T, D, B, ptr(dx), D, ptr(de), D, T * D, stream_ptr()),
             "dot_interaction_bwd")
        return dx.to(xdt), de.to(edt)


def dot_interaction(x: torch.Tensor, emb: torch.Tensor) -> torch.Tensor:
    """DLRM 'dot' interaction (modelzoo/dlrm/train.py:163-236).  CUDA: tensor-core kernel (D = 16, mma.sync) / SIMT kernel (D = 8, 32)."""
    if x.is_cuda and emb.shape[1] + 1 <= 32 and emb.shape[2] in (8, 16, 32) and _pad8(emb.shape[2] + (emb.shape[1] + 1) * emb.shape[1] // 2) <= 512:
        return _DotInteraction.apply(x, emb)
    feats = torch.cat([x.unsqueeze(1), emb], 1)
    gram = torch.bmm(feats, feats.transpose(1, 2))
    F_ = feats.shape[1]
    li, lj = torch.tril_indices(F_, F_, -1, device=x.device)
    return torch.cat([x, gram[:, li, lj]], 1)


class _FMInteraction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, emb):
        lib = _native.cuda()
        B, T, D = emb.shape
        eb = emb.to(torch.bfloat16).contiguous()
        out = torch.empty(B, D, dtype=torch.bfloat16, device=emb.device)
        ssum = torch.empty(B, D, dtype=torch.float32, device=emb.device)
        _chk(lib.dr_cuda_fm_fwd(ptr(eb), D, T * D, T, D, B, ptr(out), D, ptr(ssum), stream_ptr()), "fm_fwd")
        ctx.save_for_backward(eb, ssum)
        ctx.dt = emb.dtype
        return out.to(emb.dtype)

    @staticmethod
    def backward(ctx, g):
        lib = _native.cuda()
        eb, ssum = ctx.saved_tensors
        B, T, D = eb.shape
        gb = g.to(torch.bfloat16).contiguous()
        de = torch.empty(B, T, D, dtype=torch.bfloat16, device=g.device)
        _chk(lib.dr_cuda_fm_bwd(ptr(gb), D, ptr(eb), D, T * D, ptr(ssum), T, D, B, ptr(de), D, T * D, 0, stream_ptr()), "fm_bwd")
        return de.to(ctx.dt)


def fm_interaction(emb: torch.Tensor) -> torch.Tensor:
    """DeepFM second-order term 0.5 * ((sum_t v_t)^2 - sum_t v_t^2), emb [B, T, D] -> [B, D] (modelzoo/deepfm/train.py:178-187)."""
    if emb.is_cuda and emb.shape[2] in (8, 16, 32, 64):
        return _FMInteraction.apply(emb)
    return 0.5 * (emb.sum(1) ** 2 - (emb ** 2).sum(1))
