"""torch.nn layers on the hand-written sm_90a kernels -- the building blocks the model zoo uses on a GPU.

  * ``FusedMLP`` / ``FusedLinear``: a chain of Linear(+ReLU) layers as ONE autograd node.  Forward = wgmma/TMA GEMM with
    bias + ReLU in the epilogue (csrc/cuda/gemm_wgmma.cu); backward = split-K wgmma weight-gradient GEMMs reading both
    operands MN-major, and dX GEMMs whose epilogue applies the previous layer's ReLU mask and reduces its bias gradient,
    i.e. the same dataflow as models/dlrm_engine.py but usable from any nn.Module.  Master weights stay fp32; bf16 shadows
    are re-packed every forward by one small kernel per layer.
  * ``dot_interaction`` (DLRM) and ``fm_interaction`` (DeepFM second order) autograd functions on
    csrc/cuda/interaction_kernels.cu.
  * ``fused_gru``: a single-layer GRU over tail-padded sequences for training -- the input projection on the wgmma GEMM, the recurrence
    forward and backward through time on csrc/cuda/rnn_kernels.cu.
  * ``fused_encoder_layer``: a post-norm Transformer encoder layer with a key-padding mask for training -- in_proj, out_proj and the FFN on
    the wgmma GEMM, the multi-head self-attention core forward and backward on csrc/cuda/mha_kernels.cu.
  * ``fused_din_attention``: DIN's attention unit (the weighted sum of the history, or DIEN's softmax weights) for training, forward and backward
    on csrc/cuda/din_att_kernels.cu.
  * ``FusedMaskBlock``: MaskNet's MaskBlock as one autograd node -- the mask MLP's GEMMs with their BatchNorm statistics in the epilogue,
    the last BatchNorm fused with the instance-guided product, and the block's Linear with LayerNorm + ReLU in the GEMM epilogue.
  * ``fused_expert_mlps`` / ``fused_moe_mix`` (``FUSED_MOE``): MMoE's and PLE's same-shaped expert and tower MLPs as grouped wgmma GEMMs, and a
    mixture layer's softmax gates as one kernel (csrc/cuda/moe_kernels.cu).

The reference runs these through cuBLAS (stream_executor/cuda/cuda_blas.cc) and ~10 TF ops per interaction
(modelzoo/dlrm/train.py:163-236, modelzoo/deepfm/train.py:178-187).  CPU tensors fall back to the equivalent torch expression.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, List, NamedTuple, Optional, Sequence

import torch
from torch import nn
from torch.nn import functional as F

from .. import _native
from .._native import check, ptr, stream_ptr


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


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
        check(_native.cuda().dr_cuda_cast_pad(ptr(x), M, K, ptr(y), Kp, stream_ptr()), "cast_pad")
        return y
    y = x.to(torch.bfloat16)
    if Kp != K:
        y = F.pad(y, (0, Kp - K))
    return y.contiguous()


def _pack_weight(W: torch.Tensor, Np: int, Kp: int):
    """fp32 master W [N, K] -> (bf16 W [Np, Kp], bf16 W^T [Kp, Np]), zero padded: the B operands of the forward and the dX GEMM."""
    N, K = W.shape
    Wp = W.detach().float()
    if (Np, Kp) != (N, K):
        Wp = F.pad(Wp, (0, Kp - K, 0, Np - N))
    Wp = Wp.contiguous()
    wb = torch.empty(Np, Kp, dtype=torch.bfloat16, device=W.device)
    wt = torch.empty(Kp, Np, dtype=torch.bfloat16, device=W.device)
    check(_native.cuda().dr_cuda_pack_weights(ptr(Wp), Np, Kp, ptr(wb), ptr(wt), Np, stream_ptr()), "pack_weights")
    return wb, wt


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
            wb, wt = _pack_weight(W, Np, Kp)
            bias = b.detach().float() if b is not None else None
            if bias is not None and Np != N:
                bias = F.pad(bias, (0, Np - N))
            relu = int(i + 1 < nl or last_act)
            out = torch.empty(M, Np, dtype=torch.bfloat16, device=dev)
            check(lib.dr_cuda_gemm_tn_ex(ptr(acts[-1]), Kp, ptr(wb), Kp, M, Np, Kp, ptr(bias) if bias is not None else None, relu, None, 0, 0,
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
            check(lib.dr_cuda_bn_bwd_apply_v2(ptr(g), ptr(acts[-1]), M, Np, Np, ptr(one), ptr(zero), ptr(zero), ptr(zero), ptr(zero), ptr(da), 1, ptr(db), s),
                  "relu_bwd")
        else:
            da = g
            check(lib.dr_cuda_colstats(ptr(da), None, M, Np, Np, Np, ptr(db), None, s), "colstats")
        for i in range(nl - 1, -1, -1):
            N, K, Np, Kp, has_bias = dims[i]
            dW = torch.zeros(Np, Kp, dtype=torch.float32, device=dev)
            check(lib.dr_cuda_gemm_dw(ptr(da), Np, ptr(acts[i]), Kp, M, Np, Kp, ptr(dW), Kp, 0, s), "gemm_dw")
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
                check(lib.dr_cuda_gemm_tn_ex(ptr(da), Np, ptr(wts[i]), Np, M, Kp, Np, None, 0, ptr(acts[i]), Kp, 1, ptr(prev), Kp, None,
                                             ptr(db) if fused else None, None, 0, 0, s), "gemm_dx")
                if not fused:
                    check(lib.dr_cuda_colstats(ptr(prev), None, M, Kp, Kp, Kp, ptr(db), None, s), "colstats")
            else:
                check(lib.dr_cuda_gemm_tn_ex(ptr(da), Np, ptr(wts[i]), Np, M, Kp, Np, None, 0, None, 0, 0, ptr(prev), Kp, None, None, None, 0, 0, s), "gemm_dx")
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
        check(lib.dr_cuda_dot_interaction_fwd(ptr(xb), D, ptr(eb), D, T * D, T, D, B, ptr(Z), Zp, stream_ptr()), "dot_interaction_fwd")
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
        check(lib.dr_cuda_dot_interaction_bwd(ptr(g), Zp, ptr(xb), D, ptr(eb), D, T * D, T, D, B, ptr(dx), D, ptr(de), D, T * D, stream_ptr()),
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
        check(lib.dr_cuda_fm_fwd(ptr(eb), D, T * D, T, D, B, ptr(out), D, ptr(ssum), stream_ptr()), "fm_fwd")
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
        check(lib.dr_cuda_fm_bwd(ptr(gb), D, ptr(eb), D, T * D, ptr(ssum), T, D, B, ptr(de), D, T * D, 0, stream_ptr()), "fm_bwd")
        return de.to(ctx.dt)


def fm_interaction(emb: torch.Tensor) -> torch.Tensor:
    """DeepFM second-order term 0.5 * ((sum_t v_t)^2 - sum_t v_t^2), emb [B, T, D] -> [B, D] (modelzoo/deepfm/train.py:178-187)."""
    if emb.is_cuda and emb.shape[2] in (8, 16, 32, 64):
        return _FMInteraction.apply(emb)
    return 0.5 * (emb.sum(1) ** 2 - (emb ** 2).sum(1))


# ---- GRU ---------------------------------------------------------------------------------------------------------------------
GRU_HIDDEN = (16, 32, 48, 64)         # hidden sizes csrc/cuda/rnn_kernels.cu is compiled for


class _GRURecurrenceFn(torch.autograd.Function):
    """gi [B L, 3H] bf16 (x W_ih^T + b_ih) -> y [B, L, H] fp32: the recurrence of a GRU with W_hh, b_hh, sample b running lengths[b] steps."""

    @staticmethod
    def forward(ctx, gi, w_hh, b_hh, lengths, B: int, L: int):
        H = w_hh.shape[1]
        w, b = w_hh.detach().float().contiguous(), b_hh.detach().float().contiguous()
        y = torch.empty(B, L, H, dtype=torch.float32, device=gi.device)
        check(_native.cuda().dr_cuda_gru_fwd(ptr(gi), ptr(w), ptr(b), ptr(lengths), B, L, H, ptr(y), stream_ptr()), "gru_fwd")
        ctx.save_for_backward(gi, w, b, lengths, y)
        ctx.shape = (B, L, H)
        return y

    @staticmethod
    def backward(ctx, dy):
        gi, w, b, lengths, y = ctx.saved_tensors
        B, L, H = ctx.shape
        dev = gi.device
        dgi = torch.empty(B * L, 3 * H, dtype=torch.bfloat16, device=dev)
        dgh = torch.empty(B * L, 3 * H, dtype=torch.bfloat16, device=dev)
        hprev = torch.empty(B * L, H, dtype=torch.bfloat16, device=dev)
        dw = torch.zeros(3 * H, H, dtype=torch.float32, device=dev)
        db = torch.zeros(3 * H, dtype=torch.float32, device=dev)
        dy = dy.float().contiguous()
        check(_native.cuda().dr_cuda_gru_bwd(ptr(gi), ptr(w), ptr(b), ptr(lengths), ptr(y), ptr(dy), B, L, H, ptr(dgi), ptr(dgh), ptr(hprev),
                                             ptr(dw), ptr(db), stream_ptr()), "gru_bwd")
        return dgi, dw, db, None, None, None


def fused_gru(x: torch.Tensor, gru: nn.GRU, lengths: torch.Tensor) -> torch.Tensor:
    """Single-layer, batch-first, unidirectional ``gru`` over ``x`` [B, L, I] whose sample b is ``lengths[b]`` (0..L) steps long, the rest
    being tail padding: y [B, L, H] is h_t for t < lengths[b] and 0 past it (``tf.nn.dynamic_rnn(..., sequence_length=)``), h_0 = 0.
    Trains the module's own parameters, so checkpoints keep its tensor names.  CUDA: the input projection on the wgmma GEMM (bf16), the
    recurrence forward and backward on mma.sync kernels (bf16 operands, fp32 state), fp32 weight gradients; H must be one of
    ``GRU_HIDDEN``.  CPU: the module itself, its outputs past the length zeroed."""
    if gru.num_layers != 1 or not gru.batch_first or gru.bidirectional or not gru.bias or getattr(gru, "proj_size", 0):
        raise ValueError("fused_gru: needs a single-layer, batch-first, unidirectional nn.GRU with biases")
    B, L, I = x.shape
    H = gru.hidden_size
    if not x.is_cuda:
        y, _ = gru(x.to(gru.weight_ih_l0.dtype))
        valid = torch.arange(L, device=x.device)[None] < lengths.to(x.device)[:, None]
        return y * valid.unsqueeze(-1).to(y.dtype)
    if H not in GRU_HIDDEN:
        raise ValueError(f"fused_gru: hidden size {H} is not supported on CUDA (one of {GRU_HIDDEN})")
    gi = _FusedMLPFn.apply(x.reshape(B * L, I).to(torch.bfloat16), False, gru.weight_ih_l0, gru.bias_ih_l0)
    return _GRURecurrenceFn.apply(gi.contiguous(), gru.weight_hh_l0, gru.bias_hh_l0, lengths.to(device=x.device, dtype=torch.int32).contiguous(), B, L)


# ---- Transformer encoder layer -----------------------------------------------------------------------------------------------
MHA_HEAD_DIMS = (8, 16, 32)           # head sizes csrc/cuda/mha_kernels.cu is compiled for
MHA_MAX_LEN = 128                     # longest sequence it takes


class _MHACoreFn(torch.autograd.Function):
    """qkv bf16 [B S, 3E] (in_proj output, [q | k | v] per token), valid uint8 [B, S] (key mask) -> o bf16 [B S, E]: softmax(q k^T / sqrt(dh)
    + key mask) v per (sample, head).  The backward recomputes the probabilities from qkv; it returns d(qkv) bf16 [B S, 3E]."""

    @staticmethod
    def forward(ctx, qkv, valid, B: int, S: int, heads: int):
        E = qkv.shape[1] // 3
        o = torch.empty(B * S, E, dtype=torch.bfloat16, device=qkv.device)
        check(_native.cuda().dr_cuda_mha_fwd(ptr(qkv), ptr(valid), B, S, E, heads, ptr(o), stream_ptr()), "mha_fwd")
        ctx.save_for_backward(qkv, valid, o)
        ctx.shape = (B, S, heads)
        return o

    @staticmethod
    def backward(ctx, do):
        qkv, valid, o = ctx.saved_tensors
        B, S, heads = ctx.shape
        dqkv = torch.empty_like(qkv)
        do = do.to(torch.bfloat16).contiguous()
        check(_native.cuda().dr_cuda_mha_bwd(ptr(qkv), ptr(valid), ptr(o), ptr(do), B, S, qkv.shape[1] // 3, heads, ptr(dqkv), stream_ptr()),
              "mha_bwd")
        return dqkv, None, None, None, None


def _check_encoder_layer(layer: nn.TransformerEncoderLayer) -> None:
    at = layer.self_attn
    if layer.norm_first:
        raise ValueError("fused_encoder_layer: needs a post-norm layer (norm_first=False)")
    if getattr(layer, "activation_relu_or_gelu", 0) != 1:
        raise ValueError("fused_encoder_layer: needs the ReLU activation")
    if not at.batch_first:
        raise ValueError("fused_encoder_layer: needs batch_first=True")
    if (at.in_proj_weight is None or at.in_proj_bias is None or at.out_proj.bias is None or layer.linear1.bias is None or layer.linear2.bias is None
            or layer.norm1.bias is None or layer.norm2.bias is None or at.bias_k is not None):
        raise ValueError("fused_encoder_layer: needs a layer with biases (and a packed in_proj, no bias_k / bias_v)")
    if layer.training and max(at.dropout, layer.dropout.p, layer.dropout1.p, layer.dropout2.p) > 0:
        raise ValueError("fused_encoder_layer: dropout > 0 while training is not supported")


def fused_encoder_layer(x: torch.Tensor, layer: nn.TransformerEncoderLayer, valid: torch.Tensor) -> torch.Tensor:
    """``layer(x, src_key_padding_mask=~valid)`` for a post-norm, batch-first, ReLU ``nn.TransformerEncoderLayer`` with biases over
    ``x`` [B, S, E] with key mask ``valid`` (bool [B, S], True = the position takes part as a key; every query row is computed).  Trains the
    module's own parameters, so state-dict names and the op-program export keep working.

    CUDA: in_proj, the attention core (csrc/cuda/mha_kernels.cu: mma.sync, fp32 softmax, no atomics), out_proj and the FFN (linear1 + ReLU +
    linear2, one node) on the wgmma GEMMs with bf16 activations and fp32 weight gradients; the residual adds and ``norm1`` / ``norm2`` are the
    module's own, in ``x``'s dtype.  dh = E / heads must be one of ``MHA_HEAD_DIMS`` and S at most ``MHA_MAX_LEN``.  One deliberate
    difference: a sample with no valid key gives attention output 0 where PyTorch gives NaN.  CPU: the module itself."""
    _check_encoder_layer(layer)
    if not x.is_cuda:
        return layer(x, src_key_padding_mask=~valid.to(torch.bool))
    B, S, E = x.shape
    at = layer.self_attn
    heads = at.num_heads
    if E % heads or E // heads not in MHA_HEAD_DIMS or S > MHA_MAX_LEN:
        raise ValueError(f"fused_encoder_layer: head size {E / heads:g} (E = {E}, {heads} heads) and S = {S} are not supported on CUDA "
                         f"(head size one of {MHA_HEAD_DIMS}, S <= {MHA_MAX_LEN})")
    x2 = x.reshape(B * S, E)
    qkv = _FusedMLPFn.apply(x2.to(torch.bfloat16), False, at.in_proj_weight, at.in_proj_bias)
    o = _MHACoreFn.apply(qkv.contiguous(), valid.to(device=x.device, dtype=torch.uint8).contiguous(), B, S, heads)
    a = _FusedMLPFn.apply(o, False, at.out_proj.weight, at.out_proj.bias)
    h = layer.norm1(x2 + a.to(x.dtype))
    f = _FusedMLPFn.apply(h.to(torch.bfloat16), False, layer.linear1.weight, layer.linear1.bias, layer.linear2.weight, layer.linear2.bias)
    return layer.norm2(h + f.to(h.dtype)).reshape(B, S, E)


# ---- DIN attention unit ------------------------------------------------------------------------------------------------------
DIN_ATT_DIMS = (16, 32, 48, 64)       # widths of q and k csrc/cuda/din_att_kernels.cu is compiled for
DIN_ATT_MAX_H1, DIN_ATT_MAX_H2, DIN_ATT_MAX_LEN = 128, 64, 128


class _DinAttentionFn(torch.autograd.Function):
    """q [B, D], k [B, L, D], mask [B, L] and the unit's parameters -> out fp32 [B, D] (mode 0) or w fp32 [B, L] (mode 1) on
    csrc/cuda/din_att_kernels.cu.  The backward recomputes the unit from q, k and the mask; b3 gets an exact 0 gradient."""

    @staticmethod
    def forward(ctx, q, k, mask, mode: int, W1, b1, W2, b2, W3, b3):
        B, L, D = k.shape
        qf = q.detach().float().contiguous()
        kd = k.detach()
        if kd.dtype not in (torch.bfloat16, torch.float32):
            kd = kd.float()
        kd = kd.contiguous()
        mk = mask.to(device=q.device, dtype=torch.bool).contiguous()
        ws = [t.detach().float().contiguous() for t in (W1, b1, W2, b2, W3.reshape(-1))]
        out = torch.empty((B, D) if mode == 0 else (B, L), dtype=torch.float32, device=q.device)
        check(_native.cuda().dr_cuda_din_att_fwd(ptr(qf), ptr(kd), int(kd.dtype == torch.bfloat16), ptr(mk), B, L, D, ptr(ws[0]), ptr(ws[1]),
                                                 W1.shape[0], ptr(ws[2]), ptr(ws[3]), W2.shape[0], ptr(ws[4]), mode, ptr(out), stream_ptr()),
              "din_att_fwd")
        ctx.save_for_backward(qf, kd, mk, *ws)
        ctx.mode, ctx.dtypes, ctx.w3_shape = mode, (q.dtype, k.dtype, b3.dtype), W3.shape
        return out

    @staticmethod
    def backward(ctx, g):
        qf, kd, mk, W1, b1, W2, b2, w3 = ctx.saved_tensors
        B, L, D = kd.shape
        H1, H2 = W1.shape[0], W2.shape[0]
        dev = qf.device
        gf = g.detach().float().contiguous()
        dq, dk = torch.empty_like(qf), torch.empty_like(kd)
        dW1, db1, dW2, db2 = torch.empty_like(W1), torch.empty_like(b1), torch.empty_like(W2), torch.empty_like(b2)
        dw3, db3 = torch.empty_like(w3), torch.empty(1, dtype=torch.float32, device=dev)
        scratch = torch.empty(B * L * (2 * D + 2 * H1 + H2), dtype=torch.bfloat16, device=dev)
        check(_native.cuda().dr_cuda_din_att_bwd(ptr(qf), ptr(kd), int(kd.dtype == torch.bfloat16), ptr(mk), ptr(gf), B, L, D, ptr(W1), ptr(b1), H1,
                                                 ptr(W2), ptr(b2), H2, ptr(w3), ctx.mode, ptr(dq), ptr(dk), ptr(dW1), ptr(db1), ptr(dW2), ptr(db2),
                                                 ptr(dw3), ptr(db3), ptr(scratch), stream_ptr()), "din_att_bwd")
        tq, tk, tb3 = ctx.dtypes
        return (dq.to(tq), dk.to(tk), None, None, dW1, db1, dW2, db2, dw3.view(ctx.w3_shape), db3.to(tb3))


def _check_din_unit(q: torch.Tensor, k: torch.Tensor, att: nn.Module) -> None:
    from ..ops.attention import _fusable
    if not _fusable(att):
        raise ValueError("fused_din_attention: needs the Linear-Sigmoid-Linear-Sigmoid-Linear(1) unit with biases")
    D = q.shape[-1]
    if k.dim() != 3 or k.shape[-1] != D or att[0].in_features != 4 * D or att[2].in_features != att[0].out_features \
            or att[4].in_features != att[2].out_features:
        raise ValueError(f"fused_din_attention: q [B, D], k [B, L, D] and a unit over 4 D = {4 * D} inputs are needed "
                         f"(got q {tuple(q.shape)}, k {tuple(k.shape)}, first layer in_features {att[0].in_features})")


def fused_din_attention(q: torch.Tensor, k: torch.Tensor, mask: torch.Tensor, att: nn.Module, weights: bool = False) -> torch.Tensor:
    """DIN's attention unit over the behaviour history: scores ``att(cat[q, k_t, q - k_t, q * k_t])`` for ``q`` [B, D], ``k`` [B, L, D], a
    masked softmax over the positions with ``mask`` (bool [B, L], True = valid), then the weighted sum of the keys [B, D] (``weights=False``,
    DIN; 0 for a sample with no valid position) or the softmax weights fp32 [B, L] (``weights=True``, DIEN; 1 / L everywhere for a sample
    with no valid position).  ``att`` is the Linear-Sigmoid-Linear-Sigmoid-Linear(1) unit; the op trains its own parameters, so state dicts
    and exports do not change.

    CUDA: one autograd node on csrc/cuda/din_att_kernels.cu (mma.sync with bf16 operands, fp32 softmax and gradients, no floating-point atomics,
    no host synchronisation, so it can be captured in a CUDA graph).  No gradient reaches a masked position or a sample with no valid position.
    D must be one of ``DIN_ATT_DIMS``, the hidden widths multiples of 16 (<= 128) and 8 (<= 64), L at most ``DIN_ATT_MAX_LEN``.  Elsewhere (CPU,
    the kernel emulation, ``DEEPREC_FUSED_NN=0``): the torch expressions ``ops.attention.din_attention`` (sum) and DIEN's inline softmax."""
    _check_din_unit(q, k, att)
    if not (_fused_nn(q) and q.is_cuda):
        if not weights:
            from ..ops.attention import din_attention
            return din_attention(q, k, mask, att)
        qe = q.unsqueeze(1).expand_as(k)
        s = att(torch.cat([qe, k, qe - k, qe * k], -1)).squeeze(-1).masked_fill(~mask, -2 ** 31)
        return torch.softmax(s, -1)
    B, L, D = k.shape
    H1, H2 = att[0].out_features, att[2].out_features
    if D not in DIN_ATT_DIMS or H1 % 16 or H1 > DIN_ATT_MAX_H1 or H2 % 8 or H2 > DIN_ATT_MAX_H2 or not 1 <= L <= DIN_ATT_MAX_LEN or B < 1:
        raise ValueError(f"fused_din_attention: D = {D}, H1 = {H1}, H2 = {H2}, L = {L} are not supported on CUDA (D one of {DIN_ATT_DIMS}, "
                         f"H1 a multiple of 16 up to {DIN_ATT_MAX_H1}, H2 a multiple of 8 up to {DIN_ATT_MAX_H2}, 1 <= L <= {DIN_ATT_MAX_LEN})")
    l1, l2, l3 = att[0], att[2], att[4]
    out = _DinAttentionFn.apply(q, k, mask, 1 if weights else 0, l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias)
    return out if weights else out.to(q.dtype)


# ---- MaskNet MaskBlock -------------------------------------------------------------------------------------------------------
MASKBLOCK_MAX_OUT = 128               # the LayerNorm GEMM epilogue holds a whole output row in one tile


def _bn_tf(x: torch.Tensor, bn: nn.BatchNorm1d) -> torch.Tensor:
    """``tf.layers.batch_normalization`` of [B, N]: batch statistics while training, the moving averages updated with the biased batch
    variance at decay ``1 - bn.momentum`` (what dr_cuda_bn_finalize does; torch's BatchNorm1d would use the unbiased variance); the moving
    averages in eval mode."""
    if not bn.training:
        return F.batch_norm(x, bn.running_mean, bn.running_var, bn.weight, bn.bias, False, 0.0, bn.eps)
    with torch.no_grad():
        xf = x.detach().float()
        bn.running_mean.mul_(1.0 - bn.momentum).add_(xf.mean(0), alpha=bn.momentum)
        bn.running_var.mul_(1.0 - bn.momentum).add_(xf.var(0, unbiased=False), alpha=bn.momentum)
    return F.batch_norm(x, None, None, bn.weight, bn.bias, True, 0.0, bn.eps)


class _FusedMaskBlockFn(torch.autograd.Function):
    """out = relu(LN(W3 (BN2(relu(W2 BN1(relu(W1 v_emb + b1)) + b2)) * v_hidden)))  on the kernels; ``params`` = W1, b1, gamma1, beta1, W2, b2,
    gamma2, beta2, W3, gamma_ln, beta_ln (fp32 masters).  The BatchNorm moving averages of ``blk`` are updated in place by dr_cuda_bn_finalize.
    Widths are zero padded to multiples of 8: padded weight rows / columns, BatchNorm scale and shift are 0, so padded columns stay 0."""

    @staticmethod
    def forward(ctx, v_emb, v_hidden, blk, training: bool, *params):
        lib, s, dev = _native.cuda(), stream_ptr(), v_emb.device
        W1, b1, g1, be1, W2, b2, g2, be2, W3, gl, bl = params
        M, E = v_emb.shape
        H, R, O = v_hidden.shape[1], W1.shape[0], W3.shape[0]
        Ep, Hp, Rp = _pad8(E), _pad8(H), _pad8(R)
        f32 = dict(dtype=torch.float32, device=dev)
        bf = dict(dtype=torch.bfloat16, device=dev)
        xe = _to_bf16_padded(v_emb, Ep)
        xh = xe if v_hidden is v_emb else _to_bf16_padded(v_hidden, Hp)
        w1b, w1t = _pack_weight(W1, Rp, Ep)
        w2b, w2t = _pack_weight(W2, Hp, Rp)
        w3b, w3t = _pack_weight(W3, O, Hp)

        def lin_relu_bn(x, Kp, wb, b, N, Np, bn, g, be):
            """a = relu(x W^T + b) with its column statistics in the GEMM epilogue -> st = [mean | rstd | scale | shift] of the BatchNorm"""
            a = torch.empty(M, Np, **bf)
            S = torch.zeros(2, Np, **f32) if training else None
            bias = F.pad(b.detach().float(), (0, Np - N)).contiguous()
            check(lib.dr_cuda_gemm_tn_ex(ptr(x), Kp, ptr(wb), Kp, M, Np, Kp, ptr(bias), 1, None, 0, 0, ptr(a), Np, None,
                                         ptr(S[0]) if training else None, ptr(S[1]) if training else None, 0, 0, s), "gemm_tn")
            st = torch.zeros(4, Np, **f32)
            check(lib.dr_cuda_bn_finalize(ptr(S[0]) if training else None, ptr(S[1]) if training else None, N, M, ptr(g.detach().float().contiguous()),
                                          ptr(be.detach().float().contiguous()), bn.eps, 1.0 - bn.momentum, ptr(bn.running_mean), ptr(bn.running_var),
                                          ptr(st[0]), ptr(st[1]), ptr(st[2]), ptr(st[3]), int(training), s), "bn_finalize")
            return a, st

        a1, st1 = lin_relu_bn(xe, Ep, w1b, b1, R, Rp, blk.bn1, g1, be1)
        m1 = torch.empty(M, Rp, **bf)
        check(lib.dr_cuda_bn_apply(ptr(a1), M, Rp, Rp, ptr(st1[2]), ptr(st1[3]), ptr(m1), Rp, s), "bn_apply")
        a2, st2 = lin_relu_bn(m1, Rp, w2b, b2, H, Hp, blk.bn2, g2, be2)
        p = torch.empty(M, Hp, **bf)
        check(lib.dr_cuda_bn_apply_mul(ptr(a2), Hp, ptr(st2[2]), ptr(st2[3]), ptr(xh), Hp, M, Hp, ptr(p), Hp, s), "bn_apply_mul")
        y = torch.empty(M, O, **bf)
        xhat = torch.empty(M, O, **bf)
        rstd = torch.empty(M, **f32)
        glf = gl.detach().float().contiguous()
        check(lib.dr_cuda_gemm_tn_ln(ptr(p), Hp, ptr(w3b), Hp, M, O, Hp, None, ptr(glf), ptr(bl.detach().float().contiguous()), blk.ln.eps, 1,
                                     ptr(y), O, ptr(xhat), O, ptr(rstd), 0, s), "gemm_tn_ln")
        ctx.save_for_backward(xe, xh, a1, m1, a2, p, y, xhat, rstd, w1t, w2t, w3t, st1, st2, glf)
        ctx.meta = (E, H, R, O, v_emb.dtype, v_hidden.dtype)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib, s = _native.cuda(), stream_ptr()
        xe, xh, a1, m1, a2, p, y, xhat, rstd, w1t, w2t, w3t, st1, st2, glf = ctx.saved_tensors
        E, H, R, O, edt, hdt = ctx.meta
        M, Ep, Hp, Rp = xe.shape[0], xe.shape[1], xh.shape[1], a1.shape[1]
        dev = gy.device
        f32 = dict(dtype=torch.float32, device=dev)
        bf = dict(dtype=torch.bfloat16, device=dev)
        g = gy.to(torch.bfloat16).contiguous()
        # LayerNorm + ReLU, then the block's Linear (no bias)
        dh = torch.empty(M, O, **bf)
        dgl, dbl = torch.zeros(O, **f32), torch.zeros(O, **f32)
        check(lib.dr_cuda_ln_relu_bwd(ptr(g), O, ptr(y), O, ptr(xhat), O, ptr(rstd), ptr(glf), M, O, ptr(dh), O, ptr(dgl), ptr(dbl), s), "ln_relu_bwd")
        dW3 = torch.zeros(O, Hp, **f32)
        check(lib.dr_cuda_gemm_dw(ptr(dh), O, ptr(p), Hp, M, O, Hp, ptr(dW3), Hp, 0, s), "gemm_dw")
        dp = torch.empty(M, Hp, **bf)
        check(lib.dr_cuda_gemm_tn_ex(ptr(dh), O, ptr(w3t), O, M, Hp, O, None, 0, None, 0, 0, ptr(dp), Hp, None, None, None, 0, 0, s), "gemm_dx")
        # p = BN2(a2) * v_hidden: dv_hidden, and the BatchNorm-backward sums of dm = dp * v_hidden
        dv = torch.empty(M, Hp, **bf)
        dm = torch.empty(M, Hp, **bf)
        S = torch.zeros(2, Hp, **f32)
        check(lib.dr_cuda_bn_mul_bwd(ptr(dp), Hp, ptr(a2), Hp, ptr(xh), Hp, ptr(st2[2]), ptr(st2[3]), M, Hp, ptr(dv), Hp, ptr(dm), Hp, ptr(S[0]), ptr(S[1]), s),
              "bn_mul_bwd")

        def bn_relu_lin_bwd(dy, a, st, S, N, Np, x, Kp):
            """BatchNorm backward (with the ReLU mask of a) from the sums S, then the Linear's weight and bias gradients against its input x"""
            dg, dbe, c = torch.zeros(N, **f32), torch.zeros(N, **f32), torch.zeros(2, Np, **f32)
            check(lib.dr_cuda_bn_bwd_finalize(ptr(S[0]), ptr(S[1]), N, M, ptr(st[0]), ptr(st[1]), ptr(dg), ptr(dbe), ptr(c[0]), ptr(c[1]), 1.0, s),
                  "bn_bwd_finalize")
            da, db = torch.empty(M, Np, **bf), torch.zeros(Np, **f32)
            check(lib.dr_cuda_bn_bwd_apply_v2(ptr(dy), ptr(a), M, Np, Np, ptr(st[2]), ptr(st[0]), ptr(st[1]), ptr(c[0]), ptr(c[1]), ptr(da), 1, ptr(db), s),
                  "bn_bwd_apply")
            dW = torch.zeros(Np, Kp, **f32)
            check(lib.dr_cuda_gemm_dw(ptr(da), Np, ptr(x), Kp, M, Np, Kp, ptr(dW), Kp, 0, s), "gemm_dw")
            return da, dW, db, dg, dbe

        da2, dW2, db2, dg2, dbe2 = bn_relu_lin_bwd(dm, a2, st2, S, H, Hp, m1, Rp)
        # dm1 = da2 W2, with the BatchNorm-backward sums of layer 1 (sum dm1, sum dm1 * a1) in the GEMM epilogue
        dm1 = torch.empty(M, Rp, **bf)
        S = torch.zeros(2, Rp, **f32)
        check(lib.dr_cuda_gemm_tn_ex(ptr(da2), Hp, ptr(w2t), Hp, M, Rp, Hp, None, 0, ptr(a1), Rp, 2, ptr(dm1), Rp, None, ptr(S[0]), ptr(S[1]), 0, 0, s),
              "gemm_dx")
        da1, dW1, db1, dg1, dbe1 = bn_relu_lin_bwd(dm1, a1, st1, S, R, Rp, xe, Ep)
        dxe = None
        if ctx.needs_input_grad[0]:
            dxe = torch.empty(M, Ep, **bf)
            check(lib.dr_cuda_gemm_tn_ex(ptr(da1), Rp, ptr(w1t), Rp, M, Ep, Rp, None, 0, None, 0, 0, ptr(dxe), Ep, None, None, None, 0, 0, s), "gemm_dx")
            dxe = dxe[:, :E].to(edt)
        dxh = dv[:, :H].to(hdt) if ctx.needs_input_grad[1] else None
        return (dxe, dxh, None, None, dW1[:R, :E], db1[:R], dg1, dbe1, dW2[:H, :R], db2[:H], dg2, dbe2, dW3[:, :H], dgl, dbl)


class FusedMaskBlock(nn.Module):
    """MaskNet's MaskBlock (modelzoo/masknet/train.py:150-177):

        V_mask = BN(ReLU(Linear(BN(ReLU(Linear(V_emb, hidden_in * reduction_ratio))), hidden_in)))
        out    = ReLU(LayerNorm(Linear(V_mask * V_hidden, out_dim, bias=False)))

    with tf's defaults: BatchNorm eps 1e-3 and decay 0.99 (torch momentum 0.01; the moving variance takes the biased batch variance, as
    ``_bn_tf``), LayerNorm eps 1e-3.  ``forward(v_emb [B, emb_in], v_hidden [B, hidden_in]) -> [B, out_dim]``.

    On CUDA (and on the kernel emulation), unless ``DEEPREC_FUSED_NN=0``: one autograd node on the sm_90a kernels -- bf16 activations, fp32
    statistics and weight gradients, the BatchNorm moving averages updated inside the step (so a captured CUDA graph updates them too);
    ``out_dim`` must be a multiple of 8 and at most ``MASKBLOCK_MAX_OUT``.  Otherwise the same expression in torch ops, which is the oracle."""

    def __init__(self, hidden_in: int, emb_in: int, out_dim: int = 64, reduction_ratio: int = 1, bn_eps: float = 1e-3, bn_momentum: float = 0.01,
                 ln_eps: float = 1e-3, device=None):
        super().__init__()
        self.hidden_in, self.emb_in, self.out_dim = hidden_in, emb_in, out_dim
        r = hidden_in * reduction_ratio
        self.fc1 = nn.Linear(emb_in, r, device=device)
        self.bn1 = nn.BatchNorm1d(r, eps=bn_eps, momentum=bn_momentum, device=device)
        self.fc2 = nn.Linear(r, hidden_in, device=device)
        self.bn2 = nn.BatchNorm1d(hidden_in, eps=bn_eps, momentum=bn_momentum, device=device)
        self.fc3 = nn.Linear(hidden_in, out_dim, bias=False, device=device)
        self.ln = nn.LayerNorm(out_dim, eps=ln_eps, device=device)
        for fc in (self.fc1, self.fc2, self.fc3):                 # tf.layers.dense: glorot_uniform kernel, zero bias
            nn.init.xavier_uniform_(fc.weight)
            if fc.bias is not None:
                nn.init.zeros_(fc.bias)

    def forward(self, v_emb: torch.Tensor, v_hidden: torch.Tensor) -> torch.Tensor:
        import os
        if _native.on_device(v_emb) and os.environ.get("DEEPREC_FUSED_NN", "1") != "0":
            if self.out_dim % 8 or self.out_dim > MASKBLOCK_MAX_OUT:
                raise ValueError(f"FusedMaskBlock: out_dim {self.out_dim} is not supported on CUDA (a multiple of 8, at most {MASKBLOCK_MAX_OUT})")
            return _FusedMaskBlockFn.apply(v_emb, v_hidden, self, self.training, self.fc1.weight, self.fc1.bias, self.bn1.weight, self.bn1.bias,
                                           self.fc2.weight, self.fc2.bias, self.bn2.weight, self.bn2.bias, self.fc3.weight, self.ln.weight, self.ln.bias)
        return self.expression(v_emb, v_hidden)

    def expression(self, v_emb: torch.Tensor, v_hidden: torch.Tensor) -> torch.Tensor:
        """The block in torch ops (the CPU path and the oracle of the kernels)."""
        m = _bn_tf(torch.relu(self.fc1(v_emb)), self.bn1)
        m = _bn_tf(torch.relu(self.fc2(m)), self.bn2)
        return torch.relu(self.ln(self.fc3(m * v_hidden)))


# ---- expert mixtures (MMoE, PLE) ---------------------------------------------------------------------------------------------
GEMM_MAX_GROUPS = 12                  # kMaxGroups of csrc/cuda/gemm_wgmma.cu: groups one grouped-GEMM launch takes (more are split)
MOE_MAX_GATES, MOE_MAX_EXPERTS, MOE_MAX_H = 8, 32, 512   # limits of one csrc/cuda/moe_kernels.cu launch


def _fused_nn(t: torch.Tensor) -> bool:
    import os
    return _native.on_device(t) and os.environ.get("DEEPREC_FUSED_NN", "1") != "0"


def _ptrs(vals):
    return (C.c_void_p * len(vals))(*[v.value if isinstance(v, C.c_void_p) else v for v in vals])


def _i64s(vals):
    return (C.c_int64 * len(vals))(*vals)


def _ints(vals):
    return (C.c_int * len(vals))(*vals)


def _gemm_tn_grouped(A, lda, B, ldb, M: int, N: int, K: int, out, ldc, bias=None, relu: int = 0, mask=None, ld_mask=None, S1=None) -> None:
    """dr_cuda_gemm_tn_grouped over per-group lists (raw pointers / pitches), GEMM_MAX_GROUPS groups per launch."""
    lib, s = _native.cuda(), stream_ptr()
    for i in range(0, len(A), GEMM_MAX_GROUPS):
        j = slice(i, i + GEMM_MAX_GROUPS)
        check(lib.dr_cuda_gemm_tn_grouped(len(A[j]), _ptrs(A[j]), _i64s(lda[j]), _ptrs(B[j]), _i64s(ldb[j]), M, N, K,
                                          _ptrs(bias[j]) if bias else None, relu, _ptrs(mask[j]) if mask else None,
                                          _i64s(ld_mask[j]) if mask else None, _ptrs(out[j]), _i64s(ldc[j]), _ptrs(S1[j]) if S1 else None, 0, s),
              "gemm_tn_grouped")


def _gemm_dw_grouped(dY, ldy, X, ldx, batch: int, N_out: int, K_in: int, dW, ldw) -> None:
    """dr_cuda_gemm_dw_grouped over per-group lists, GEMM_MAX_GROUPS groups per launch."""
    lib, s = _native.cuda(), stream_ptr()
    for i in range(0, len(dY), GEMM_MAX_GROUPS):
        j = slice(i, i + GEMM_MAX_GROUPS)
        check(lib.dr_cuda_gemm_dw_grouped(len(dY[j]), _ptrs(dY[j]), _i64s(ldy[j]), _ptrs(X[j]), _i64s(ldx[j]), batch, N_out, K_in, _ptrs(dW[j]),
                                          _i64s(ldw[j]), 0, s), "gemm_dw_grouped")


def _addr(t: torch.Tensor, elems: int = 0) -> int:
    """address of element ``elems`` of t's storage (a column offset into a packed row-major buffer)"""
    return t.data_ptr() + elems * t.element_size()


def _mlp_layers(m: nn.Module):
    """(weights, biases, last_act) of a ReLU MLP as :func:`models.zoo.mlp` builds it: a ``FusedMLP``, or an ``nn.Sequential`` of Linear / ReLU."""
    if isinstance(m, FusedMLP):
        if m.biases is None:
            raise ValueError("fused_expert_mlps: needs MLPs with biases")
        return list(m.weights), list(m.biases), m.last_act
    if isinstance(m, nn.Sequential):
        ws, bs, acts = [], [], []
        for mod in m:
            if isinstance(mod, nn.Linear) and mod.bias is not None:
                ws.append(mod.weight); bs.append(mod.bias); acts.append(False)
            elif isinstance(mod, nn.ReLU) and acts and not acts[-1]:
                acts[-1] = True
            else:
                raise ValueError(f"fused_expert_mlps: {type(mod).__name__} in an expert MLP (Linear with bias / ReLU only)")
        if ws and all(acts[:-1]):
            return ws, bs, acts[-1]
    raise ValueError(f"fused_expert_mlps: {type(m).__name__} is not a Linear + ReLU chain")


class _FusedExpertsFn(torch.autograd.Function):
    """G same-shaped MLPs -> their outputs packed side by side [M, G Np_last] (bf16); ``args`` = the inputs (one shared or G), then W, b of every
    layer of group 0, group 1, ...  Widths are zero padded to multiples of 8; group g's layer-l activation is columns [g Np, g Np + Np) of one
    [M, G Np] buffer.  Layer 1 over a shared input is one GEMM over the row-concatenated weights (and its dX one GEMM with K = G Np, so the
    groups' input gradients add up in the accumulator); every other layer is a grouped GEMM, forward, dX (the ReLU mask and the bias gradient
    of the layer below in its epilogue) and dW."""

    @staticmethod
    def forward(ctx, nx: int, G: int, nl: int, last_act: bool, *args):
        lib, s = _native.cuda(), stream_ptr()
        xs, params = args[:nx], args[nx:]
        shared = nx == 1
        M, K0 = xs[0].shape
        dev = xs[0].device
        bf = dict(dtype=torch.bfloat16, device=dev)
        xin = [_to_bf16_padded(x, _pad8(K0)) for x in xs]
        acts: List[torch.Tensor] = []
        wts: List[torch.Tensor] = []
        dims = []
        for l in range(nl):
            N, K = params[2 * l].shape
            Np, Kp = _pad8(N), _pad8(K)
            Ws = [params[2 * (g * nl + l)] for g in range(G)]
            bias = torch.cat([F.pad(params[2 * (g * nl + l) + 1].detach().float(), (0, Np - N)) for g in range(G)])
            relu = int(l + 1 < nl or last_act)
            out = torch.empty(M, G * Np, **bf)
            if l == 0 and shared:
                Wcat = torch.cat([F.pad(W.detach().float(), (0, Kp - K, 0, Np - N)) for W in Ws])
                wb, wt = _pack_weight(Wcat, G * Np, Kp)
                check(lib.dr_cuda_gemm_tn_ex(ptr(xin[0]), Kp, ptr(wb), Kp, M, G * Np, Kp, ptr(bias), relu, None, 0, 0, ptr(out), G * Np, None, None, None,
                                             0, 0, s), "gemm_tn")
            else:
                packs = [_pack_weight(W, Np, Kp) for W in Ws]
                wt = torch.stack([p[1] for p in packs])                              # [G, Kp, Np]: the dX B operands
                A = [_addr(xin[g]) for g in range(G)] if l == 0 else [_addr(acts[-1], g * Kp) for g in range(G)]
                _gemm_tn_grouped(A, [Kp if l == 0 else G * Kp] * G, [_addr(p[0]) for p in packs], [Kp] * G, M, Np, Kp,
                                 [_addr(out, g * Np) for g in range(G)], [G * Np] * G, bias=[_addr(bias, g * Np) for g in range(G)], relu=relu)
            acts.append(out); wts.append(wt); dims.append((N, K, Np, Kp))
        ctx.save_for_backward(*xin, *acts, *wts)
        ctx.meta = (nx, G, nl, last_act, dims, [x.dtype for x in xs], K0)
        return acts[-1].to(xs[0].dtype)

    @staticmethod
    def backward(ctx, gy):
        lib, s = _native.cuda(), stream_ptr()
        nx, G, nl, last_act, dims, xdt, K0 = ctx.meta
        saved = ctx.saved_tensors
        xin, acts, wts = saved[:nx], saved[nx: nx + nl], saved[nx + nl:]
        shared = nx == 1
        dev = gy.device
        f32 = dict(dtype=torch.float32, device=dev)
        bf = dict(dtype=torch.bfloat16, device=dev)
        M = gy.shape[0]
        Np = dims[-1][2]
        g = gy.to(torch.bfloat16).contiguous()
        db = torch.zeros(G * Np, **f32)
        if last_act:
            one, zero = _const_vec(dev, G * Np, 1.0), _const_vec(dev, G * Np, 0.0)
            da = torch.empty(M, G * Np, **bf)
            check(lib.dr_cuda_bn_bwd_apply_v2(ptr(g), ptr(acts[-1]), M, G * Np, G * Np, ptr(one), ptr(zero), ptr(zero), ptr(zero), ptr(zero), ptr(da), 1,
                                              ptr(db), s), "relu_bwd")
        else:
            da = g
            check(lib.dr_cuda_colstats(ptr(da), None, M, G * Np, G * Np, G * Np, ptr(db), None, s), "colstats")
        need_dx = any(ctx.needs_input_grad[4: 4 + nx])
        grads: List[Optional[torch.Tensor]] = [None] * (2 * G * nl)
        dxs: List[Optional[torch.Tensor]] = [None] * nx
        for l in range(nl - 1, -1, -1):
            N, K, Np, Kp = dims[l]
            dY = [_addr(da, gi * Np) for gi in range(G)]
            if l == 0 and shared:
                dW = torch.zeros(G * Np, Kp, **f32)
                check(lib.dr_cuda_gemm_dw(ptr(da), G * Np, ptr(xin[0]), Kp, M, G * Np, Kp, ptr(dW), Kp, 0, s), "gemm_dw")
                dW = dW.view(G, Np, Kp)
            else:
                dW = torch.zeros(G, Np, Kp, **f32)
                X = [_addr(xin[gi]) for gi in range(G)] if l == 0 else [_addr(acts[l - 1], gi * Kp) for gi in range(G)]
                _gemm_dw_grouped(dY, [G * Np] * G, X, [Kp if l == 0 else G * Kp] * G, M, Np, Kp, [_addr(dW[gi]) for gi in range(G)], [Kp] * G)
            for gi in range(G):
                grads[2 * (gi * nl + l)] = dW[gi, :N, :K]
                grads[2 * (gi * nl + l) + 1] = db[gi * Np: gi * Np + N]
            if l > 0:
                prev = torch.empty(M, G * Kp, **bf)
                db = torch.zeros(G * Kp, **f32)
                _gemm_tn_grouped(dY, [G * Np] * G, [_addr(wts[l][gi]) for gi in range(G)], [Np] * G, M, Kp, Np, [_addr(prev, gi * Kp) for gi in range(G)],
                                 [G * Kp] * G, mask=[_addr(acts[l - 1], gi * Kp) for gi in range(G)], ld_mask=[G * Kp] * G,
                                 S1=[_addr(db, gi * Kp) for gi in range(G)])
                da = prev
            elif need_dx and shared:
                dx = torch.empty(M, Kp, **bf)
                check(lib.dr_cuda_gemm_tn_ex(ptr(da), G * Np, ptr(wts[0]), G * Np, M, Kp, G * Np, None, 0, None, 0, 0, ptr(dx), Kp, None, None, None, 0, 0, s),
                      "gemm_dx")
                dxs[0] = dx[:, :K0].to(xdt[0])
            elif need_dx:
                dx = torch.empty(M, G * Kp, **bf)
                _gemm_tn_grouped(dY, [G * Np] * G, [_addr(wts[0][gi]) for gi in range(G)], [Np] * G, M, Kp, Np, [_addr(dx, gi * Kp) for gi in range(G)],
                                 [G * Kp] * G)
                dxs = [dx[:, gi * Kp: gi * Kp + K0].to(xdt[gi]) for gi in range(G)]
        return (None, None, None, None, *dxs, *grads)


def fused_expert_mlps(x, mlps: Sequence[nn.Module]) -> torch.Tensor:
    """Runs G same-shaped ReLU MLPs (``models.zoo.mlp``: a ``FusedMLP``, or the ``nn.Sequential`` of Linear / ReLU it builds off the GPU) over one
    shared input ``x`` [M, K] or over one input each (``x`` a list of G [M, K] tensors), and returns their outputs side by side: [M, G H], group g
    in columns [g H, g H + H).  Trains the modules' own parameters, so state dicts, checkpoints and the op-program export are unchanged.

    On CUDA (and on the kernel emulation), unless ``DEEPREC_FUSED_NN=0``: one autograd node (bf16 activations, output in ``x``'s dtype).  A shared input's first layer is one
    GEMM over the row-concatenated weights; every other layer runs the G groups as one grouped wgmma GEMM (csrc/cuda/gemm_wgmma.cu), forward
    and backward, with fp32 weight gradients.  H must be a multiple of 8 there.  Otherwise the modules themselves, concatenated."""
    xs = list(x) if isinstance(x, (list, tuple)) else [x]
    if len(xs) not in (1, len(mlps)):
        raise ValueError(f"fused_expert_mlps: {len(xs)} inputs for {len(mlps)} MLPs (one shared input, or one each)")
    if not _fused_nn(xs[0]):
        return torch.cat([m(xs[0] if len(xs) == 1 else xi) for m, xi in zip(mlps, xs * len(mlps) if len(xs) == 1 else xs)], -1)
    layers = [_mlp_layers(m) for m in mlps]
    shapes = [[tuple(w.shape) for w in ws] for ws, _, _ in layers]
    if any(sh != shapes[0] for sh in shapes) or any(la != layers[0][2] for _, _, la in layers):
        raise ValueError("fused_expert_mlps: the MLPs differ in shape or in their last activation")
    H = shapes[0][-1][0]
    if H % 8:
        raise ValueError(f"fused_expert_mlps: output width {H} is not a multiple of 8")
    params = [t for ws, bs, _ in layers for w, b in zip(ws, bs) for t in (w, b)]
    return _FusedExpertsFn.apply(len(xs), len(mlps), len(shapes[0]), layers[0][2], *[xi.reshape(-1, xi.shape[-1]) for xi in xs], *params)


class _MoEMixFn(torch.autograd.Function):
    """mix_t = sum_e softmax(x_t W_t^T + b_t)_e X[:, sel_t[e]] for the T gates of one mixture layer on csrc/cuda/moe_kernels.cu; ``args`` = the
    gate inputs, weights and biases (T each).  X: the packed experts [M, E_total H] (bf16)."""

    @staticmethod
    def forward(ctx, T: int, E_total: int, H: int, sel, X, *args):
        lib, s = _native.cuda(), stream_ptr()
        xs = [x.to(torch.bfloat16).contiguous() for x in args[:T]]
        Ws = [w.detach().float().contiguous() for w in args[T: 2 * T]]
        bs = [b.detach().float().contiguous() for b in args[2 * T:]]
        M, dev = X.shape[0], X.device
        mix = [torch.empty(M, H, dtype=torch.bfloat16, device=dev) for _ in range(T)]
        g = [torch.empty(M, len(sl), dtype=torch.float32, device=dev) for sl in sel]
        sel_a = _ints([i for sl in sel for i in list(sl) + [0] * (MOE_MAX_EXPERTS - len(sl))])
        check(lib.dr_cuda_moe_mix_fwd(ptr(X), X.shape[1], M, E_total, H, T, _ptrs([x.data_ptr() for x in xs]), _i64s([x.shape[1] for x in xs]),
                                      _ints([x.shape[1] for x in xs]), _ints([len(sl) for sl in sel]), _ptrs([w.data_ptr() for w in Ws]),
                                      _ptrs([b.data_ptr() for b in bs]), sel_a, _ptrs([m.data_ptr() for m in mix]), _i64s([H] * T),
                                      _ptrs([t.data_ptr() for t in g]), s), "moe_mix_fwd")
        ctx.save_for_backward(X, *xs, *Ws, *g)
        ctx.meta = (T, E_total, H, sel, [x.dtype for x in args[:T]])
        return tuple(m.to(x.dtype) for m, x in zip(mix, args[:T]))

    @staticmethod
    def backward(ctx, *dmix):
        lib, s = _native.cuda(), stream_ptr()
        T, E_total, H, sel, xdt = ctx.meta
        saved = ctx.saved_tensors
        X, xs, Ws, g = saved[0], saved[1: 1 + T], saved[1 + T: 1 + 2 * T], saved[1 + 2 * T:]
        M, dev = X.shape[0], X.device
        dm = [d.to(torch.bfloat16).contiguous() if d is not None else torch.zeros(M, H, dtype=torch.bfloat16, device=dev) for d in dmix]
        dX = torch.empty(M, E_total * H, dtype=torch.bfloat16, device=dev)
        need = [ctx.needs_input_grad[5 + t] for t in range(T)]
        dx = [torch.empty(M, x.shape[1], dtype=torch.bfloat16, device=dev) if n else None for x, n in zip(xs, need)]
        dWb = [torch.zeros(w.numel() + w.shape[0], dtype=torch.float32, device=dev) for w in Ws]
        sel_a = _ints([i for sl in sel for i in list(sl) + [0] * (MOE_MAX_EXPERTS - len(sl))])
        check(lib.dr_cuda_moe_mix_bwd(ptr(X), X.shape[1], M, E_total, H, T, _ptrs([x.data_ptr() for x in xs]), _i64s([x.shape[1] for x in xs]),
                                      _ints([x.shape[1] for x in xs]), _ints([len(sl) for sl in sel]), _ptrs([w.data_ptr() for w in Ws]), sel_a,
                                      _ptrs([t.data_ptr() for t in g]), _ptrs([d.data_ptr() for d in dm]), _i64s([H] * T), ptr(dX), E_total * H,
                                      _ptrs([d.data_ptr() if d is not None else 0 for d in dx]), _i64s([x.shape[1] for x in xs]),
                                      _ptrs([d.data_ptr() for d in dWb]), s), "moe_mix_bwd")
        dxs = [d.to(dt) if d is not None else None for d, dt in zip(dx, xdt)]
        dWs = [d[: w.numel()].view_as(w) for d, w in zip(dWb, Ws)]
        dbs = [d[w.numel():] for d, w in zip(dWb, Ws)]
        return (None, None, None, None, dX, *dxs, *dWs, *dbs)


def fused_moe_mix(xs: Sequence[torch.Tensor], gates: Sequence[nn.Linear], experts: torch.Tensor, select: Sequence[Sequence[int]]) -> List[torch.Tensor]:
    """One mixture layer of MMoE / PLE: for every gate t, ``softmax(gates[t](xs[t])) . experts[:, select[t]]`` -> [M, H], where ``experts`` is
    [M, E, H] (expert e's output in ``experts[:, e]``, e.g. a view of :func:`fused_expert_mlps`' packed output) and ``select[t]`` the experts
    gate t mixes, in the order of its logits.

    On CUDA (and on the kernel emulation), unless ``DEEPREC_FUSED_NN=0``: one autograd node on csrc/cuda/moe_kernels.cu -- fp32 logits and
    softmax from bf16 inputs and the fp32 gate weights, a bf16 mix (returned in ``xs[t]``'s dtype); the backward sums each expert's gradient over the gates that read it in gate
    order, with no atomics.  At most MOE_MAX_GATES gates, MOE_MAX_EXPERTS experts, H a multiple of 8 up to MOE_MAX_H.  Otherwise the same
    expression in torch ops, which is the oracle."""
    if len(xs) != len(gates) or len(gates) != len(select):
        raise ValueError("fused_moe_mix: xs, gates and select differ in length")
    M, E_total, H = experts.shape
    if not _fused_nn(experts):
        return [(torch.softmax(gate(x), -1).unsqueeze(-1) * experts[:, list(sl)]).sum(1) for x, gate, sl in zip(xs, gates, select)]
    T = len(gates)
    if T > MOE_MAX_GATES or E_total > MOE_MAX_EXPERTS or H % 8 or H > MOE_MAX_H or any(not 1 <= len(sl) <= MOE_MAX_EXPERTS for sl in select):
        raise ValueError(f"fused_moe_mix: {T} gates over {E_total} experts of width {H} is not supported on CUDA (at most {MOE_MAX_GATES} gates and "
                         f"{MOE_MAX_EXPERTS} experts, H a multiple of 8 up to {MOE_MAX_H})")
    if any(g.bias is None for g in gates):
        raise ValueError("fused_moe_mix: needs gates with biases")
    X = experts.reshape(M, E_total * H).to(torch.bfloat16).contiguous()
    sel = tuple(tuple(int(i) for i in sl) for sl in select)
    return list(_MoEMixFn.apply(T, E_total, H, sel, X, *[x.reshape(M, -1) for x in xs], *[g.weight for g in gates], *[g.bias for g in gates]))


class MoEOps(NamedTuple):
    """The expert-mixture ops a model's ``tower_logits(f, moe=...)`` runs its experts, gates and towers through."""
    expert_mlps: Callable
    mix: Callable


FUSED_MOE = MoEOps(fused_expert_mlps, fused_moe_mix)
