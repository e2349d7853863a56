"""Shared cases for the multi-head self-attention kernels (csrc/cuda/mha_kernels.cu), ``nn.fused_encoder_layer`` and BST on FusedRecEngine,
with the float64 oracle they are checked against.

The oracle takes the kernels' bf16 inputs (qkv, do) and, for the backward, the kernel's own bf16 o (D = rowsum(do * o) is formed from it, as
the kernel forms it); everything else is float64 and unrounded.  The kernels' rounding points (the comment at the top of mha_kernels.cu) bound
the difference (u = 2^-24, the fp32 unit roundoff; b = 2^-9, half a bf16 ulp):
  * P: the scores are fp32 sums of exact bf16 products (dh u relative to sum |q||k|), then __expf (ex2.approx of an fp32 product), an fp32 sum
    of at most 128 terms and rcp: P is within 2^-16 P of the exact probabilities (|s| < 2^5 at these input scales);
  * o = bf16(bf16(P) V): bf16(P) is within (b + 2^-16) P of P, the fp32 sum adds S u, the output rounding b |o|:
    |o - o_ref| <= 2^-8 (P |V| + |o_ref|)                                                                         (TOL)
  * dS = P (dP - D) scale in fp32: the error of P (2^-16 P |dP - D|) and of dP, D (fp32 sums of exact products, dh u relative to their
    magnitudes) give |dS - dS_ref| <= 2^-15 P (|dO| |V|^T + |dO| . |o|) scale =: 2^-15 A; the bf16 operand adds b |dS|:
    |dq - dq_ref| <= 2^-8 (|dS| |K| + |dq_ref|) + 2^-15 A |K|,  |dk - dk_ref| <= 2^-8 (|dS|^T |Q| + |dk_ref|) + 2^-15 A^T |Q|   (TOL, TOL_A)
  * dv = bf16(sum over tiles of bf16(P)^T dO): |dv - dv_ref| <= 2^-8 (P^T |dO| + |dv_ref|)                                    (TOL)
Exact: dk and dv of a masked key are 0; o and dq of a sample with no valid key are 0 (PyTorch gives NaN there).
"""
from __future__ import annotations

import copy
import math

import numpy as np
import torch

TOL = 2.0 ** -8
TOL_A = 2.0 ** -15
MASKS = ("all", "last", "random", "empty")


def make_valid(kind: str, B: int, S: int, seed: int = 0) -> torch.Tensor:
    """uint8 [B, S] key mask: every key, only the last position, ~60 % at random positions, or random with every third sample empty."""
    g = torch.Generator().manual_seed(seed)
    if kind == "all":
        return torch.ones(B, S, dtype=torch.uint8)
    if kind == "last":
        v = torch.zeros(B, S, dtype=torch.uint8)
        v[:, -1] = 1
        return v
    v = (torch.rand(B, S, generator=g) < 0.6).to(torch.uint8)
    if kind == "empty":
        v[::3] = 0
    return v


def make_case(B: int, S: int, heads: int, dh: int, seed: int, dev):
    """qkv bf16 [B S, 3E] (N(0, 1), the scale of in_proj outputs of a unit-variance input), do bf16 [B S, E]."""
    g = torch.Generator().manual_seed(seed)
    E = heads * dh
    qkv = torch.randn(B * S, 3 * E, generator=g).to(torch.bfloat16)
    do = torch.randn(B * S, E, generator=g).to(torch.bfloat16)
    return qkv.to(dev), do.to(dev)


def run_kernels(qkv, valid, do, B: int, S: int, heads: int):
    """dr_cuda_mha_fwd and dr_cuda_mha_bwd into NaN-filled buffers: (o, dqkv)."""
    from deeprec_b200 import _native
    from deeprec_b200._native import ptr, stream_ptr
    lib = _native.cuda()
    E = qkv.shape[1] // 3
    o = torch.full((B * S, E), float("nan"), dtype=torch.bfloat16, device=qkv.device)
    dqkv = torch.full((B * S, 3 * E), float("nan"), dtype=torch.bfloat16, device=qkv.device)
    assert lib.dr_cuda_mha_fwd(ptr(qkv), ptr(valid), B, S, E, heads, ptr(o), stream_ptr()) == 0
    assert lib.dr_cuda_mha_bwd(ptr(qkv), ptr(valid), ptr(o), ptr(do), B, S, E, heads, ptr(dqkv), stream_ptr()) == 0
    return o, dqkv


def _heads(t, B, S, heads, dh):
    """[B S, heads dh] -> float64 [B, heads, S, dh]."""
    return t.double().contiguous().view(B, S, heads, dh).permute(0, 2, 1, 3)


def oracle(qkv, valid, o, do, B: int, S: int, heads: int, dh: int):
    """float64 forward and backward with the bounds of the module docstring: dict name -> (reference, bound), each [B, heads, S, dh]."""
    E = heads * dh
    q, k, v = (_heads(qkv[:, i * E:(i + 1) * E], B, S, heads, dh) for i in range(3))
    scale = float(np.float32(1.0 / math.sqrt(dh)))
    keep = valid.bool()[:, None, None, :]                                           # [B, 1, 1, S] keys
    s = (q @ k.transpose(-1, -2)) * scale
    s = s.masked_fill(~keep, float("-inf"))
    P = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)                               # samples with no valid key: 0
    O = P @ v
    dO, Ok = _heads(do, B, S, heads, dh), _heads(o, B, S, heads, dh)
    D = (dO * Ok).sum(-1, keepdim=True)
    dP = dO @ v.transpose(-1, -2)
    dS = P * (dP - D) * scale
    A = P * (dO.abs() @ v.abs().transpose(-1, -2) + (dO.abs() * Ok.abs()).sum(-1, keepdim=True)) * scale
    dQ, dK, dV = dS @ k, dS.transpose(-1, -2) @ q, P.transpose(-1, -2) @ dO
    return {
        "o": (O, TOL * (P @ v.abs() + O.abs())),
        "dq": (dQ, TOL * (dS.abs() @ k.abs() + dQ.abs()) + TOL_A * (A @ k.abs())),
        "dk": (dK, TOL * (dS.abs().transpose(-1, -2) @ q.abs() + dK.abs()) + TOL_A * (A.transpose(-1, -2) @ q.abs())),
        "dv": (dV, TOL * (P.transpose(-1, -2) @ dO.abs() + dV.abs())),
    }


def check_kernels(B: int, S: int, heads: int, dh: int, kind: str, dev, seed: int = 0):
    E = heads * dh
    valid = make_valid(kind, B, S, seed + 31 * B + S).to(dev)
    qkv, do = make_case(B, S, heads, dh, seed + 7 * B + S, dev)
    o, dqkv = run_kernels(qkv, valid, do, B, S, heads)
    torch.cuda.synchronize()
    assert not bool(torch.isnan(o.float()).any()) and not bool(torch.isnan(dqkv.float()).any()), "an output element was not written"
    got = {"o": o, "dq": dqkv[:, :E], "dk": dqkv[:, E:2 * E], "dv": dqkv[:, 2 * E:]}
    got = {n: _heads(t, B, S, heads, dh) for n, t in got.items()}
    # exact zeros: dK, dV of masked keys; o, dq of samples with no valid key
    masked = ~valid.bool()[:, None, :, None].expand(B, heads, S, dh)
    assert bool((got["dk"][masked] == 0).all()) and bool((got["dv"][masked] == 0).all()), "dk / dv of a masked key is not exactly 0"
    empty = ~valid.bool().any(1)
    if bool(empty.any()):
        assert bool((got["o"][empty] == 0).all()) and bool((got["dq"][empty] == 0).all()), "o / dq of a sample with no valid key is not 0"
    for name, (ref, bound) in oracle(qkv, valid, o, do, B, S, heads, dh).items():
        err = (got[name] - ref).abs()
        bad = err > bound
        assert not bool(bad.any()), (name, float(err.max()), float((err - bound).max()), int(bad.sum()))


# ---- the layer ----------------------------------------------------------------------------------------------------------------------
LAYER_TOL = 2.0 ** -5


def encoder_layer(E: int, heads: int, dev, seed: int = 0, **kw):
    torch.manual_seed(seed)
    return torch.nn.TransformerEncoderLayer(E, heads, 4 * E, dropout=0.0, batch_first=True, device=dev, **kw)


def bst_valid(B: int, S: int, seed: int) -> torch.Tensor:
    """bool [B, S] as BST builds it: a random history mask (padding anywhere, some histories empty) and the last (target) position valid."""
    v = make_valid("random", B, S, seed).bool()
    v[::4, :-1] = False
    v[:, -1] = True
    return v


def layer_vs_module(B: int, S: int, E: int, heads: int, dev, seed: int = 0):
    """fused_encoder_layer against fp32 nn.TransformerEncoderLayer autograd: outputs at every position, dx and every parameter gradient, each
    within LAYER_TOL of the largest magnitude of its reference.  The fused path rounds the operands of its five GEMMs and of the attention
    products to bf16 (2^-9 relative each, 2^-8 with the rounding of their outputs); along the longest chain (in_proj, scores, P V, out_proj,
    norm1, linear1, linear2, norm2, and the same back) about a dozen such roundings add up, which 2^-5 covers with margin.  linear1's
    gradients are the exception: where a pre-activation lies within its rounding error of 0 the two ReLU masks differ, which drops or adds
    one whole term |d relu_out| |h| of the sum over rows rather than 2^-8 of it.  Their bound is therefore LAYER_TOL times the sum of the
    magnitudes of those terms (|d relu_out|^T |h| for the weight, sum |d relu_out| for the bias), from the reference's own activations."""
    from deeprec_b200.nn import fused_encoder_layer
    layer = encoder_layer(E, heads, dev, seed)
    ref = copy.deepcopy(layer)
    valid = bst_valid(B, S, seed).to(dev)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(B, S, E, generator=g).to(dev)
    R = torch.randn(B, S, E, generator=g).to(dev)
    x1 = x.clone().requires_grad_(True)
    y = fused_encoder_layer(x1, layer, valid)
    (y * R).sum().backward()
    x2 = x.clone().requires_grad_(True)
    seen = {}
    hooks = [ref.linear1.register_forward_hook(lambda m, i, o: seen.__setitem__("h", i[0].detach())),
             ref.linear2.register_forward_hook(lambda m, i, o: [i[0].register_hook(lambda g: seen.__setitem__("g", g.detach()))] and None)]
    y2 = ref(x2, src_key_padding_mask=~valid)
    (y2 * R).sum().backward()
    for hk in hooks:
        hk.remove()
    g_abs, h_abs = seen["g"].reshape(-1, seen["g"].shape[-1]).abs().double(), seen["h"].reshape(-1, E).abs().double()
    term_mag = {"linear1.weight": g_abs.t() @ h_abs, "linear1.bias": g_abs.sum(0)}

    def close(a, b, what):
        err, mag = float((a.detach().float() - b.detach().float()).abs().max()), float(b.detach().float().abs().max())
        assert err <= LAYER_TOL * mag + 1e-6, (what, err, mag)
    close(y, y2, "y")
    close(x1.grad, x2.grad, "dx")
    for (n, p), (_, pr) in zip(layer.named_parameters(), ref.named_parameters()):
        assert p.grad is not None and p.grad.dtype == torch.float32, n
        if n in term_mag:
            err = (p.grad.double() - pr.grad.double()).abs()
            assert bool((err <= LAYER_TOL * term_mag[n] + 1e-6).all()), (n, float(err.max()), float(term_mag[n].max()))
        else:
            close(p.grad, pr.grad, n)


# ---- BST on the engine ----------------------------------------------------------------------------------------------------------------
def bst_engine(dev, B, model=None, **kw):
    import pooled_bag_cases as K
    from deeprec_b200.models.rec_engine import din_engine
    model = model if model is not None else K.seq_model("bst", dev)
    return din_engine(model, B, K.L, table_rows=K.CARDS, device=None if dev.type == "cpu" else dev, **kw)


def run_bst_vs_replica(dev, graph: bool = False, steps: int = 6, B: int = 256):
    """Adagrad on the tables and the dense net, BST engine against the zoo model with nn.Embedding tables and nn.TransformerEncoderLayer: per-step
    loss, then rows of the user / item tables.  taobao_like has padded histories and empty ones."""
    import gru_cases as G
    import pooled_bag_cases as K
    from deeprec_b200.models.rec_engine import din_ids
    eng = bst_engine(dev, B, learning_rate=0.05)
    rep = G._seq_replica(eng, dev)
    opt = torch.optim.Adagrad(rep.parameters(), lr=0.05, initial_accumulator_value=0.1, eps=0.0)
    le, lr_ = [], []
    for s in range(steps):
        b = K.taobao_like(B, 100 + s)
        eng.load_batch(din_ids(b).to(dev), b["labels"].to(dev))
        if graph and s == 0:
            eng.capture(warmup=1)
        else:
            eng.train_step()
        le.append(eng.loss_value())
        loss = rep.loss({k: v.to(dev) for k, v in b.items()})
        opt.zero_grad()
        loss.backward()
        opt.step()
        lr_.append(loss.item())
    for a, r in zip(le, lr_):
        assert abs(a - r) < 0.03 * max(1.0, abs(r)), (le, lr_)
    hk = b["hist_item"].to(dev)
    keys = hk[hk >= 0][:64]
    assert (eng.tables[1].lookup(keys) - rep.item.emb.weight[keys]).abs().max().item() < 0.05
    uk = b["user"].to(dev)[:64]
    assert (eng.tables[0].lookup(uk) - rep.user.emb.weight[uk]).abs().max().item() < 0.05
    p = eng.predict()
    assert p.shape == (B,) and bool(((p >= 0) & (p <= 1)).all())
    return eng


def train_bst(dev, graph: bool, steps: int = 6, B: int = 1024, **kw):
    """Parameters, losses and every table row after ``steps`` BST engine steps."""
    import pooled_bag_cases as K
    from deeprec_b200.models.rec_engine import din_ids
    eng = bst_engine(dev, B, learning_rate=0.05, **kw)
    losses = []
    for s in range(steps):
        b = K.taobao_like(B, 1300 + s)
        eng.load_batch(din_ids(b).to(dev), b["labels"].to(dev))
        if graph and s == 0:
            eng.capture(warmup=1)
        else:
            eng.train_step()
        losses.append(eng.loss_value())
    probe = [torch.arange(c, device=eng.dev) for c in K.CARDS]
    return eng.params.clone(), losses, [eng.tables[t].lookup(probe[t]).clone() for t in range(3)]
