"""Float64 transcription of the dense DLRM step's memory-bound ops, with a bound on the error of their fp32 evaluation.

The rules are transcribed from the reference (DeepRec), not from csrc/cuda/dense_kernels.cu, and this module calls no native code.  It is the
oracle the kernel tests (tests/dense_cases.py) compare k_colstats, the BatchNorm kernels, the fold / fix-up, the logit head, weight packing and
input casting against.

Values are :class:`optim_ref.E`: a float64 value ``v`` computed from the kernel's own inputs and ``e``, a first-order bound on how far an fp32
evaluation of the same expression can be from it (u = 2^-24 per + - *, 4 u for rsqrt / division / the exp and log1p library calls; see the
optim_ref docstring).  A result passes when |x - v| <= 2 e + 1e-30.  On top of that:

- bf16 rounding.  A value stored as bf16 gets a relative allowance of 2^-9 on top of its fp32 error (tol = 2 e then covers the 2^-8 half ulp
  of round-to-nearest-even).
- Exact products.  The product of two bf16 values has at most 16 significant bits, so it is exact in fp32 (:func:`mul_exact`).
- Summation depth.  The batch sums of k_colstats, k_bn_bwd_apply_v2 and k_head are added in a tree: each thread adds its rows in order, the
  row-groups (warps for the head) of a block are added in order, k_det_colsum adds the block partials in order, and the result is added into
  the destination.  Its depth is at most rows_per_thread + rows_par + grid + 1 <= ceil(B / rows_par) + rows_par + 2, because grid <=
  ceil(B / rows_par) / 2 (every block gets at least two row-groups).  So the error is at most depth u (sum |x| + |S0|) whatever the grid, and
  the same bound holds on an H100 and on the emulation (num_sms() == 2).  It is much tighter than the n u of ``E.sum``: dropping one row of a
  batch of B = 4097 at N = 512 (rows_par = 4) moves a sum by about sum |x| / 4097, while the bound is 1030 u sum |x| = 6e-5 sum |x|.
- The exp of the head is __expf = ex2.approx(z log2 e) on the device: the rounding of z log2 e is an absolute error u |z| log2 e of the
  exponent, i.e. a relative error u |z| of the result, plus 2 ulp of ex2.  Flush-to-zero (fast math) can turn results below 2^-126 into 0,
  so values that may be subnormal carry an absolute 2^-126.
"""
from __future__ import annotations

import torch

from optim_ref import C_APPROX, E, U, f32

UB = 2.0 ** -9          # bf16 store allowance: tol = 2 e makes it the 2^-8 half ulp of round-to-nearest-even
TINY = 2.0 ** -126      # flush-to-zero of subnormal results


def bf16(x: E) -> E:
    """The value of ``x`` after it is stored as bf16."""
    return E(x.v, x.e + UB * x.v.abs())


def exact(t: torch.Tensor) -> E:
    """An input as the kernel reads it (a bf16 or fp32 tensor): no error."""
    return E(t.detach().double().cpu())


def mul_exact(a: E, b: E) -> E:
    """a * b of two bf16 values: the fp32 product is exact, only the operands' errors pass on."""
    return E(a.v * b.v, a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e)


def tree_sum(x: E, depth: int, dim: int = 0, init: E | None = None) -> E:
    """``init + sum(x, dim)`` added in a tree of ``depth`` levels (the block reductions and k_det_colsum, see the module docstring)."""
    v, a, e = x.v.sum(dim), x.v.abs().sum(dim), x.e.sum(dim)
    if init is not None:
        v, a, e = v + init.v, a + init.v.abs(), e + init.e
    return E(v, e + depth * U * a)


def colsum_depth(B: int, N: int) -> int:
    """Depth bound of a k_colstats / k_bn_bwd_apply_v2 batch sum at B rows of N columns (8 columns per thread, 256 threads)."""
    rows_par = 256 // (N // 8)
    return -(-B // rows_par) + rows_par + 2


def head_depth(B: int) -> int:
    """Depth bound of a k_head batch sum: 8 warps per block take the place of rows_par; +1 for the per-warp scaling of the loss."""
    return -(-B // 8) + 8 + 3


def inv_batch(B: int) -> E:
    """1.0f / (float)B as the wrappers compute it."""
    return E(torch.tensor(1.0 / B, dtype=torch.float64), torch.tensor(U / B, dtype=torch.float64))


# ---------------------------------------------------------------------------------------------------------------------------------------
# BatchNorm forward.  tf.layers.batch_normalization on the 2-D activations of modelzoo/dlrm/train.py:181 takes the non-fused path:
#   keras/layers/normalization.py:736-739  mean, variance = self._moments(inputs, ...)  -> nn_impl.py:1271-1321 nn.moments: the mean and the
#       BIASED variance mean((x - mean)^2) (divided by B, not B - 1);
#   nn_impl.py:1527-1533  inv = rsqrt(variance + eps) * scale;  y = x * inv + (offset - mean * inv);
#   keras/layers/normalization.py:467-478  _assign_moving_average: moving -= (moving - value) * (1 - momentum), i.e.
#       moving = momentum * moving + (1 - momentum) * value, with value the batch mean and the biased batch variance;
#   keras/layers/normalization.py:741-748  at inference (training = False) mean / variance are the moving statistics.
# The kernels compute the variance in one pass, S2 / B - mean^2, clamped at 0: the bound below is that of the one-pass form, so it grows
# with mean^2 / var (the cancellation), which a two-pass variance would not have.

def bn_stats(S1: E, S2: E, B: int) -> tuple[E, E]:
    """Batch mean and biased variance from the column sums S1 = sum a, S2 = sum a^2."""
    ib = inv_batch(B)
    m = S1 * ib
    var = (S2 * ib - m * m).maximum(0.0)
    return m, var


def bn_scale_shift(m: E, var: E, gamma: E, beta: E, eps: float) -> tuple[E, E, E]:
    """rstd = rsqrt(var + eps), scale = gamma rstd, shift = beta - mean scale."""
    rs = (var + f32(eps)).rsqrt()
    sc = gamma * rs
    return rs, sc, beta - m * sc


def moving_average(moving: E, value: E, momentum: float) -> E:
    """moving = momentum moving + (1 - momentum) value, with the fp32 momentum (1 - momentum is then exact for momentum in [0.5, 1])."""
    m = f32(momentum)
    return moving * m + value * (1.0 - m)


def bn_forward(S1: E, S2: E, B: int, gamma: E, beta: E, eps: float, momentum: float, running_mean: E, running_var: E, training: bool):
    """dict of mean, rstd, scale, shift and the running statistics after one k_bn_finalize / k_bn_fold."""
    if training:
        m, var = bn_stats(S1, S2, B)
        rm, rv = moving_average(running_mean, m, momentum), moving_average(running_var, var, momentum)
    else:
        m, var, rm, rv = running_mean, running_var, running_mean, running_var
    rs, sc, sh = bn_scale_shift(m, var, gamma, beta, eps)
    return dict(mean=m, var=var, rstd=rs, scale=sc, shift=sh, running_mean=rm, running_var=rv)


def bn_apply(a: E, scale: E, shift: E) -> E:
    """y = bf16(a scale + shift) (with or without an fma: the bound of the two-rounding form covers both)."""
    return bf16(a * scale + shift)


def bn_fold(W: E, b: E, scale: E, shift: E, K: int, Kp: int) -> tuple[E, E]:
    """Fold y = s a + t into the next Linear: W' = bf16(W diag(s)) (0 in the padding columns K <= k < Kp), b' = b + W t over k < K."""
    s = E(torch.cat([scale.v, torch.zeros(Kp - K, dtype=torch.float64)]), torch.cat([scale.e, torch.zeros(Kp - K, dtype=torch.float64)]))
    t = E(torch.cat([shift.v, torch.zeros(Kp - K, dtype=torch.float64)]), torch.cat([shift.e, torch.zeros(Kp - K, dtype=torch.float64)]))
    Wf = bf16(W * s)
    prod = W * t
    depth = -(-Kp // 256) + 5 + 8 + 1               # per-thread k loop, warp shuffle tree, 8 warps in order, + b
    bf = E(b.v + prod.v.sum(-1), b.e + prod.e.sum(-1) + depth * U * (prod.v.abs().sum(-1) + b.v.abs()))
    return Wf, bf


# ---------------------------------------------------------------------------------------------------------------------------------------
# BatchNorm backward: the gradient of y = gamma xhat + beta, xhat = (a - mean) rstd through the batch statistics (the reference gets it from
# TF's autodiff of the graph above):
#   dbeta = sum dy;  dgamma = sum dy xhat = rstd (sum dy a - mean sum dy);  c1 = dbeta / B;  c2 = dgamma / B;
#   da = relu'(a) scale (dy - c1 - xhat c2)   (relu' of the layer's ReLU, whose output a is, folded in: a > 0).

def bn_bwd_finalize(S1: E, S2: E, B: int, mean: E, rstd: E, dgamma0: E, dbeta0: E, grad_accum_scale: float = 1.0):
    """From S1 = sum dy, S2 = sum dy a: dgamma += s dxhat, dbeta += s sum dy, c1, c2 (dict)."""
    ib = inv_batch(B)
    dxhat = rstd * (S2 - mean * S1)
    return dict(dgamma=dgamma0 + dxhat * grad_accum_scale, dbeta=dbeta0 + S1 * grad_accum_scale, c1=S1 * ib, c2=dxhat * ib)


def bn_bwd_apply(dy: E, a: E, scale: E, mean: E, rstd: E, c1: E, c2: E, relu_mask: bool) -> tuple[E, torch.Tensor]:
    """(da before its bf16 store, relu mask as a bool tensor).  Columns broadcast along dim 0."""
    xhat = (a - mean) * rstd
    g = scale * (dy - c1 - xhat * c2)
    keep = a.v > 0 if relu_mask else torch.ones_like(a.v, dtype=torch.bool)
    return g.where(keep, E(torch.zeros_like(g.v))), keep


def dw_fixup(G: E, db: E, scale: E, shift: E, K: int, Kp: int) -> E:
    """dW = G diag(s) + db t^T over k < K, 0 in the padding columns (the weight gradient of a Linear whose input is a folded BatchNorm)."""
    out = E(G.v[:, :K], G.e[:, :K]) * scale + E(db.v[:, None], db.e[:, None]) * shift
    v = torch.zeros(G.v.shape[0], Kp, dtype=torch.float64)
    e = torch.zeros_like(v)
    v[:, :K], e[:, :K] = out.v, out.e
    return E(v, e)


# ---------------------------------------------------------------------------------------------------------------------------------------
# Logit head: Dense(1) + sigmoid + binary cross-entropy, modelzoo/dlrm/train.py:228-243 (tf.layers.dense, tf.math.sigmoid,
# tf.keras.losses.BinaryCrossentropy on the logits).  The loss of one row is the stable form of nn_impl.py:186-191
# (sigmoid_cross_entropy_with_logits): max(z, 0) - z y + log1p(exp(-|z|)); the mean over the global batch is sum * inv_batch.
# Backward: dz = (p - y) inv_batch;  dh = dz w (* relu'(h));  dw = sum_b dz h;  db = sum_b dz;  dbias_h = sum_b dh (before the bf16 store).

def expm(x: E) -> E:
    """exp(x) as __expf evaluates it (module docstring); x <= 0 here, so the result is at most 1."""
    r = x.v.exp()
    return E(r, r * x.e + (C_APPROX + x.v.abs()) * U * r + TINY)


def log1p(x: E) -> E:
    r = x.v.log1p()
    return E(r, x.e / (1.0 + x.v) + C_APPROX * U * r.abs() + TINY)


def head(h: E, w: E, b0: float, labels: torch.Tensor, inv: float, relu_mask: bool = True):
    """dict of the per-row terms z, p, loss * inv, dz, dh (before its bf16 store) and dz h; the batch sums (loss, dw, db = sum dz,
    dbias_h = sum dh) are taken by the caller with :func:`tree_sum` at the head's depth."""
    K = h.v.shape[1]
    R = K // 256
    prod = h * w                                      # fp32 h * w (w is fp32): one rounding, or none inside an fma
    dot = E(prod.v.sum(1), prod.e.sum(1) + (8 * R + 5) * U * prod.v.abs().sum(1))
    z = dot + b0
    ez = expm(-z)                                     # 1 / (1 + exp(-z)) with z of either sign
    p = 1.0 / (1.0 + ez)
    p = E(p.v, p.e + TINY)
    y = labels.double().cpu()
    az = z.abs()
    loss = z.maximum(0.0) - z * y + log1p(expm(-az))
    loss_i = loss * inv
    dz = (p - y) * inv
    dzb = E(dz.v[:, None], dz.e[:, None])
    dh = dzb * w
    if relu_mask:
        dh = dh.where(h.v > 0, E(torch.zeros_like(dh.v)))
    dwt = dzb * h
    return dict(z=z, p=p, loss=loss_i, dz=dz, dh=dh, dw=dwt)


def cast_pad(x: torch.Tensor, Cp: int) -> torch.Tensor:
    """fp32 [B, C] -> bf16 [B, Cp] zero padded: round to nearest even, which is what torch's .bfloat16() does."""
    out = torch.zeros(x.shape[0], Cp, dtype=torch.bfloat16)
    out[:, : x.shape[1]] = x.detach().cpu().bfloat16()
    return out
