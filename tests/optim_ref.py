"""Float64 transcription of the reference optimizer rules, with a per-element error bound for one fp32 step of each.

The rules are transcribed from the reference (DeepRec, tensorflow/core/kernels/), not from csrc/common/ev_types.h, and this module calls no
native code: it is the oracle the kernel tests compare csrc/cuda/optimizer_kernels.cu, comm_kernels.cu and the host engine against.

Error bound.  Every quantity is an :class:`E`: its float64 value ``v`` computed from the kernel's fp32 inputs, and ``e``, a first-order bound on
how far an fp32 evaluation of the same expression can be from ``v``.  Each fp32 operation rounds its exact result r with |err| <= c u |r|,
u = 2^-24, and passes its operands' errors on to first order:
- + - * : c = 1 (round to nearest; an fma contraction only removes a rounding);
- / , sqrt, rsqrt : c = 4.  The library is built with --use_fast_math, so these are the approximate instructions (div.full, sqrt.approx,
  rsqrt.approx), each within 2 ulp, and one ulp of r is at most 2u|r|.  On the host (emulation, host engine) they are correctly rounded;
- pow(a, p) for lr_power != -0.5: __powf = ex2(p lg2 a).  lg2.approx is within 2^-22 (= 4u) absolute, the product rounds with u |p lg2 a|,
  and ex2 turns an absolute error d of its argument into a relative error d ln 2 plus its own 2 ulp:  c = 4 + ln2 (4 |p| + |p lg2 a|) + 1;
- a sum of n terms in an unspecified order: n u sum |t_i| (the FTRL row norm, the gradient accumulation);
- max / clamp and a branch on a comparison are exact; a branch taken within ``e`` of its threshold is ambiguous (see ftrl_*).
Propagation: e(a +- b) = e_a + e_b, e(a b) = |a| e_b + |b| e_a, e(a / b) = (e_a + |a / b| e_b) / |b|, e(sqrt a) = e_a / (2 sqrt a),
e(a^p) = |p| |a^p| e_a / a.  Kernel results must satisfy |x - v| <= 2 e + 1e-30 (factor 2 for the dropped second-order terms).  Hyper-
parameters enter as the fp32 values the kernel holds, so they carry no error; multi-step tests restart the oracle from the kernel's fp32
state after every step, so the bound never compounds.  Adam's alpha = lr sqrt(1 - b2^t) / (1 - b1^t) is an E of the fp32 beta powers the
kernel read.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24
C_APPROX = 4.0
LN2 = math.log(2.0)


def f32(x: float) -> float:
    """The fp32 value of a hyper-parameter, as the kernel holds it."""
    return float(torch.tensor(x, dtype=torch.float32))


class E:
    """A float64 value with a bound on the error of its fp32 evaluation."""

    def __init__(self, v, e=None):
        self.v = v.double() if torch.is_tensor(v) else torch.tensor(float(v), dtype=torch.float64)
        self.e = torch.zeros_like(self.v) if e is None else e

    @staticmethod
    def of(x) -> "E":
        return x if isinstance(x, E) else E(x)

    def _r(self, v, e, c=1.0) -> "E":
        return E(v, e + c * U * v.abs())

    def __add__(self, o):
        o = E.of(o)
        return self._r(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = E.of(o)
        return self._r(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return E.of(o) - self

    def __neg__(self):
        return E(-self.v, self.e)

    def __mul__(self, o):
        o = E.of(o)
        return self._r(self.v * o.v, self.v.abs() * o.e + o.v.abs() * self.e + self.e * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = E.of(o)
        q = self.v / o.v
        return self._r(q, (self.e + q.abs() * o.e) / (o.v.abs() - o.e).clamp_min(o.v.abs() * 0.5), C_APPROX)

    def __rtruediv__(self, o):
        return E.of(o) / self

    def sqrt(self) -> "E":
        s = self.v.clamp_min(0).sqrt()
        e = torch.where(s > 0, self.e / (2 * s).clamp_min(1e-300), self.e.sqrt())
        return self._r(s, e, C_APPROX)

    def rsqrt(self) -> "E":
        r = self.v.rsqrt()
        return self._r(r, 0.5 * r * self.e / self.v, C_APPROX)

    def pow(self, p: float) -> "E":
        r = self.v.pow(p)
        c = 4.0 + LN2 * (4.0 * abs(p) + (p * self.v.log2()).abs()) + 1.0
        return E(r, abs(p) * r * self.e / self.v + c * U * r)

    def abs(self) -> "E":
        return E(self.v.abs(), self.e)

    def sum(self, dim=-1) -> "E":
        n = self.v.shape[dim]
        return E(self.v.sum(dim), self.e.sum(dim) + n * U * self.v.abs().sum(dim))

    def maximum(self, floor: float) -> "E":
        return E(self.v.clamp_min(floor), self.e)

    def where(self, mask, other: "E") -> "E":
        other = E.of(other)
        return E(torch.where(mask, self.v, other.v), torch.where(mask, self.e, other.e.expand_as(self.e)))

    def tol(self):
        return 2.0 * self.e + 1e-30


def _branch(value: E, cond_lhs: E, threshold: float) -> E:
    """``value if cond_lhs > threshold else 0`` where value -> 0 as cond_lhs -> threshold (the FTRL shrinkage is continuous there): inside
    the comparison's own error band either branch is right, so the bound widens to cover 0."""
    take = cond_lhs.v > threshold
    amb = (cond_lhs.v - threshold).abs() <= 2 * cond_lhs.e
    out = value.where(take, E(torch.zeros_like(value.v)))
    out.e = torch.where(amb, torch.maximum(out.e, value.e + value.v.abs()), out.e)
    return out


# ---------------------------------------------------------------------------------------------------------------------------------------
# Element-wise rules.  w, s0, s1, g: E or float64 tensors.  Every function returns the new (w, s0, s1) it updates.

def sgd(w, g, lr):
    """training_ali_ops.cc:2871 (KvResourceSparseApplyGradientDescent): v -= lr * g."""
    return E.of(w) - f32(lr) * E.of(g)


def adagrad(w, a, g, lr):
    """training_ali_ops.cc:152-156: a += g^2 ; v -= lr * g * rsqrt(a)."""
    w, a, g = E.of(w), E.of(a), E.of(g)
    a = a + g * g
    return w - f32(lr) * g * a.rsqrt(), a


def adagrad_decay_due(global_step: int, decay_step: int, power: float) -> bool:
    """training_ali_ops.cc:946-950 (dense) and :1316 (EV): decay once when global_step / decay_step (integer division) exceeds the decay
    power; the power then advances by one."""
    return decay_step > 0 and (global_step // decay_step) > power


def adagrad_decay(w, a, g, lr, decay_now: bool, decay_rate, decay_baseline):
    """training_ali_ops.cc:1316-1323: if due, a = max(a * decay_rate, decay_baseline); a += g^2; v -= lr * g * rsqrt(a)."""
    w, a, g = E.of(w), E.of(a), E.of(g)
    if decay_now:
        a = (a * f32(decay_rate)).maximum(f32(decay_baseline))
    a = a + g * g
    return w - f32(lr) * g * a.rsqrt(), a


def adam_alpha(lr, beta1_power, beta2_power) -> E:
    """training_ali_ops.cc:1500: alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power), from the fp32 powers."""
    return f32(lr) * (1.0 - E(beta2_power)).sqrt() / (1.0 - E(beta1_power))


def adam(w, m, v, g, alpha: E, beta1, beta2, eps):
    """training_ali_ops.cc:1521-1523: m += (g - m)(1 - b1); v += (g^2 - v)(1 - b2); var -= m alpha / (sqrt(v) + eps)."""
    w, m, v, g = E.of(w), E.of(m), E.of(v), E.of(g)
    m = m + (g - m) * (1.0 - f32(beta1))
    v = v + (g * g - v) * (1.0 - f32(beta2))
    return w - m * alpha / (v.sqrt() + f32(eps)), m, v


def adamw(w, m, v, g, alpha: E, beta1, beta2, eps, weight_decay):
    """training_ali_ops.cc:3149-3153: Adam's moments; var -= m alpha / (sqrt(v) + eps) + weight_decay * var (decay on the old var)."""
    w, m, v, g = E.of(w), E.of(m), E.of(v), E.of(g)
    m = m + (g - m) * (1.0 - f32(beta1))
    v = v + (g * g - v) * (1.0 - f32(beta2))
    return w - (m * alpha / (v.sqrt() + f32(eps)) + f32(weight_decay) * w), m, v


def adam_async(w, m, v, g, alpha: E, beta1, beta2, eps):
    """training_ali_ops.cc:2475-2477: m = m b1 + g (1 - b1); v = v b2 + g^2 (1 - b2); var -= m alpha / (sqrt(v) + eps)."""
    w, m, v, g = E.of(w), E.of(m), E.of(v), E.of(g)
    m = m * f32(beta1) + g * (1.0 - f32(beta1))
    v = v * f32(beta2) + g * g * (1.0 - f32(beta2))
    return w - m * alpha / (v.sqrt() + f32(eps)), m, v


def adam_async_rmsprop(w, m, v, g, lr, beta1, beta2, eps):
    """training_ali_ops.cc:2425-2432 (apply_sparse_rmsprop): v = v b2 + g^2 (1 - b2); m = m b1 + rsqrt(v + eps) lr g; var -= m."""
    w, m, v, g = E.of(w), E.of(m), E.of(v), E.of(g)
    v = v * f32(beta2) + g * g * (1.0 - f32(beta2))
    m = m * f32(beta1) + (v + f32(eps)).rsqrt() * f32(lr) * g
    return w - m, m, v


def _ftrl_pow(x: E, lr_power: float) -> E:
    return x.sqrt() if f32(lr_power) == -0.5 else x.pow(-f32(lr_power))


def ftrl_ev(w, accum, linear, g, lr, l1, l2, l2_shrinkage, lr_power):
    """EmbeddingVariable FTRL, KvSparseApplyFtrlOp (training_ali_ops.cc:558-590), row-wise over the last axis:
    gs = g + 2 l2_shrinkage var; new_accum = accum + gs^2; linear += gs - (new_accum^-p - accum^-p) / lr * var;
    n = ||linear||; var = n > l1 ? (l1 - n) / ((new_accum^-p / lr + 2 l2) n) * linear : 0; accum += g^2 (the raw gradient)."""
    w, a, lin, g = E.of(w), E.of(accum), E.of(linear), E.of(g)
    lr, l1, l2 = f32(lr), f32(l1), f32(l2)
    gs = g + 2.0 * f32(l2_shrinkage) * w
    na = a + gs * gs
    lin = lin + (gs - (_ftrl_pow(na, lr_power) - _ftrl_pow(a, lr_power)) / lr * w)
    norm = (lin * lin).sum(-1).sqrt()
    eta_rec = _ftrl_pow(na, lr_power) / lr
    nb = E(norm.v.unsqueeze(-1).expand_as(lin.v), norm.e.unsqueeze(-1).expand_as(lin.v))
    coef = (l1 - nb) / ((eta_rec + 2.0 * l2) * nb)
    w_new = _branch(coef * lin, nb, l1)
    return w_new, a + g * g, lin


def ftrl_dense(w, accum, linear, g, lr, l1, l2, l2_shrinkage, lr_power):
    """Dense FTRL, ApplyFtrlV2 (training_ops.cc:370-396), element-wise:  gs = g + 2 l2_shrinkage var; new_accum = accum + g^2 (the RAW
    gradient); linear += gs - (new_accum^-p - accum^-p) / lr * var; var = |linear| > l1 ? (sign(linear) l1 - linear) / (new_accum^-p / lr
    + 2 l2) : 0; accum = new_accum."""
    w, a, lin, g = E.of(w), E.of(accum), E.of(linear), E.of(g)
    lr, l1, l2 = f32(lr), f32(l1), f32(l2)
    gs = g + 2.0 * f32(l2_shrinkage) * w
    na = a + g * g
    lin = lin + (gs - (_ftrl_pow(na, lr_power) - _ftrl_pow(a, lr_power)) / lr * w)
    quad = _ftrl_pow(na, lr_power) / lr + 2.0 * l2
    w_new = _branch((l1 * lin.v.sign() - lin) / quad, lin.abs(), l1)
    return w_new, na, lin


# ---------------------------------------------------------------------------------------------------------------------------------------
# Dispatch by the kernel's DrOptKind (csrc/common/ev_types.h).

SGD, ADAGRAD, ADAGRAD_DECAY, ADAM, ADAM_ASYNC, ADAMW, FTRL, ADAM_ASYNC_RMSPROP = range(8)
NUM_SLOTS = {SGD: 0, ADAGRAD: 1, ADAGRAD_DECAY: 1, ADAM: 2, ADAM_ASYNC: 2, ADAMW: 2, FTRL: 2, ADAM_ASYNC_RMSPROP: 2}


def apply(kind: int, hp: dict, w, s0, s1, g, decay_now: bool = False, dense: bool = True):
    """One step of rule ``kind`` with hyper-parameters ``hp`` (the fields of DrOptHyper; beta powers as the kernel held them).
    ``dense`` selects the FTRL form: ApplyFtrlV2 for dense variables, KvSparseApplyFtrlOp (row-wise) for EmbeddingVariable rows.
    Returns (w, s0, s1) as E; slots the rule does not have come back as given."""
    if kind == SGD:
        return sgd(w, g, hp["lr"]), E.of(s0), E.of(s1)
    if kind == ADAGRAD:
        return (*adagrad(w, s0, g, hp["lr"]), E.of(s1))
    if kind == ADAGRAD_DECAY:
        return (*adagrad_decay(w, s0, g, hp["lr"], decay_now, hp["decay_rate"], hp["decay_baseline"]), E.of(s1))
    if kind == ADAM_ASYNC_RMSPROP:
        return adam_async_rmsprop(w, s0, s1, g, hp["lr"], hp["beta1"], hp["beta2"], hp["epsilon"])
    if kind == FTRL:
        f = ftrl_dense if dense else ftrl_ev
        return f(w, s0, s1, g, hp["lr"], hp["l1"], hp["l2"], hp["l2_shrinkage"], hp["lr_power"])
    alpha = adam_alpha(hp["lr"], hp["beta1_power"], hp["beta2_power"])
    if kind == ADAM:
        return adam(w, s0, s1, g, alpha, hp["beta1"], hp["beta2"], hp["epsilon"])
    if kind == ADAMW:
        return adamw(w, s0, s1, g, alpha, hp["beta1"], hp["beta2"], hp["epsilon"], hp["weight_decay"])
    if kind == ADAM_ASYNC:
        return adam_async(w, s0, s1, g, alpha, hp["beta1"], hp["beta2"], hp["epsilon"])
    raise ValueError(kind)
