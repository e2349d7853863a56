"""Optimizers that update both dense parameters and EmbeddingVariables.

Rule parity (all eight sparse rules share ``csrc/common/ev_types.h::dr_apply_elem``):
  Adagrad            python/training/adagrad.py:141-160, kernels/training_ali_ops.cc:73-210
  AdagradDecay       python/training/adagrad_decay.py:35, training_ali_ops.cc:1203
  Adam / AdamW       training_ali_ops.cc:1396 / :3016, weight_decay_optimizers.py:297
  AdamAsync          python/training/adam_async.py:40, training_ali_ops.cc:2298 (+ sparse RMSProp)
  Ftrl               training_ali_ops.cc:431
  GradientDescent    training_ali_ops.cc:2871
Sparse gradients are de-duplicated with unique-with-counts + segment-sum before the apply
(python/training/optimizer.py:91,1101); the per-key counts feed frequency admission.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

import torch
from torch import nn

from .._native import OptHyper
from ..embedding_variable import DynamicEmbeddingVariable, EmbeddingVariable, PartitionedEmbeddingVariable

OPT_SGD, OPT_ADAGRAD, OPT_ADAGRAD_DECAY, OPT_ADAM, OPT_ADAM_ASYNC, OPT_ADAMW, OPT_FTRL, OPT_ADAM_ASYNC_RMSPROP = range(8)

# ---- the fused engines' optimizer table (models/dlrm_engine.py, models/rec_engine.py): one rule for the dense net and the tables -------
OPT_KIND = {"sgd": OPT_SGD, "gradientdescent": OPT_SGD, "adagrad": OPT_ADAGRAD, "adagraddecay": OPT_ADAGRAD_DECAY,
            "adam": OPT_ADAM, "adamasync": OPT_ADAM_ASYNC, "adamw": OPT_ADAMW, "ftrl": OPT_FTRL}
OPT_SLOTS = {OPT_SGD: 0, OPT_ADAGRAD: 1, OPT_ADAGRAD_DECAY: 1, OPT_ADAM: 2, OPT_ADAM_ASYNC: 2, OPT_ADAMW: 2, OPT_FTRL: 2}


def slot0_init(kind: int, initial_accumulator_value: float) -> float:
    """The value slot 0 starts at: the accumulator of Adagrad / AdagradDecay / FTRL, the first moment (0) otherwise."""
    return initial_accumulator_value if kind in (OPT_ADAGRAD, OPT_ADAGRAD_DECAY, OPT_FTRL) else 0.0


def engine_hyper(kind: int, lr: float, initial_accumulator_value: float) -> OptHyper:
    """The fused engines' hyper-parameters: the reference optimizers' defaults at learning rate ``lr``, global step 0."""
    hp = OptHyper()
    hp.kind, hp.lr = kind, lr
    hp.beta1, hp.beta2, hp.epsilon = 0.9, 0.999, 1e-8
    hp.beta1_power, hp.beta2_power = 0.9, 0.999
    hp.weight_decay, hp.l1, hp.l2, hp.l2_shrinkage, hp.lr_power = 0.0, 0.0, 0.0, 0.0, -0.5
    hp.decay_rate, hp.decay_baseline, hp.init_accum = 0.9, initial_accumulator_value, initial_accumulator_value
    hp.decay_step, hp.global_step = 100000, 0
    return hp


class GlobalStep:
    """``tf.train.get_or_create_global_step`` analogue."""

    def __init__(self, value: int = 0):
        self.value = int(value)

    def increment(self) -> int:
        self.value += 1
        return self.value

    def __int__(self) -> int:
        return self.value


_GLOBAL_STEP = GlobalStep()


def get_or_create_global_step() -> GlobalStep:
    return _GLOBAL_STEP


def collect_embedding_variables(module_or_list) -> List[EmbeddingVariable]:
    out: List[EmbeddingVariable] = []
    items = module_or_list.modules() if isinstance(module_or_list, nn.Module) else module_or_list
    for m in items:
        if isinstance(m, EmbeddingVariable):
            out.append(m)
        elif isinstance(m, (PartitionedEmbeddingVariable, DynamicEmbeddingVariable)) and not isinstance(module_or_list, nn.Module):
            out.extend(x for x in m.modules() if isinstance(x, EmbeddingVariable))
    seen, uniq = set(), []
    for e in out:
        if id(e) not in seen:
            seen.add(id(e)); uniq.append(e)
    return uniq


class DeepRecOptimizer(torch.optim.Optimizer):
    """Base: ``params`` are dense tensors (anchor parameters of EVs are filtered out),
    ``embedding_variables`` are updated with the native sparse apply."""

    kind = OPT_SGD
    slot_names: Sequence[str] = ()
    has_scalars = False

    def __init__(self, params: Iterable, embedding_variables=None, lr: float = 0.01,
                 global_step: Optional[GlobalStep] = None, **defaults):
        evs = collect_embedding_variables(embedding_variables) if embedding_variables is not None else []
        anchors = {id(e._anchor) for e in evs}
        if isinstance(params, nn.Module):
            if embedding_variables is None:
                evs = collect_embedding_variables(params)
                anchors = {id(e._anchor) for e in evs}
            params = params.parameters()
        plist = [p for p in params if id(p) not in anchors and p.numel() > 0]
        if not plist:
            plist = [torch.zeros(1, requires_grad=True)]   # torch.optim needs a non-empty list
            self._no_dense = True
        else:
            self._no_dense = False
        defaults = dict(lr=lr, **defaults)
        super().__init__(plist, defaults)
        self.evs = evs
        self.global_step = global_step or get_or_create_global_step()
        self.beta1_power = defaults.get("beta1", 0.0)
        self.beta2_power = defaults.get("beta2", 0.0)
        for e in self.evs:
            e._set_slots(self.slot_names, self._slot_init(), self.has_scalars, owner=id(self) & 0x7FFFFFFF)

    # -- subclass hooks -----------------------------------------------------------------------
    def _slot_init(self) -> List[float]:
        return [0.0] * len(self.slot_names)

    def _hyper(self, group) -> OptHyper:
        hp = OptHyper()
        hp.kind = self.kind
        hp.lr = float(group["lr"])
        hp.beta1 = float(group.get("beta1", 0.9)); hp.beta2 = float(group.get("beta2", 0.999))
        hp.epsilon = float(group.get("eps", 1e-8))
        hp.beta1_power = float(self.beta1_power); hp.beta2_power = float(self.beta2_power)
        hp.weight_decay = float(group.get("weight_decay", 0.0))
        hp.l1 = float(group.get("l1", 0.0)); hp.l2 = float(group.get("l2", 0.0))
        hp.l2_shrinkage = float(group.get("l2_shrinkage", 0.0)); hp.lr_power = float(group.get("lr_power", -0.5))
        hp.decay_rate = float(group.get("decay_rate", 1.0)); hp.decay_baseline = float(group.get("decay_baseline", 0.0))
        hp.init_accum = float(group.get("initial_accumulator_value", 0.1))
        hp.decay_step = int(group.get("decay_step", 0))
        hp.global_step = int(self.global_step)
        hp.apply_sparse_rmsprop = int(bool(group.get("apply_sparse_rmsprop", False)))
        return hp

    def _dense_update(self, p: torch.Tensor, g: torch.Tensor, state: dict, group: dict, hp: OptHyper) -> None:
        p.add_(g, alpha=-group["lr"])

    def _dense_update_many(self, ps: List[torch.Tensor], gs: List[torch.Tensor], states: List[dict], group: dict, hp: OptHyper) -> None:
        """All dense parameters of a group at once.  Subclasses with a multi-tensor (``torch._foreach_*``) form override this: a model
        with dozens of small parameters then costs a handful of launches per step instead of several per parameter."""
        for p, g, st in zip(ps, gs, states):
            self._dense_update(p, g, st, group, hp)

    def _sparse_param_update(self, p: torch.Tensor, grad: torch.Tensor, state: dict, group: dict, hp: OptHyper) -> None:
        """``SparseApply{Adagrad, AdagradDecay, Adam, AdamAsync, Ftrl, ...}`` on a plain (non-EV) variable (training_ali_ops.cc:994,2111):
        the optimizer's rule applied to the touched rows only (lazy: untouched rows keep their slots -- no decay, no update)."""
        g = grad.coalesce()
        idx, vals = g.indices()[0], g.values()
        if idx.numel() == 0:
            return
        if not state:      # slots start from the rule's own initial values (uniform per element): run the rule once on a zero row to get them
            tmp: dict = {}
            z = torch.zeros_like(p[:1])
            self._dense_update(z, torch.zeros_like(z), tmp, group, hp)
            for k, v in tmp.items():
                state[k] = v.expand_as(p).clone() if torch.is_tensor(v) and v.dim() == p.dim() else v
        rows = p.data.index_select(0, idx)
        sub = {k: (v.index_select(0, idx) if torch.is_tensor(v) and v.dim() == p.dim() and v.shape[0] == p.shape[0] else v) for k, v in state.items()}
        self._dense_update(rows, vals.to(rows.dtype), sub, group, hp)
        p.data.index_copy_(0, idx, rows)
        for k, v in sub.items():
            if torch.is_tensor(v) and v.dim() == p.dim() and torch.is_tensor(state[k]) and state[k].shape[0] == p.shape[0]:
                state[k].index_copy_(0, idx, v)
            else:
                state[k] = v

    def _after_step(self, group) -> None:
        pass

    # -------------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        group = self.param_groups[0]
        hp = self._hyper(group)
        if not self._no_dense:
            for g_ in self.param_groups:
                ps = [p for p in g_["params"] if p.grad is not None and not p.grad.is_sparse]
                if ps:
                    self._dense_update_many(ps, [p.grad for p in ps], [self.state[p] for p in ps], g_, hp)
                for p in g_["params"]:
                    if p.grad is not None and p.grad.is_sparse:          # nn.Embedding(sparse=True): SparseApply* on a plain variable
                        self._sparse_param_update(p, p.grad, self.state[p], g_, hp)
        from ..ops.host_group import apply_group_pending
        apply_group_pending(self.evs, hp)          # grouped host lookups: one native dedup + apply call per group
        for ev in self.evs:
            if ev.device.type == "cuda":
                if ev._table is not None:
                    ev._table.apply_step(hp)      # one fused launch per (device, dim) context; idempotent
                continue
            if hasattr(ev.table, "apply_segments"):           # plain host table: one native dedup + apply over all recorded segments
                segs = ev.pop_sparse_segments()
                if segs:
                    ev.table.apply_segments(segs, hp)
                continue
            sg = ev.pop_sparse_grads()
            if sg is None:
                continue
            ids, grads = sg
            ev.table.apply_raw(ids, grads, hp)
        self._after_step(group)
        self.global_step.increment()
        return loss

    def zero_grad(self, set_to_none: bool = True):
        super().zero_grad(set_to_none)
        for ev in self.evs:
            ev._pending.clear()
            ev._group_pending.clear()


class GradientDescentOptimizer(DeepRecOptimizer):
    kind = OPT_SGD

    def _dense_update_many(self, ps, gs, states, group, hp):
        torch._foreach_add_(ps, gs, alpha=-group["lr"])


class AdagradOptimizer(DeepRecOptimizer):
    kind = OPT_ADAGRAD
    slot_names = ("accumulator",)

    def __init__(self, params, embedding_variables=None, lr=0.01, initial_accumulator_value=0.1, **kw):
        self._init_acc = float(initial_accumulator_value)
        super().__init__(params, embedding_variables, lr, initial_accumulator_value=initial_accumulator_value, **kw)

    def _slot_init(self):
        return [self._init_acc]

    def _dense_update(self, p, g, state, group, hp):
        if "acc" not in state:
            state["acc"] = torch.full_like(p, group["initial_accumulator_value"])
        a = state["acc"]
        a.addcmul_(g, g)
        p.addcdiv_(g, a.sqrt(), value=-group["lr"])

    def _dense_update_many(self, ps, gs, states, group, hp):
        for p, st in zip(ps, states):
            if "acc" not in st:
                st["acc"] = torch.full_like(p, group["initial_accumulator_value"])
        accs = [st["acc"] for st in states]
        torch._foreach_addcmul_(accs, gs, gs)
        torch._foreach_addcdiv_(ps, gs, torch._foreach_sqrt(accs), value=-group["lr"])


class AdagradDecayOptimizer(DeepRecOptimizer):
    """Accumulator is decayed by ``accumulator_decay_rate`` every ``accumulator_decay_step`` global
    steps and floored at ``accumulator_baseline`` (adagrad_decay.py:35-120)."""
    kind = OPT_ADAGRAD_DECAY
    slot_names = ("accumulator",)
    has_scalars = True

    def __init__(self, params, embedding_variables=None, lr=0.01, initial_accumulator_value=0.1,
                 accumulator_decay_step=100000, accumulator_decay_rate=0.9, **kw):
        self._init_acc = float(initial_accumulator_value)
        super().__init__(params, embedding_variables, lr, initial_accumulator_value=initial_accumulator_value,
                         decay_step=int(accumulator_decay_step), decay_rate=float(accumulator_decay_rate),
                         decay_baseline=float(initial_accumulator_value), **kw)

    def _slot_init(self):
        return [self._init_acc]

    def _dense_update(self, p, g, state, group, hp):
        if "acc" not in state:
            state["acc"] = torch.full_like(p, group["initial_accumulator_value"])
            state["decay_power"] = 0
        a = state["acc"]
        if group["decay_step"] > 0 and int(self.global_step) // group["decay_step"] > state["decay_power"]:
            a.mul_(group["decay_rate"]).clamp_(min=group["decay_baseline"])
            state["decay_power"] += 1
        a.addcmul_(g, g)
        p.addcdiv_(g, a.sqrt(), value=-group["lr"])


class AdamOptimizer(DeepRecOptimizer):
    kind = OPT_ADAM
    slot_names = ("m", "v")

    def __init__(self, params, embedding_variables=None, lr=0.001, beta1=0.9, beta2=0.999, eps=1e-8, **kw):
        super().__init__(params, embedding_variables, lr, beta1=beta1, beta2=beta2, eps=eps, **kw)

    def _dense_update(self, p, g, state, group, hp):
        if "m" not in state:
            state["m"] = torch.zeros_like(p); state["v"] = torch.zeros_like(p)
        m, v = state["m"], state["v"]
        alpha = group["lr"] * (1 - self.beta2_power) ** 0.5 / (1 - self.beta1_power)
        m.add_(g - m, alpha=1 - group["beta1"])
        v.add_(g * g - v, alpha=1 - group["beta2"])
        p.addcdiv_(m, v.sqrt().add_(group["eps"]), value=-alpha)

    def _moments(self, ps, gs, states, group):
        """m <- m + (1 - b1)(g - m), v <- v + (1 - b2)(g^2 - v) for every parameter; returns (ms, sqrt(v) + eps, step size)."""
        for p, st in zip(ps, states):
            if "m" not in st:
                st["m"] = torch.zeros_like(p); st["v"] = torch.zeros_like(p)
        ms, vs = [st["m"] for st in states], [st["v"] for st in states]
        torch._foreach_lerp_(ms, gs, 1 - group["beta1"])
        torch._foreach_lerp_(vs, torch._foreach_mul(gs, gs), 1 - group["beta2"])
        denom = torch._foreach_sqrt(vs)
        torch._foreach_add_(denom, group["eps"])
        return ms, denom, group["lr"] * (1 - self.beta2_power) ** 0.5 / (1 - self.beta1_power)

    def _dense_update_many(self, ps, gs, states, group, hp):
        ms, denom, alpha = self._moments(ps, gs, states, group)
        torch._foreach_addcdiv_(ps, ms, denom, value=-alpha)

    def _after_step(self, group):
        self.beta1_power *= group["beta1"]
        self.beta2_power *= group["beta2"]


class AdamWOptimizer(AdamOptimizer):
    kind = OPT_ADAMW

    def __init__(self, params, embedding_variables=None, lr=0.001, weight_decay=0.01, beta1=0.9, beta2=0.999, eps=1e-8, **kw):
        super().__init__(params, embedding_variables, lr, beta1, beta2, eps, weight_decay=weight_decay, **kw)

    def _dense_update(self, p, g, state, group, hp):
        if "m" not in state:
            state["m"] = torch.zeros_like(p); state["v"] = torch.zeros_like(p)
        m, v = state["m"], state["v"]
        alpha = group["lr"] * (1 - self.beta2_power) ** 0.5 / (1 - self.beta1_power)
        m.add_(g - m, alpha=1 - group["beta1"])
        v.add_(g * g - v, alpha=1 - group["beta2"])
        upd = m * alpha / (v.sqrt() + group["eps"]) + group["weight_decay"] * p
        p.sub_(upd)

    def _dense_update_many(self, ps, gs, states, group, hp):
        ms, denom, alpha = self._moments(ps, gs, states, group)
        torch._foreach_mul_(ps, 1.0 - group["weight_decay"])             # decoupled decay on the pre-update weights
        torch._foreach_addcdiv_(ps, ms, denom, value=-alpha)


class AdamAsyncOptimizer(DeepRecOptimizer):
    """adam_async.py:40 -- beta powers advance once per apply (per variable in the reference);
    ``apply_sparse_rmsprop`` switches sparse updates to the RMSProp-with-momentum form."""
    kind = OPT_ADAM_ASYNC
    slot_names = ("m", "v")

    def __init__(self, params, embedding_variables=None, lr=0.001, beta1=0.9, beta2=0.999, eps=1e-8,
                 apply_sparse_rmsprop=False, **kw):
        if apply_sparse_rmsprop:
            self.kind = OPT_ADAM_ASYNC_RMSPROP
        super().__init__(params, embedding_variables, lr, beta1=beta1, beta2=beta2, eps=eps,
                         apply_sparse_rmsprop=apply_sparse_rmsprop, **kw)

    def _dense_update(self, p, g, state, group, hp):
        if "m" not in state:
            state["m"] = torch.zeros_like(p); state["v"] = torch.zeros_like(p)
        m, v = state["m"], state["v"]
        alpha = group["lr"] * (1 - self.beta2_power) ** 0.5 / (1 - self.beta1_power)
        m.mul_(group["beta1"]).add_(g, alpha=1 - group["beta1"])
        v.mul_(group["beta2"]).addcmul_(g, g, value=1 - group["beta2"])
        p.addcdiv_(m, v.sqrt().add_(group["eps"]), value=-alpha)

    def _dense_update_many(self, ps, gs, states, group, hp):
        for p, st in zip(ps, states):
            if "m" not in st:
                st["m"] = torch.zeros_like(p); st["v"] = torch.zeros_like(p)
        ms, vs = [st["m"] for st in states], [st["v"] for st in states]
        alpha = group["lr"] * (1 - self.beta2_power) ** 0.5 / (1 - self.beta1_power)
        torch._foreach_mul_(ms, group["beta1"]); torch._foreach_add_(ms, gs, alpha=1 - group["beta1"])
        torch._foreach_mul_(vs, group["beta2"]); torch._foreach_addcmul_(vs, gs, gs, value=1 - group["beta2"])
        denom = torch._foreach_sqrt(vs)
        torch._foreach_add_(denom, group["eps"])
        torch._foreach_addcdiv_(ps, ms, denom, value=-alpha)

    def _after_step(self, group):
        self.beta1_power *= group["beta1"]
        self.beta2_power *= group["beta2"]


class FtrlOptimizer(DeepRecOptimizer):
    kind = OPT_FTRL
    slot_names = ("accum", "linear")

    def __init__(self, params, embedding_variables=None, lr=0.01, learning_rate_power=-0.5,
                 initial_accumulator_value=0.1, l1_regularization_strength=0.0, l2_regularization_strength=0.0,
                 l2_shrinkage_regularization_strength=0.0, **kw):
        self._init_acc = float(initial_accumulator_value)
        super().__init__(params, embedding_variables, lr, lr_power=learning_rate_power,
                         initial_accumulator_value=initial_accumulator_value, l1=l1_regularization_strength,
                         l2=l2_regularization_strength, l2_shrinkage=l2_shrinkage_regularization_strength, **kw)

    def _slot_init(self):
        return [self._init_acc, 0.0]

    def _dense_update(self, p, g, state, group, hp):
        # dense FTRL-proximal, ApplyFtrlV2 (training_ops.cc:370-396): element-wise l1 shrinkage; the l2-shrinkage gradient enters
        # `linear` only, the accumulator takes the raw gradient (same rule as csrc/common/ev_types.h::dr_ftrl_dense_elem)
        if "accum" not in state:
            state["accum"] = torch.full_like(p, group["initial_accumulator_value"]); state["linear"] = torch.zeros_like(p)
        acc, lin = state["accum"], state["linear"]
        lr, l1, l2, lp = group["lr"], group["l1"], group["l2"], group["lr_power"]
        gs = g + 2 * group["l2_shrinkage"] * p
        new_acc = acc + g * g
        lin.add_(gs - (new_acc.pow(-lp) - acc.pow(-lp)) / lr * p)
        quad = new_acc.pow(-lp) / lr + 2 * l2
        p.copy_(torch.where(lin.abs() > l1, (l1 * lin.sign() - lin) / quad, torch.zeros_like(p)))
        acc.add_(g * g)


# torch-style aliases
Adagrad, AdagradDecay, Adam, AdamW, AdamAsync, Ftrl, SGD = (AdagradOptimizer, AdagradDecayOptimizer, AdamOptimizer,
                                                           AdamWOptimizer, AdamAsyncOptimizer, FtrlOptimizer,
                                                           GradientDescentOptimizer)

OPTIMIZERS = {
    "adagrad": AdagradOptimizer, "adagraddecay": AdagradDecayOptimizer, "adam": AdamOptimizer,
    "adamw": AdamWOptimizer, "adamasync": AdamAsyncOptimizer, "ftrl": FtrlOptimizer,
    "gradientdescent": GradientDescentOptimizer, "sgd": GradientDescentOptimizer,
}


def make_optimizer(name: str, params, embedding_variables=None, **kw) -> DeepRecOptimizer:
    """modelzoo ``--optimizer`` switch (modelzoo/dlrm/train.py:238-270)."""
    return OPTIMIZERS[name.lower()](params, embedding_variables, **kw)
