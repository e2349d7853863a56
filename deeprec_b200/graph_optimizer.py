"""Module-graph optimizer: the reference's auto graph fusion (core/graph/optimizer_fusion_engine*.{h,cc} + template_*.h matched by
``do_op_fusion``), grappler fusions (dice_fusion.cc, concat_cast_fusing.cc) and the inference-time BatchNorm folding of
tools/low_precision_optimize -- re-thought for an eager PyTorch framework: the "graph" is the ``nn.Module`` tree, a *template* matches
a run of consecutive children of an ``nn.Sequential`` (or a single module anywhere) and replaces it by one module backed by a fused
sm_90a kernel.  Fused modules keep the ORIGINAL ``nn.Parameter`` objects, so optimizers / checkpoints created before or after the
rewrite see the same tensors.

    report = deeprec_b200.graph_optimizer.optimize(model, OptimizerOptions(do_op_fusion=True))
    enable_sample_awared_graph_compression(...)            # re-exported from serving.sample_aware

Templates (``register_template`` adds more):
  LinearReluChain      Linear [ReLU] Linear [ReLU] ...      -> nn.FusedMLP      (wgmma GEMMs, bias+ReLU epilogue, one autograd node)
  LinearBatchNormFold  Linear BatchNorm1d   (eval only)     -> Linear           (W' = diag(s) W, b' = s b + t; no normalisation pass)
  LayerNorm            nn.LayerNorm                         -> FusedLayerNorm   (one pass, fused mean/var/scale; fused_layer_norm op)
  Gelu                 nn.GELU                              -> FusedGelu
  Dice                 Dice (eval only)                     -> FusedDice        (sigmoid(BN(x)) gate in one kernel, dice_fusion.cc)
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from .nn.layers import FusedMLP
from .ops import fused_ops
from .serving.sample_aware import enable_sample_awared_graph_compression  # noqa: F401  (tf.graph_optimizer namespace parity)


@dataclass
class OptimizerOptions:
    """GraphOptions.OptimizerOptions (config.proto): ``do_op_fusion`` switches the template engine on; the rest select templates."""
    do_op_fusion: bool = True
    fuse_mlp: bool = True
    fuse_layer_norm: bool = True
    fuse_gelu: bool = True
    fuse_dice: bool = True
    fold_batchnorm: bool = True          # only applied to modules in eval mode
    min_chain: int = 1                   # Linear layers a chain needs before it is rewritten
    min_width: int = 8                   # narrower layers (e.g. the final logit) stay plain Linear: no GEMM tile to fill
    mxfp8_inference: bool = False        # eval-mode Linear(+ReLU) -> block-scaled fp8 layer (ops/mxfp8.py: e4m3 wgmma per 32-element scale block)


@dataclass
class FusionReport:
    rewrites: List[Tuple[str, str, int]] = field(default_factory=list)      # (path, template, modules replaced)

    def count(self, template: Optional[str] = None) -> int:
        return sum(1 for _, t, _ in self.rewrites if template is None or t == template)

    def __str__(self) -> str:
        return "\n".join(f"{p}: {t} ({n} modules)" for p, t, n in self.rewrites) or "(no rewrites)"


# ------------------------------------------------------------------------------------------------------------ fused modules
class FusedLayerNorm(nn.Module):
    def __init__(self, ln: nn.LayerNorm):
        super().__init__()
        if len(ln.normalized_shape) != 1 or ln.weight is None:
            raise ValueError("FusedLayerNorm needs a 1-D affine LayerNorm")
        self.weight, self.bias, self.eps = ln.weight, ln.bias, ln.eps
        if self.bias is None:
            self.bias = nn.Parameter(torch.zeros_like(ln.weight), requires_grad=False)

    def forward(self, x):
        return fused_ops.fused_layer_norm(x, self.weight, self.bias, self.eps)


class FusedGelu(nn.Module):
    def __init__(self, approximate: bool):
        super().__init__()
        self.approximate = approximate

    def forward(self, x):
        return fused_ops.gelu(x, self.approximate)


class Dice(nn.Module):
    """DIN's Dice activation: p = sigmoid(BN(x)) (BN without affine), y = p x + (1 - p) alpha x (modelzoo/din/train.py dice())."""

    def __init__(self, dim: int, eps: float = 1e-9, device=None):
        super().__init__()
        self.bn = nn.BatchNorm1d(dim, eps=eps, affine=False, device=device)
        self.alpha = nn.Parameter(torch.zeros(dim, device=device))

    def forward(self, x):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1])
        p = torch.sigmoid(self.bn(x2))
        return (p * x2 + (1 - p) * self.alpha * x2).view(shape)


class FusedDice(nn.Module):
    """Inference form of ``Dice``: running statistics + gate + blend in one kernel."""

    def __init__(self, d: Dice):
        super().__init__()
        self.alpha, self.eps = d.alpha, d.bn.eps
        self.register_buffer("mean", d.bn.running_mean.detach().clone())
        self.register_buffer("var", d.bn.running_var.detach().clone())

    def forward(self, x):
        return fused_ops.dice(x, self.alpha.detach() if not torch.is_grad_enabled() else self.alpha, self.mean, self.var, self.eps)


# ------------------------------------------------------------------------------------------------------------ template engine
class FusionTemplate:
    """One pattern.  ``match`` looks at ``mods[i:]`` (consecutive children of a Sequential; a 1-element list for a lone module) and
    returns ``(n_consumed, replacement modules)`` or ``None``."""
    name = "template"

    def enabled(self, opts: OptimizerOptions) -> bool:
        return True

    def match(self, mods: Sequence[nn.Module], i: int, opts: OptimizerOptions) -> Optional[Tuple[int, List[nn.Module]]]:
        raise NotImplementedError


class LinearReluChain(FusionTemplate):
    name = "LinearReluChain"

    def enabled(self, opts):
        return opts.fuse_mlp

    def match(self, mods, i, opts):
        j, lins, acts = i, [], []
        while j < len(mods) and type(mods[j]) is nn.Linear and mods[j].out_features >= opts.min_width \
                and (not lins or (mods[j].in_features == lins[-1].out_features and acts[-1] and (mods[j].bias is None) == (lins[0].bias is None))):
            lins.append(mods[j]); j += 1
            if j < len(mods) and type(mods[j]) is nn.ReLU:
                acts.append(True); j += 1
            else:
                acts.append(False)
        # inner layers all have ReLU (loop condition); only the last one may end without activation
        if len(lins) < max(1, opts.min_chain):
            return None
        fused = FusedMLP.__new__(FusedMLP)
        nn.Module.__init__(fused)
        fused.in_dim, fused.sizes, fused.last_act = lins[0].in_features, [l.out_features for l in lins], acts[-1]
        fused.weights = nn.ParameterList([l.weight for l in lins])                        # the SAME Parameter objects
        fused.biases = nn.ParameterList([l.bias for l in lins]) if lins[0].bias is not None else None
        return j - i, [fused]


class LinearToMXFP8(FusionTemplate):
    """Inference-only: Linear (+ReLU) in eval mode -> MXFP8Linear (weights quantised once with one power-of-two scale per 32 inputs,
    activations per call; the GEMM applies both scales per 32-element block).  The low-precision rewrite of tools/low_precision_optimize."""
    name = "LinearToMXFP8"

    def enabled(self, opts):
        return opts.mxfp8_inference

    def match(self, mods, i, opts):
        m = mods[i]
        if type(m) is not nn.Linear or m.training or m.out_features < opts.min_width or m.in_features < 32:
            return None
        from .ops.mxfp8 import MXFP8Linear
        relu = i + 1 < len(mods) and type(mods[i + 1]) is nn.ReLU
        return (2 if relu else 1), [MXFP8Linear(m, relu=relu)]


class LinearBatchNormFold(FusionTemplate):
    name = "LinearBatchNormFold"

    def enabled(self, opts):
        return opts.fold_batchnorm

    def match(self, mods, i, opts):
        if i + 1 >= len(mods) or type(mods[i]) is not nn.Linear or type(mods[i + 1]) is not nn.BatchNorm1d:
            return None
        lin, bn = mods[i], mods[i + 1]
        if bn.training or bn.running_mean is None or bn.num_features != lin.out_features:
            return None
        with torch.no_grad():
            s = torch.rsqrt(bn.running_var + bn.eps) * (bn.weight if bn.affine else 1.0)
            t = (bn.bias if bn.affine else 0.0) - bn.running_mean * s
            out = nn.Linear(lin.in_features, lin.out_features, bias=True, device=lin.weight.device, dtype=lin.weight.dtype)
            out.weight.copy_(lin.weight * s[:, None])
            out.bias.copy_((lin.bias if lin.bias is not None else 0.0) * s + t)
        out.train(lin.training)
        return 2, [out]


class _Single(FusionTemplate):
    src: type = nn.Module

    def build(self, m):
        raise NotImplementedError

    def ok(self, m) -> bool:
        return True

    def match(self, mods, i, opts):
        m = mods[i]
        if type(m) is not self.src or not self.ok(m):
            return None
        return 1, [self.build(m)]


class LayerNormTemplate(_Single):
    name, src = "LayerNorm", nn.LayerNorm

    def enabled(self, opts):
        return opts.fuse_layer_norm

    def ok(self, m):
        return len(m.normalized_shape) == 1 and m.elementwise_affine

    def build(self, m):
        return FusedLayerNorm(m)


class GeluTemplate(_Single):
    name, src = "Gelu", nn.GELU

    def enabled(self, opts):
        return opts.fuse_gelu

    def build(self, m):
        return FusedGelu(m.approximate == "tanh")


class DiceTemplate(_Single):
    name, src = "Dice", Dice

    def enabled(self, opts):
        return opts.fuse_dice

    def ok(self, m):
        return not m.training

    def build(self, m):
        return FusedDice(m)


_TEMPLATES: List[FusionTemplate] = [LinearBatchNormFold(), LinearToMXFP8(), LinearReluChain(), LayerNormTemplate(), GeluTemplate(), DiceTemplate()]


def register_template(t: FusionTemplate, first: bool = False) -> None:
    """Add a user template (matched before the built-in ones when ``first``)."""
    _TEMPLATES.insert(0, t) if first else _TEMPLATES.append(t)


def _rewrite_sequence(mods: List[nn.Module], opts: OptimizerOptions, path: str, report: FusionReport) -> List[nn.Module]:
    changed = True
    while changed:                                   # to a fixed point: BN folding exposes longer Linear/ReLU chains
        changed = False
        for t in _TEMPLATES:
            if not t.enabled(opts):
                continue
            out, i = [], 0
            while i < len(mods):
                m = t.match(mods, i, opts)
                if m is None:
                    out.append(mods[i]); i += 1
                    continue
                n, repl = m
                report.rewrites.append((f"{path}[{i}:{i + n}]", t.name, n))
                out.extend(repl); i += n
                changed = True
            mods = out
    return mods


def optimize(model: nn.Module, options: Optional[OptimizerOptions] = None) -> FusionReport:
    """Rewrite ``model`` in place; returns what was fused.  Idempotent (fused modules match no template)."""
    opts = options or OptimizerOptions()
    report = FusionReport()
    if not opts.do_op_fusion:
        return report

    def visit(mod: nn.Module, path: str):
        if isinstance(mod, nn.Sequential):
            new = _rewrite_sequence(list(mod.children()), opts, path, report)
            if len(new) != len(mod) or any(a is not b for a, b in zip(new, mod.children())):
                for k in list(mod._modules):
                    del mod._modules[k]
                for k, m in enumerate(new):
                    mod.add_module(str(k), m)
        else:
            for name, child in list(mod.named_children()):
                if isinstance(child, nn.Sequential):
                    continue
                new = _rewrite_sequence([child], opts, f"{path}.{name}" if path else name, report)
                if new[0] is not child:
                    if isinstance(mod, nn.ModuleList):
                        mod[int(name)] = new[0]
                    else:
                        setattr(mod, name, new[0])
        for name, child in mod.named_children():
            if not isinstance(child, (FusedMLP, FusedLayerNorm, FusedGelu, FusedDice)):
                visit(child, f"{path}.{name}" if path else name)

    visit(model, "")
    return report
