"""Export a trained model for the native serving runtime (``CollectiveStrategy.export_saved_model`` / SavedModel analogue).

Layout:  <dir>/saved_model.json                      architecture + version + bundle path
         <dir>/variables/variables.{data,index}      tensor bundle: dense params, BatchNorm moving statistics, per-table
                                                     keys / values / freqs / versions / default matrix
         <root>/serving_versions.json                version file polled by the ModelUpdater (full + delta versions)
Delta exports (``export_delta``) contain only rows touched since the previous export (dirty bits) + the dense block."""
from __future__ import annotations

import json
import os
from typing import Optional

import torch

from ..checkpoint.saver import BundleWriter


def _write_versions(root: str, full: Optional[dict] = None, delta: Optional[dict] = None) -> None:
    p = os.path.join(root, "serving_versions.json")
    st = {"full": None, "deltas": []}
    if os.path.exists(p):
        with open(p) as f:
            st = json.load(f)
    if full is not None:
        st["full"], st["deltas"] = full, []
    if delta is not None:
        st["deltas"].append(delta)
    tmp = p + ".tmp"
    with open(tmp, "w") as f:
        json.dump(st, f)
    os.replace(tmp, p)


def export_saved_model(engine, export_dir: str, version: Optional[int] = None, root: Optional[str] = None) -> str:
    """Full export of a :class:`DLRMEngine` (rank-local tables; rank 0 also writes the dense block)."""
    cfg = engine.cfg
    version = int(version if version is not None else engine.global_step())
    os.makedirs(os.path.join(export_dir, "variables"), exist_ok=True)
    w = BundleWriter(os.path.join(export_dir, "variables", "variables"))
    for name, (o, n) in engine.views.items():
        w.add("dense/" + name, engine.params[o:o + n])
    for L in engine.bot:
        w.add(f"bn/{L.name}/moving_mean", L.running_mean)
        w.add(f"bn/{L.name}/moving_variance", L.running_var)
    for t, tbl in engine.tables.items():
        s = tbl.snapshot()
        w.add(f"table/{t}-keys", s["keys"]); w.add(f"table/{t}-values", s["rows"][:, : engine.D].contiguous())
        w.add(f"table/{t}-freqs", s["freqs"]); w.add(f"table/{t}-versions", s["versions"])
        w.add(f"table/{t}-default", tbl.default_matrix)
        tbl.clear_dirty()
    w.close()
    meta = {"model": "dlrm", "version": version, "num_dense": cfg.num_dense, "num_tables": engine.T, "embedding_dim": engine.D,
            "mlp_bot": list(cfg.mlp_bot), "mlp_top": list(cfg.mlp_top), "bn_eps": cfg.bn_eps, "variables": "variables/variables",
            "signature": {"inputs": {"dense": ["B", cfg.num_dense], "ids": [engine.T, "B"]}, "outputs": {"probabilities": ["B"]}}}
    with open(os.path.join(export_dir, "saved_model.json"), "w") as f:
        json.dump(meta, f)
    _write_versions(root or export_dir, full={"version": version, "dir": os.path.abspath(export_dir)})
    return export_dir


def export_delta(engine, root: str, base_version: int, version: Optional[int] = None) -> str:
    """Incremental export: rows touched since the last export + the (small) dense block."""
    version = int(version if version is not None else engine.global_step())
    d = os.path.join(root, ".incr")
    os.makedirs(d, exist_ok=True)
    prefix = os.path.join(d, f"delta-{version}")
    w = BundleWriter(prefix)
    for name, (o, n) in engine.views.items():
        w.add("dense/" + name, engine.params[o:o + n])
    for L in engine.bot:
        w.add(f"bn/{L.name}/moving_mean", L.running_mean)
        w.add(f"bn/{L.name}/moving_variance", L.running_var)
    for t, tbl in engine.tables.items():
        s = tbl.snapshot(dirty_only=True)
        w.add(f"table/{t}-sparse_incr_keys", s["keys"]); w.add(f"table/{t}-sparse_incr_values", s["rows"][:, : engine.D].contiguous())
        tbl.clear_dirty()
    w.close()
    _write_versions(root, delta={"version": version, "base": int(base_version), "prefix": os.path.abspath(prefix)})
    return prefix


# ---------------------------------------------------------------------------------------------------------------------------------
# the same saved-model format from the framework-API DLRM module (deeprec_b200.models.dlrm.DLRM) -- CPU training -> CPU / GPU serving
# ---------------------------------------------------------------------------------------------------------------------------------
def _pad_k(w: torch.Tensor) -> torch.Tensor:
    """Linear weight [N, K] -> [N, pad8(K)] (the runtimes read kernels with the K dimension padded to a multiple of 8)."""
    n, k = w.shape
    kp = (k + 7) // 8 * 8
    out = torch.zeros(n, kp, dtype=torch.float32)
    out[:, :k] = w.detach().float().cpu()
    return out.contiguous()


def _module_dense_tensors(model) -> dict:
    import torch.nn as nn
    out = {}
    bot = [m for m in model.bot if isinstance(m, (nn.Linear, nn.BatchNorm1d))]
    for l in range(len(bot) // 2):
        lin, bn = bot[2 * l], bot[2 * l + 1]
        nm = f"mlp_bot_{l}"
        out[f"dense/{nm}/kernel"], out[f"dense/{nm}/bias"] = _pad_k(lin.weight), lin.bias.detach().float().cpu().contiguous()
        out[f"dense/{nm}/bn_gamma"], out[f"dense/{nm}/bn_beta"] = bn.weight.detach().float().cpu().contiguous(), bn.bias.detach().float().cpu().contiguous()
        out[f"bn/{nm}/moving_mean"], out[f"bn/{nm}/moving_variance"] = bn.running_mean.detach().float().cpu().contiguous(), bn.running_var.detach().float().cpu().contiguous()
    for l, lin in enumerate(m for m in model.top if isinstance(m, nn.Linear)):
        out[f"dense/mlp_top_{l}/kernel"], out[f"dense/mlp_top_{l}/bias"] = _pad_k(lin.weight), lin.bias.detach().float().cpu().contiguous()
    out["dense/logits/kernel"] = model.logits.weight.detach().float().cpu().reshape(-1).contiguous()
    out["dense/logits/bias"] = model.logits.bias.detach().float().cpu().reshape(-1).contiguous()
    return out


def export_saved_model_module(model, export_dir: str, version: int, root: Optional[str] = None) -> str:
    """Full export of a ``models.dlrm.DLRM`` module (dot interaction, EmbeddingVariable tables) in the format both serving runtimes load."""
    import torch.nn as nn
    if getattr(model, "interaction_op", "dot") != "dot":
        raise ValueError("the serving runtimes implement the dot interaction")
    evs = model.embedding_variables()
    lin_bot = [m for m in model.bot if isinstance(m, nn.Linear)]
    lin_top = [m for m in model.top if isinstance(m, nn.Linear)]
    bns = [m for m in model.bot if isinstance(m, nn.BatchNorm1d)]
    os.makedirs(os.path.join(export_dir, "variables"), exist_ok=True)
    w = BundleWriter(os.path.join(export_dir, "variables", "variables"))
    for name, t in _module_dense_tensors(model).items():
        w.add(name, t)
    D = evs[0].embedding_dim
    for t, ev in enumerate(evs):
        s = ev.table.snapshot()
        w.add(f"table/{t}-keys", s["keys"].cpu()); w.add(f"table/{t}-values", s["rows"][:, :D].contiguous().cpu())
        w.add(f"table/{t}-freqs", s["freqs"].cpu()); w.add(f"table/{t}-versions", s["versions"].cpu())
        w.add(f"table/{t}-default", ev.default_matrix.detach().float().cpu().contiguous())
        ev.table.clear_dirty()
    w.close()
    meta = {"model": "dlrm", "version": int(version), "num_dense": lin_bot[0].in_features, "num_tables": len(evs), "embedding_dim": D,
            "mlp_bot": [m.out_features for m in lin_bot], "mlp_top": [m.out_features for m in lin_top], "bn_eps": float(bns[0].eps),
            "variables": "variables/variables",
            "signature": {"inputs": {"dense": ["B", lin_bot[0].in_features], "ids": [len(evs), "B"]}, "outputs": {"probabilities": ["B"]}}}
    with open(os.path.join(export_dir, "saved_model.json"), "w") as f:
        json.dump(meta, f)
    _write_versions(root or export_dir, full={"version": int(version), "dir": os.path.abspath(export_dir)})
    return export_dir


def export_delta_module(model, root: str, base_version: int, version: int) -> str:
    """Incremental export of a ``models.dlrm.DLRM`` module: rows touched since the last export + the dense block."""
    d = os.path.join(root, ".incr")
    os.makedirs(d, exist_ok=True)
    prefix = os.path.join(d, f"delta-{int(version)}")
    w = BundleWriter(prefix)
    for name, t in _module_dense_tensors(model).items():
        w.add(name, t)
    for t, ev in enumerate(model.embedding_variables()):
        s = ev.table.snapshot(dirty_only=True)
        w.add(f"table/{t}-sparse_incr_keys", s["keys"].cpu()); w.add(f"table/{t}-sparse_incr_values", s["rows"][:, : ev.embedding_dim].contiguous().cpu())
        ev.table.clear_dirty()
    w.close()
    _write_versions(root, delta={"version": int(version), "base": int(base_version), "prefix": os.path.abspath(prefix)})
    return prefix


# ---------------------------------------------------------------------------------------------------------------------------------
# any zoo model -> a servable directory (the reference's SavedModel works for every model; the native Processors are DLRM-shaped, every
# other model is served by the python SessionGroup / HTTP front-end from this format)
# ---------------------------------------------------------------------------------------------------------------------------------
def export_zoo_model(model, name: str, export_dir: str, version: int, build_kwargs: Optional[dict] = None) -> str:
    """Write ``saved_model.json`` (zoo name + constructor arguments + version) and a full checkpoint (dense parameters, BatchNorm statistics,
    every EmbeddingVariable with its metadata) of ``model`` -- a model built by ``models.zoo.build_model(name, **build_kwargs)``."""
    from ..checkpoint.saver import Saver
    os.makedirs(os.path.join(export_dir, "variables"), exist_ok=True)
    prefix = Saver(model).save(os.path.join(export_dir, "variables", "variables"), global_step=int(version))
    meta = {"model": name, "zoo": True, "version": int(version), "build_kwargs": dict(build_kwargs or {}), "variables": os.path.relpath(prefix, export_dir)}
    tmp = os.path.join(export_dir, "saved_model.json.tmp")
    with open(tmp, "w") as f:
        json.dump(meta, f)
    os.replace(tmp, os.path.join(export_dir, "saved_model.json"))          # the directory becomes visible as a model only when complete
    return export_dir


def load_zoo_model(export_dir: str, device: str = "cpu"):
    """Rebuild the model of ``export_zoo_model`` for serving: EmbeddingVariables are created in inference mode (lookups never create
    keys, filters are ignored -- ``INFERENCE_MODE``), state restored, ``eval()`` set.  Returns ``(model, version)``."""
    from ..checkpoint.saver import Saver
    from ..models.zoo import build_model
    with open(os.path.join(export_dir, "saved_model.json")) as f:
        meta = json.load(f)
    if not meta.get("zoo"):
        raise ValueError(f"{export_dir} is an engine / DLRM-module export: load it with serving.Processor")
    prev = os.environ.get("INFERENCE_MODE")
    os.environ["INFERENCE_MODE"] = "1"
    try:
        model = build_model(meta["model"], device=device, **meta.get("build_kwargs", {}))
        Saver(model).restore(os.path.join(export_dir, meta["variables"]))
    finally:
        if prev is None:
            os.environ.pop("INFERENCE_MODE", None)
        else:
            os.environ["INFERENCE_MODE"] = prev
    return model.eval(), int(meta["version"])


# ------------------------------------------------------------------------------------------------------------------------------------
# Op-program export: Criteo-style zoo models other than DLRM for the native CPU Processor (csrc/host/cpu_serving.cc::Program).
# The reference's processor executes whatever graph the SavedModel holds; here the inference graph of a model is written as a short
# list of ops over named [B, width] buffers -- inputs "dense" [B, num_dense] and "emb" [B, T * D] -- with BatchNorm folded into the
# following Linear at export time (moving statistics), so the runtime only needs concat / linear / affine / fm / cross / mul_add / add / mul / layernorm.
# ------------------------------------------------------------------------------------------------------------------------------------
class _ProgramBuilder:
    def __init__(self):
        self.ops, self.tensors, self._n = [], {}, 0

    def _name(self, base):
        self._n += 1
        return f"{base}{self._n}"

    def concat(self, srcs):
        out = self._name("cat"); self.ops.append({"op": "concat", "out": out, "in": list(srcs)}); return out

    def linear(self, src, weight, bias, relu=False):
        out = self._name("lin")
        self.tensors[f"prog/{out}/kernel"] = weight.detach().float().cpu().contiguous()                 # [N, K]
        self.tensors[f"prog/{out}/bias"] = (bias.detach().float().cpu() if bias is not None else torch.zeros(weight.shape[0])).contiguous()
        self.ops.append({"op": "linear", "out": out, "in": [src], "relu": bool(relu)}); return out

    def affine(self, src, scale, shift):
        out = self._name("aff")
        self.tensors[f"prog/{out}/scale"] = scale.detach().float().cpu().contiguous(); self.tensors[f"prog/{out}/shift"] = shift.detach().float().cpu().contiguous()
        self.ops.append({"op": "affine", "out": out, "in": [src]}); return out

    def fm(self, emb):
        out = self._name("fm"); self.ops.append({"op": "fm", "out": out, "in": [emb]}); return out

    def cross(self, x0, x, w, b):
        out = self._name("cross")
        self.tensors[f"prog/{out}/w"] = w.detach().float().cpu().contiguous(); self.tensors[f"prog/{out}/b"] = b.detach().float().cpu().contiguous()
        self.ops.append({"op": "cross", "out": out, "in": [x0, x]}); return out

    def mul_add(self, a, b, c):
        out = self._name("fma"); self.ops.append({"op": "mul_add", "out": out, "in": [a, b, c]}); return out

    def add(self, a, b):
        out = self._name("add"); self.ops.append({"op": "add", "out": out, "in": [a, b]}); return out

    def slice(self, src, start, length):
        out = self._name("slice"); self.ops.append({"op": "slice", "out": out, "in": [src], "start": int(start), "len": int(length)}); return out

    def mul(self, a, b):
        out = self._name("mul"); self.ops.append({"op": "mul", "out": out, "in": [a, b]}); return out

    def layernorm(self, src, ln, relu=False):
        out = self._name("ln")
        self.tensors[f"prog/{out}/scale"] = ln.weight.detach().float().cpu().contiguous(); self.tensors[f"prog/{out}/shift"] = ln.bias.detach().float().cpu().contiguous()
        self.ops.append({"op": "layernorm", "out": out, "in": [src], "eps": float(ln.eps), "relu": bool(relu)}); return out

    # ---- sequence models (DIN): the id rows of a request are COLUMNS over shared tables (meta "col_table") --------------------------------
    def valid_mask(self, start, length):
        """[B, length]: 1.0 where the id of lookup column ``start + l`` is >= 0 (padding of a history is -1)."""
        out = self._name("valid"); self.ops.append({"op": "valid_mask", "out": out, "in": ["emb"], "start": int(start), "len": int(length)}); return out

    def seq_zip(self, a, b, L):
        out = self._name("zip"); self.ops.append({"op": "seq_zip", "out": out, "in": [a, b], "len": int(L)}); return out

    def seq_mask(self, x, mask, L):
        out = self._name("smask"); self.ops.append({"op": "seq_mask", "out": out, "in": [x, mask], "len": int(L)}); return out

    def seq_sum(self, x, L):
        out = self._name("ssum"); self.ops.append({"op": "seq_sum", "out": out, "in": [x], "len": int(L)}); return out

    def prelu(self, src, alpha, width):
        out = self._name("prelu")
        a = alpha.detach().float().cpu().reshape(-1)
        self.tensors[f"prog/{out}/alpha"] = (a.expand(width) if a.numel() == 1 else a).contiguous()
        self.ops.append({"op": "prelu", "out": out, "in": [src]}); return out

    # ---- recurrent / transformer sequence models (DIEN, BST) -------------------------------------------------------------------------------
    def gru(self, x, L, gru):
        """Single-layer batch-first ``nn.GRU`` over ``x [B, L * I]`` -> every hidden state ``[B, L * H]`` (h0 = 0, PyTorch gate order r, z, n)."""
        if gru.num_layers != 1 or gru.bidirectional or not gru.batch_first:
            raise TypeError("op-program export: single-layer, unidirectional, batch_first GRU only")
        out = self._name("gru")
        for nm, t in (("w_ih", gru.weight_ih_l0), ("w_hh", gru.weight_hh_l0), ("b_ih", gru.bias_ih_l0), ("b_hh", gru.bias_hh_l0)):
            self.tensors[f"prog/{out}/{nm}"] = t.detach().float().cpu().contiguous()
        self.ops.append({"op": "gru", "out": out, "in": [x], "len": int(L)}); return out

    def seq_last(self, x, mask, L):
        """``x [B, L * W]`` at the last valid position of every row (``max(sum(mask), 1) - 1``) -> ``[B, W]``."""
        out = self._name("last"); self.ops.append({"op": "seq_last", "out": out, "in": [x, mask], "len": int(L)}); return out

    def seq_linear(self, src, weight, bias, L, relu=False):
        """The same Linear at every one of the L positions of ``src [B, L * K]`` -> ``[B, L * N]`` (one GEMM over B * L rows)."""
        out = self._name("slin")
        self.tensors[f"prog/{out}/kernel"] = weight.detach().float().cpu().contiguous()
        self.tensors[f"prog/{out}/bias"] = (bias.detach().float().cpu() if bias is not None else torch.zeros(weight.shape[0])).contiguous()
        self.ops.append({"op": "linear", "out": out, "in": [src], "relu": bool(relu), "len": int(L)}); return out

    def seq_layernorm(self, src, ln, L):
        out = self._name("sln")
        self.tensors[f"prog/{out}/scale"] = ln.weight.detach().float().cpu().contiguous(); self.tensors[f"prog/{out}/shift"] = ln.bias.detach().float().cpu().contiguous()
        self.ops.append({"op": "layernorm", "out": out, "in": [src], "eps": float(ln.eps), "relu": False, "len": int(L)}); return out

    def mha(self, qkv, valid, S, heads):
        """Multi-head self-attention core over ``qkv [B, S * 3E]`` (per position ``[q | k | v]``), keys with ``valid [B, S] == 0`` masked -> ``[B, S * E]``."""
        out = self._name("mha"); self.ops.append({"op": "mha", "out": out, "in": [qkv, valid], "len": int(S), "heads": int(heads)}); return out

    def seq_mean(self, x, valid, S):
        """Mean of ``x [B, S * W]`` over the valid positions -> ``[B, W]``."""
        out = self._name("smean"); self.ops.append({"op": "seq_mean", "out": out, "in": [x, valid], "len": int(S)}); return out

    def din_attention(self, q, k, mask, att, weights=False):
        """Linear(4W, H1)-Sigmoid-Linear(H1, H2)-Sigmoid-Linear(H2, 1) attention unit, masked softmax, weighted sum of the keys
        (``weights=True``: the softmax weights ``[B, L]`` themselves -- DIEN scales its hidden states with them)."""
        import torch.nn as nn
        mods = list(att)
        if not (len(mods) == 5 and all(isinstance(mods[i], nn.Linear) for i in (0, 2, 4)) and all(isinstance(mods[i], nn.Sigmoid) for i in (1, 3)) and mods[4].out_features == 1):
            raise TypeError("op-program export: din_attention needs the Linear-Sigmoid-Linear-Sigmoid-Linear(1) unit")
        out = self._name("att")
        for nm, t in (("w1", mods[0].weight), ("b1", mods[0].bias), ("w2", mods[2].weight), ("b2", mods[2].bias), ("w3", mods[4].weight), ("b3", mods[4].bias)):
            self.tensors[f"prog/{out}/{nm}"] = t.detach().float().cpu().reshape(-1).contiguous()
        self.ops.append({"op": "din_attention", "out": out, "in": [q, k, mask], "mode": 1 if weights else 0}); return out

    def tile(self, src):
        """Broadcast row 0 of a buffer computed once per request (``rows1`` ops, sample-aware compression) to every row of the batch."""
        out = self._name("tile"); self.ops.append({"op": "tile", "out": out, "in": [src]}); return out

    def softmax(self, src):
        out = self._name("softmax"); self.ops.append({"op": "softmax", "out": out, "in": [src]}); return out

    def cosine(self, a, b):
        out = self._name("cos"); self.ops.append({"op": "cosine", "out": out, "in": [a, b]}); return out

    def mixture(self, gate, experts, width):
        """sum_e gate[:, e] * expert_e: the experts concatenated [B, E * width], weighted position-wise, summed over E."""
        n = len(experts)
        return self.seq_sum(self.seq_mask(self.concat(experts), gate, n), n)

    def sequential(self, src, seq):
        """nn.Sequential of Linear / ReLU / BatchNorm1d (what ``models.zoo.mlp`` builds on CPU): a BatchNorm folds into the next Linear
        (W' = W diag(s), b' = b + W t); one left over at the end becomes an explicit affine op."""
        import torch.nn as nn
        pending = None

        def flat(m):
            if isinstance(m, nn.Sequential):
                for c in m:
                    yield from flat(c)
            else:
                yield m
        mods = list(flat(seq))
        i = 0
        while i < len(mods):
            m = mods[i]
            if isinstance(m, nn.Linear):
                W, b = m.weight.detach().float(), (m.bias.detach().float() if m.bias is not None else torch.zeros(m.out_features))
                if pending is not None:
                    s, t = pending
                    b = b + W @ t; W = W * s.unsqueeze(0); pending = None
                relu = i + 1 < len(mods) and isinstance(mods[i + 1], nn.ReLU)
                src = self.linear(src, W, b, relu)
                i += 2 if relu else 1
                if i < len(mods) and isinstance(mods[i], nn.PReLU):
                    src = self.prelu(src, mods[i].weight, m.out_features)
                    i += 1
            elif isinstance(m, nn.BatchNorm1d):
                s = m.weight.detach().float() / torch.sqrt(m.running_var.detach().float() + m.eps)
                pending = (s, m.bias.detach().float() - m.running_mean.detach().float() * s)
                i += 1
            elif isinstance(m, nn.LayerNorm):
                if pending is not None:
                    src = self.affine(src, *pending); pending = None
                relu = i + 1 < len(mods) and isinstance(mods[i + 1], nn.ReLU)
                src = self.layernorm(src, m, relu)
                i += 2 if relu else 1
            else:
                raise TypeError(f"op-program export: unsupported layer {type(m).__name__} (Linear / ReLU / PReLU / BatchNorm1d / LayerNorm chains only)")
        if pending is not None:
            src = self.affine(src, *pending)
        return src


def _build_program(model, max_len: int = 50) -> _ProgramBuilder:
    from ..models import zoo
    p = _ProgramBuilder()
    if isinstance(model, zoo.DeepFM):
        x0 = p.concat(["dense", "emb"])
        dnn = p.sequential(x0, model.dnn)
        lin = p.linear("dense", model.linear.weight, model.linear.bias)
        h = p.sequential(p.concat([lin, p.fm("emb"), dnn]), model.final)
        p.out = p.linear(h, model.out.weight, model.out.bias)
    elif isinstance(model, zoo.WDL):
        # tables 0..T-1 = deep (dim D), T..2T-1 = wide (dim 4, stored zero-padded to D); both read the same request id row
        T, D = model.num_sparse, model.emb_dim
        deep = p.linear(p.sequential(p.concat(["dense", p.slice("emb", 0, T * D)]), model.deep), model.out.weight, model.out.bias)
        sel = torch.zeros(1, T * D); sel[0, ::D] = 1.0                     # sum over tables of component 0 of the wide embedding
        wide = p.add(p.linear(p.slice("emb", T * D, T * D), sel, None), p.linear("dense", model.wide_dense.weight, model.wide_dense.bias))
        p.out = p.add(wide, deep)
        p.tables = [(ev, ev.embedding_dim) for ev in _evs_of(model.emb)] + [(ev, ev.embedding_dim) for ev in _evs_of(model.wide)]
        p.id_map = list(range(T)) + list(range(T))
    elif isinstance(model, zoo.MaskNet):                                 # serial MaskBlocks: h = ReLU(LN(W (h * mask(v))))
        h = p.layernorm("emb", model.ln_emb)
        for m, b in zip(model.masks, model.blocks):
            h = p.sequential(p.mul(h, p.sequential("emb", m)), b)
        p.out = p.sequential(p.concat([h, "dense"]), model.out)
    elif isinstance(model, zoo.DCNv2):                                   # x_{l+1} = x0 * (W x_l + b) + x_l (full-rank or low-rank W)
        x0 = p.concat(["dense", "emb"])
        x = x0
        for W in model.W:
            x = p.mul_add(x0, p.sequential(x, W), x)
        p.out = p.linear(p.concat([x, p.sequential(x0, model.deep)]), model.out.weight, model.out.bias)
    elif isinstance(model, zoo.DCN):
        x0 = p.concat(["dense", "emb"])
        x = x0
        for w, b in zip(model.cw, model.cb):
            x = p.cross(x0, x, w, b)
        p.out = p.linear(p.concat([x, p.sequential(x0, model.deep)]), model.out.weight, model.out.bias)
    elif isinstance(model, (zoo._MultiTask, zoo.DSSM)):
        # Taobao-shaped models on the pooled behaviour history: lookup columns as for DIN, features = [user | target | sum of the valid history]
        L, D = int(max_len), model.emb_dim
        p.tables = [(model.user, D), (model.item, D), (model.cat, D)]
        p.col_table = [0, 1, 2] + [1] * L + [2] * L
        p.num_dense = 1
        u, q = p.slice("emb", 0, D), p.slice("emb", D, 2 * D)
        mask = p.valid_mask(3, L)
        pooled = p.seq_sum(p.seq_mask(p.seq_zip(p.slice("emb", 3 * D, L * D), p.slice("emb", (3 + L) * D, L * D), L), mask, L), L)      # [B, 2D]
        if isinstance(model, zoo.DSSM):
            ue, ie = p.sequential(p.concat([u, pooled]), model.user_tower), p.sequential(q, model.item_tower)
            p.out = p.affine(p.cosine(ue, ie), model.scale.detach().reshape(1), torch.zeros(1))
        else:
            f = p.concat([u, q, pooled])
            tasks = list(model.tasks)
            if isinstance(model, zoo.ESMM):
                outs = [p.sequential(f, model.ctr), p.sequential(f, model.cvr)]
            elif isinstance(model, zoo.SimpleMultiTask):
                outs = [p.sequential(f, model.towers[t]) for t in tasks]
            elif isinstance(model, zoo.MMoE):
                ex = [p.sequential(f, e) for e in model.experts]
                w = model.experts[0][-2].out_features if isinstance(model.experts[0][-1], torch.nn.ReLU) else model.experts[0][-1].out_features
                outs = [p.sequential(p.mixture(p.softmax(p.linear(f, model.gates[t].weight, model.gates[t].bias)), ex, w), model.towers[t]) for t in tasks]
            elif isinstance(model, zoo.DBMTL):
                sh = p.sequential(f, model.bottom)
                a_, c_ = p.sequential(sh, model.t_ctr), p.sequential(sh, model.t_cvr)
                outs = [p.linear(a_, model.o_ctr.weight, model.o_ctr.bias), p.linear(p.sequential(p.concat([a_, c_]), model.rel), model.o_cvr.weight, model.o_cvr.bias)]
            elif isinstance(model, zoo.PLE):
                xs = {t: f for t in tasks}
                xs["shared"] = f
                for Lyr in model.layers:
                    sh = [p.sequential(xs["shared"], e) for e in Lyr["shared"]]
                    sp = {t: [p.sequential(xs[t], e) for e in Lyr[f"spec_{t}"]] for t in tasks}
                    nxt = {t: p.mixture(p.softmax(p.linear(xs[t], Lyr[f"gate_{t}"].weight, Lyr[f"gate_{t}"].bias)), sp[t] + sh, 0) for t in tasks}
                    allx = [x for t in tasks for x in sp[t]] + sh
                    nxt["shared"] = p.mixture(p.softmax(p.linear(xs["shared"], Lyr["gate_shared"].weight, Lyr["gate_shared"].bias)), allx, 0)
                    xs = nxt
                outs = [p.sequential(xs[t], model.towers[t]) for t in tasks]
            else:
                raise TypeError(f"op-program export: no builder for {type(model).__name__}")
            p.out = p.concat(outs)
            p.num_outputs, p.output_names = len(outs), tasks
    elif isinstance(model, zoo.DIN):
        # lookup columns [user | item | cat | hist_item x L | hist_cat x L] over the three tables (the layout of models.rec_engine.din_ids);
        # padding ids (-1) give masked (zeroed) history positions
        import torch.nn as nn
        L, D = int(max_len), model.emb_dim
        p.tables = [(model.user, D), (model.item, D), (model.cat, D)]
        p.col_table = [0, 1, 2] + [1] * L + [2] * L
        p.num_dense = 1                                                   # a dummy dense column keeps the request format uniform
        u, q = p.slice("emb", 0, D), p.slice("emb", D, 2 * D)
        mask = p.valid_mask(3, L)
        k = p.seq_mask(p.seq_zip(p.slice("emb", 3 * D, L * D), p.slice("emb", (3 + L) * D, L * D), L), mask, L)      # [B, L * 2D]
        x = p.concat([u, q, p.seq_sum(k, L), p.din_attention(q, k, mask, model.att)])
        p.out = p.sequential(x, nn.Sequential(model.bn, *list(model.top)))
    elif isinstance(model, (zoo.DIEN, zoo.BST)):
        L, D = int(max_len), model.emb_dim
        E = 2 * D
        p.tables = [(model.user, D), (model.item, D), (model.cat, D)]
        p.col_table = [0, 1, 2] + [1] * L + [2] * L
        p.num_dense = 1
        u, q = p.slice("emb", 0, D), p.slice("emb", D, 2 * D)
        mask = p.valid_mask(3, L)
        k = p.seq_mask(p.seq_zip(p.slice("emb", 3 * D, L * D), p.slice("emb", (3 + L) * D, L * D), L), mask, L)      # [B, L * E], padding zeroed
        if isinstance(model, zoo.DIEN):
            # interest extractor GRU -> attention weights of the target against every hidden state -> evolution GRU over the weighted states
            h1 = p.gru(k, L, model.gru1)
            qh = p.linear(q, model.qproj.weight, model.qproj.bias)
            w = p.din_attention(qh, h1, mask, model.att, weights=True)
            h2 = p.gru(p.seq_mask(h1, w, L), L, model.gru2)
            x = p.concat([u, q, p.seq_last(h2, mask, L), p.seq_sum(k, L)])
            p.out = p.sequential(x, model.top)
        else:
            # one post-norm encoder block over [history ; target] with key-padding mask, masked mean pooling
            enc = model.enc
            if enc.norm_first or enc.self_attn.batch_first is not True or not getattr(enc, "activation_relu_or_gelu", 1) == 1:
                raise TypeError("op-program export: BST needs the post-norm, batch_first, ReLU TransformerEncoderLayer")
            S = L + 1
            if S > model.pos.shape[0]:
                raise ValueError(f"op-program export: max_len {L} exceeds the model's positional table ({model.pos.shape[0] - 1})")
            x = p.affine(p.concat([k, q]), torch.ones(S * E), model.pos[:S].detach().reshape(-1))
            valid = p.concat([mask, p.affine(p.slice("dense", 0, 1), torch.zeros(1), torch.ones(1))])              # the target position is always valid
            at = enc.self_attn
            a_ = p.seq_linear(p.mha(p.seq_linear(x, at.in_proj_weight, at.in_proj_bias, S), valid, S, at.num_heads), at.out_proj.weight, at.out_proj.bias, S)
            x1 = p.seq_layernorm(p.add(x, a_), enc.norm1, S)
            f_ = p.seq_linear(p.seq_linear(x1, enc.linear1.weight, enc.linear1.bias, S, relu=True), enc.linear2.weight, enc.linear2.bias, S)
            x2 = p.seq_layernorm(p.add(x1, f_), enc.norm2, S)
            p.out = p.linear(p.sequential(p.concat([u, q, p.seq_mean(x2, valid, S)]), model.final), model.out.weight, model.out.bias)
    else:
        raise TypeError(f"op-program export: no builder for {type(model).__name__} (WDL, DeepFM, DCN, DCNv2, MaskNet, DIN, DIEN, BST, DSSM, ESMM, MMoE, DBMTL, PLE, SimpleMultiTask; DLRM has export_saved_model_module)")
    return p


# ---- sample-aware graph compression as a pass over the op program ---------------------------------------------------------------------------
_ROW_WISE = {"concat", "linear", "affine", "cross", "mul_add", "add", "mul", "layernorm", "slice", "seq_zip", "seq_mask", "seq_sum", "prelu", "softmax",
             "cosine", "din_attention", "valid_mask", "gru", "seq_last", "mha", "seq_mean"}


def compress_sample_aware(ops: list, output: str, user_columns, emb_dim: int, user_dense: bool = False):
    """Sample-aware graph compression (reference: ``python/graph_optimizer/sample_awared_graph_compression.py:26`` -- a ranking request scores N
    candidate items for ONE user, so everything that depends on user-side features only is computed once and tiled to N as late as possible).

    ``user_columns``: lookup columns (indices into the request's id rows) that carry user-side features -- identical for every row of a request;
    ``user_dense``: the dense block is user-side too.  The pass marks every op whose inputs are all user-side ``rows1`` (both native interpreters run
    it at batch 1, reading row 0 of its inputs) and inserts a ``tile`` op where a per-candidate op consumes such a buffer.  Returns
    ``(ops, output, n_compressed)``; requests stay ``[rows, B]`` -- only row 0 of the user columns is read by the compressed part (clients may
    pad the rest with -1)."""
    user_cols = set(int(c) for c in user_columns)
    D = int(emb_dim)
    user_only = {"dense": bool(user_dense), "emb": False}
    tiled, new_ops, n = {}, [], 0

    def emb_range_user(start, length):
        if start % D or length % D:
            return False
        return all(c in user_cols for c in range(start // D, (start + length) // D))

    for op in ops:
        op = dict(op)
        kind, ins = op["op"], list(op["in"])
        if kind == "slice" and ins[0] == "emb":
            u = emb_range_user(op["start"], op["len"])
        elif kind == "valid_mask":
            u = all(c in user_cols for c in range(op["start"], op["start"] + op["len"]))
        elif kind in _ROW_WISE:
            u = all(user_only.get(i, False) for i in ins)
        else:                                       # fm reads the whole embedding block; unknown ops stay per-candidate
            u = False
        if u:
            op["rows1"] = 1
            n += 1
        else:                                       # a per-candidate op: user-side inputs are tiled first (once per buffer)
            for k, i in enumerate(ins):
                if user_only.get(i, False):
                    if i not in tiled:
                        tiled[i] = f"{i}_tile"
                        new_ops.append({"op": "tile", "out": tiled[i], "in": [i]})
                        user_only[tiled[i]] = False
                    ins[k] = tiled[i]
            op["in"] = ins
        user_only[op["out"]] = u
        new_ops.append(op)
    if user_only.get(output, False):                # degenerate: the whole model is user-side
        new_ops.append({"op": "tile", "out": f"{output}_tile", "in": [output]})
        output = f"{output}_tile"
    return new_ops, output, n


def taobao_user_columns(max_len: int):
    """User-side lookup columns of the Taobao-shaped programs (``[user | item | cat | hist_item x L | hist_cat x L]``): the user id and the whole
    behaviour history; the target item / category are per candidate."""
    L = int(max_len)
    return [0] + list(range(3, 3 + 2 * L))


def _evs_of(module):
    from ..optim.optimizers import collect_embedding_variables
    return collect_embedding_variables(module)


def _program_tables(model, p):
    """[(EmbeddingVariable, its dim)] in table order, the common row width D (narrower tables are stored zero-padded), id_map or None."""
    tables = getattr(p, "tables", None) or [(ev, ev.embedding_dim) for ev in _evs_of(model.emb)]
    return tables, max(d for _, d in tables), getattr(p, "id_map", None)


def _padded(rows: torch.Tensor, d: int, D: int) -> torch.Tensor:
    rows = rows[:, :d].float().cpu()
    if d == D:
        return rows.contiguous()
    out = torch.zeros(rows.shape[0], D); out[:, :d] = rows
    return out


def export_saved_model_program(model, export_dir: str, version: int, root: Optional[str] = None, max_len: int = 50,
                               sample_aware: Optional[dict] = None) -> str:
    """Full export of a zoo model (Criteo-style ``WDL``, ``DeepFM``, ``DCN``, ``DCNv2``, ``MaskNet``; sequence model ``DIN`` with ``max_len`` history
    positions -- request ids = the ``[3 + 2 L, B]`` block of ``models.rec_engine.din_ids`` and one dummy dense column) as an op program + EmbeddingVariable tables; loaded by
    ``Processor(dir, cfg)`` (GPU runtime: wgmma GEMMs + csrc/cuda/program_kernels.cu; ``device="cpu"``: the host interpreter) exactly like a DLRM
    export (same ModelConfig, update protocol, request formats)."""
    was_training = model.training
    model.eval()
    p = _build_program(model, max_len)
    tables, D, id_map = _program_tables(model, p)
    col_table = getattr(p, "col_table", None)
    num_dense = getattr(p, "num_dense", None) or model.num_dense
    n_compressed = 0
    if sample_aware:                               # {"user_columns": [...], "user_dense": bool}: user-side sub-graph once per request
        p.ops, p.out, n_compressed = compress_sample_aware(p.ops, p.out, sample_aware["user_columns"], D, bool(sample_aware.get("user_dense", False)))
    os.makedirs(os.path.join(export_dir, "variables"), exist_ok=True)
    w = BundleWriter(os.path.join(export_dir, "variables", "variables"))
    for name, t in p.tensors.items():
        w.add(name, t)
    for t, (ev, d) in enumerate(tables):
        s = ev.table.snapshot()
        w.add(f"table/{t}-keys", s["keys"].cpu()); w.add(f"table/{t}-values", _padded(s["rows"], d, D))
        w.add(f"table/{t}-freqs", s["freqs"].cpu()); w.add(f"table/{t}-versions", s["versions"].cpu())
        w.add(f"table/{t}-default", _padded(ev.default_matrix.detach(), d, D))
        ev.table.clear_dirty()
    w.close()
    rows = (len(col_table) if col_table is not None else len(tables)) if id_map is None else max(id_map) + 1
    meta = {"model": type(model).__name__.lower(), "arch": "program", "version": int(version), "num_dense": num_dense, "num_tables": len(tables),
            "num_id_rows": rows, "embedding_dim": D, "program": p.ops, "output": p.out, "variables": "variables/variables",
            "signature": {"inputs": {"dense": ["B", num_dense], "ids": [rows, "B"]}, "outputs": {"probabilities": ["B"]}}}
    if id_map is not None:
        meta["id_map"] = id_map
    if col_table is not None:
        meta["col_table"] = col_table
    if sample_aware:
        meta["sample_aware"] = {"user_columns": [int(c) for c in sample_aware["user_columns"]], "user_dense": bool(sample_aware.get("user_dense", False)),
                                "ops_at_batch_1": int(n_compressed)}
    if getattr(p, "num_outputs", 1) > 1:                                 # multi-task: probabilities [B, num_outputs], one column per task
        meta["num_outputs"], meta["output_names"] = p.num_outputs, list(p.output_names)
        meta["signature"]["outputs"] = {"probabilities": ["B", p.num_outputs]}
    with open(os.path.join(export_dir, "saved_model.json"), "w") as f:
        json.dump(meta, f)
    _write_versions(root or export_dir, full={"version": int(version), "dir": os.path.abspath(export_dir)})
    model.train(was_training)
    return export_dir


def export_delta_program(model, root: str, base_version: int, version: int, max_len: int = 50) -> str:
    """Incremental export for an op-program model: rows touched since the last export + the (re-folded) dense tensors."""
    was_training = model.training
    model.eval()
    p = _build_program(model, max_len)
    d = os.path.join(root, ".incr")
    os.makedirs(d, exist_ok=True)
    prefix = os.path.join(d, f"delta-{int(version)}")
    w = BundleWriter(prefix)
    for name, t in p.tensors.items():
        w.add(name, t)
    tables, D, _ = _program_tables(model, p)
    for t, (ev, dd) in enumerate(tables):
        s = ev.table.snapshot(dirty_only=True)
        w.add(f"table/{t}-sparse_incr_keys", s["keys"].cpu()); w.add(f"table/{t}-sparse_incr_values", _padded(s["rows"], dd, D))
        ev.table.clear_dirty()
    w.close()
    _write_versions(root, delta={"version": int(version), "base": int(base_version), "prefix": os.path.abspath(prefix)})
    model.train(was_training)
    return prefix
