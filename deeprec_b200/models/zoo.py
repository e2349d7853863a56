"""Model zoo on the framework API (modelzoo/ in the reference: 15 models with one flag surface).

Criteo-shaped (dense [B,13], ids [T,B]):  WDL, DLRM (models/dlrm.py), DeepFM, DCN, DCNv2, MaskNet
Taobao-shaped (user/item/cat + behaviour history): DIN, DIEN, BST, DSSM, and the multi-task family ESMM, MMoE, DBMTL,
PLE, SimpleMultiTask.

Layer sizes follow the reference train.py files (wide_and_deep:101, deepfm:73-74, dcn:100, dcnv2:100, dssm:79,
din:143-188, dien, bst:66, esmm:66-70, mmoe:82-88, dbmtl:82-88, ple:83-122, simple_multitask:64, masknet:104).
Every model exposes ``forward(batch) -> logits (or dict of logits)`` and ``loss(batch)``; embeddings are
EmbeddingVariables (``--ev``), optionally grouped (``--group_embedding``) so device tables go through one fused launch.
"""
from __future__ import annotations

import copy
from typing import Dict, List, Optional, Sequence

import torch
from torch import nn
from torch.nn import functional as F

from ..config import EmbeddingVariableOption
from ..embedding_variable import EmbeddingVariable, get_embedding_variable
from ..ops.embedding_ops import SparseIds, group_embedding_lookup_sparse
from .dlrm import DLRM


def _use_fused(device) -> bool:
    """CUDA models run their MLPs on the tensor-core kernels (deeprec_b200.nn) unless DEEPREC_FUSED_NN=0."""
    import os
    return device is not None and torch.device(device).type == "cuda" and os.environ.get("DEEPREC_FUSED_NN", "1") != "0"


def _fast_onehot() -> bool:
    """DEEPREC_FAST_ONEHOT=1: one-hot group lookups skip the bag construction (ops/device_table.group_lookup_dense_device).  Off by
    default."""
    import os
    return os.environ.get("DEEPREC_FAST_ONEHOT", "0") == "1"


def mlp(sizes: Sequence[int], in_dim: int, act=nn.ReLU, bn: bool = False, last_act: bool = True, device=None) -> nn.Module:
    if act is nn.ReLU and _use_fused(device):
        from ..nn import FusedLinear, FusedMLP
        if not bn:
            return FusedMLP(in_dim, sizes, last_act=last_act, device=device)       # whole chain = one autograd node
        layers: List[nn.Module] = []
        k = in_dim
        for i, n in enumerate(sizes):
            has_act = i + 1 < len(sizes) or last_act
            layers.append(FusedLinear(k, n, relu=has_act, device=device))
            if has_act:
                layers.append(nn.BatchNorm1d(n, device=device))
            k = n
        return nn.Sequential(*layers)
    layers = []
    k = in_dim
    for i, n in enumerate(sizes):
        layers.append(nn.Linear(k, n, device=device))
        if i + 1 < len(sizes) or last_act:
            layers.append(act())
            if bn:
                layers.append(nn.BatchNorm1d(n, device=device))
        k = n
    return nn.Sequential(*layers)


class _Tables(nn.Module):
    """T one-hot categorical features -> [B, T, D] (EmbeddingVariables, optionally one fused group lookup)."""

    def __init__(self, names: Sequence[str], dim: int, ev_option: Optional[EmbeddingVariableOption], device, group: bool, prefix: str):
        super().__init__()
        self.group = group
        variant = _TABLE_VARIANT["kind"]
        if variant == "multihash":         # --multihash: Q-R compositional embeddings instead of one row per id (modelzoo/features/multihash_variable)
            from ..embedding_variable import get_multihash_variable
            self.group = False
            self.tables = nn.ModuleList([get_multihash_variable(f"{prefix}/{n}", [[_TABLE_VARIANT["q_rows"], dim], [_TABLE_VARIANT["r_rows"], dim]], device=device)
                                         for n in names])
        elif variant == "adaptive":        # --adaptive_emb: hot ids -> EmbeddingVariable, cold ids -> static hashed table (features/adaptive_embedding)
            self.group = False
            self.tables = nn.ModuleList([AdaptiveEmbedding(f"{prefix}/{n}", dim, _TABLE_VARIANT["hash_bucket_size"], _TABLE_VARIANT["hot_freq"], ev_option, device)
                                         for n in names])
        else:
            self.tables = nn.ModuleList([get_embedding_variable(f"{prefix}/{n}", dim, ev_option=copy.deepcopy(ev_option) if ev_option else None, device=device)
                                         for n in names])

    def forward(self, ids: torch.Tensor) -> torch.Tensor:          # ids [T, B]
        from ..parallel import strategy as _strategy
        st = _strategy.current()
        model_parallel = st is not None and st.in_embedding_scope and st.world_size > 1 and isinstance(self.tables[0], EmbeddingVariable)
        if not model_parallel and self.group and self.tables[0].device.type == "cuda" and _fast_onehot():
            from ..ops.device_table import group_lookup_dense_device
            out = group_lookup_dense_device(list(self.tables), ids)          # [B, T, D]; None if the tables cannot share a launch
            if out is not None:
                return out
        if not model_parallel and isinstance(self.tables[0], EmbeddingVariable) and self.tables[0].device.type == "cpu":
            from ..ops.host_group import group_lookup_dense_host
            out = group_lookup_dense_host(list(self.tables), ids)            # [B, T, D] from one native call; None for tiered tables
            if out is not None:
                return out
        if model_parallel or (self.group and self.tables[0].device.type == "cuda"):
            sps = [SparseIds.from_dense(ids[i]) for i in range(len(self.tables))]
            outs = group_embedding_lookup_sparse(list(self.tables), sps, ["sum"] * len(sps))
            return torch.stack(outs, dim=1)
        return torch.stack([t.lookup(ids[i]) for i, t in enumerate(self.tables)], dim=1)

    def embedding_variables(self) -> List[EmbeddingVariable]:
        return [t for t in self.modules() if isinstance(t, EmbeddingVariable)]


# process-wide switch set by ``table_variant(...)`` (the modelzoo's --multihash / --adaptive_emb flags pick it before build_model)
_TABLE_VARIANT = {"kind": "ev", "q_rows": 1 << 12, "r_rows": 1 << 12, "hash_bucket_size": 1 << 14, "hot_freq": 3}


def table_variant(kind: str = "ev", **kw) -> None:
    if kind not in ("ev", "multihash", "adaptive"):
        raise ValueError("table variant must be ev | multihash | adaptive")
    _TABLE_VARIANT.update(kind=kind, **kw)


class AdaptiveEmbedding(nn.Module):
    """Adaptive embedding (docs/docs_en/Adaptive-Embedding.md; embedding_ops.py:668-836): every id trains a row of a static hashed table
    until it has been seen ``hot_freq`` times, from then on it owns an EmbeddingVariable row (selected per id by the adaptive mask)."""

    def __init__(self, name: str, dim: int, hash_bucket_size: int, hot_freq: int, ev_option, device):
        super().__init__()
        opt = copy.deepcopy(ev_option) if ev_option else EmbeddingVariableOption()
        self.ev = get_embedding_variable(name, dim, ev_option=opt, device=device)
        self.hashed = nn.Embedding(hash_bucket_size, dim, device=device)
        nn.init.normal_(self.hashed.weight, 0.0, 1.0 / dim ** 0.5)
        self.hot_freq, self.embedding_dim, self.name = hot_freq, dim, name

    def lookup(self, ids: torch.Tensor) -> torch.Tensor:
        from ..ops.embedding_ops import adaptive_embedding_lookup_sparse
        flat = ids.reshape(-1)
        hot = self.ev.get_frequency(flat.to(self.ev.device)) >= self.hot_freq           # adaptive mask
        sp = SparseIds.from_dense(flat)
        hashed_ids = SparseIds.from_dense(torch.remainder(flat, self.hashed.num_embeddings))
        # the EV is looked up for every id (cold ids get a zero gradient through the mask), so occurrences of cold ids are still
        # counted by the EV's frequency and the id turns hot after ``hot_freq`` sightings
        out = adaptive_embedding_lookup_sparse(self.hashed, self.ev, sp, hashed_ids, combiner="sum", adaptive_mask_tensor=hot.to(flat.device))
        return out.view(*ids.shape, self.embedding_dim)

    forward = lookup


class CriteoModel(nn.Module):
    num_dense, num_sparse = 13, 26

    def __init__(self, emb_dim: int = 16, ev_option=None, device=None, group_embedding: bool = False, name: str = "model"):
        super().__init__()
        self.emb_dim = emb_dim
        self.emb = _Tables([f"C{i + 1}" for i in range(self.num_sparse)], emb_dim, ev_option, device, group_embedding, name)

    def logits(self, dense, embs):
        raise NotImplementedError

    def forward(self, dense: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
        return self.logits(dense, self.emb(ids).to(dense.device))

    def loss(self, dense, ids, labels):
        return F.binary_cross_entropy_with_logits(self.forward(dense, ids), labels)


class WDL(CriteoModel):
    """Wide & Deep: linear (dim-1 embeddings) + DNN [1024, 512, 256]."""

    def __init__(self, dnn_hidden_units=(1024, 512, 256), **kw):
        super().__init__(name=kw.pop("name", "wdl"), **kw)
        dev = kw.get("device")
        self.wide = _Tables([f"C{i + 1}_wide" for i in range(self.num_sparse)], 4, kw.get("ev_option"), dev, False, "wdl")
        self.wide_dense = nn.Linear(self.num_dense, 1, device=dev)
        self.deep = mlp(dnn_hidden_units, self.num_dense + self.num_sparse * self.emb_dim, device=dev)
        self.out = nn.Linear(dnn_hidden_units[-1], 1, device=dev)
        self._ids = None

    def forward(self, dense, ids):
        self._ids = ids
        return super().forward(dense, ids)

    def logits(self, dense, embs):
        wide = self.wide(self._ids).to(dense.device)[..., 0].sum(1, keepdim=True) + self.wide_dense(dense)     # linear part
        deep = self.out(self.deep(torch.cat([dense, embs.flatten(1)], 1)))
        return (wide + deep).squeeze(-1)


class DeepFM(CriteoModel):
    """FM second order 0.5((sum v)^2 - sum v^2) + linear + DNN [1024,256,32] -> final [128,64] (deepfm/train.py:178-191)."""

    def __init__(self, dnn_hidden_units=(1024, 256, 32), final_hidden_units=(128, 64), **kw):
        super().__init__(name=kw.pop("name", "deepfm"), **kw)
        dev = kw.get("device")
        self.linear = nn.Linear(self.num_dense, 1, device=dev)
        self.dnn = mlp(dnn_hidden_units, self.num_dense + self.num_sparse * self.emb_dim, bn=True, device=dev)
        self.final = mlp(final_hidden_units, dnn_hidden_units[-1] + self.emb_dim + 1, device=dev)
        self.out = nn.Linear(final_hidden_units[-1], 1, device=dev)

    def logits(self, dense, embs):
        from ..nn import fm_interaction
        fm = fm_interaction(embs)
        dnn = self.dnn(torch.cat([dense, embs.flatten(1)], 1))
        return self.out(self.final(torch.cat([self.linear(dense), fm, dnn], 1))).squeeze(-1)


class DCN(CriteoModel):
    """Deep & Cross: x_{l+1} = x0 (x_l . w_l) + b_l + x_l, DNN [1024,512,256]."""

    def __init__(self, dnn_hidden_units=(1024, 512, 256), cross_layers: int = 3, **kw):
        super().__init__(name=kw.pop("name", "dcn"), **kw)
        dev = kw.get("device")
        d = self.num_dense + self.num_sparse * self.emb_dim
        self.cw = nn.ParameterList([nn.Parameter(torch.randn(d, device=dev) * 0.01) for _ in range(cross_layers)])
        self.cb = nn.ParameterList([nn.Parameter(torch.zeros(d, device=dev)) for _ in range(cross_layers)])
        self.deep = mlp(dnn_hidden_units, d, device=dev)
        self.out = nn.Linear(d + dnn_hidden_units[-1], 1, device=dev)

    def _cross(self, x0):
        x = x0
        for w, b in zip(self.cw, self.cb):
            x = x0 * (x @ w).unsqueeze(-1) + b + x
        return x

    def logits(self, dense, embs):
        x0 = torch.cat([dense, embs.flatten(1)], 1)
        return self.out(torch.cat([self._cross(x0), self.deep(x0)], 1)).squeeze(-1)


class DCNv2(DCN):
    """DCN-v2: full-rank (or low-rank) matrix cross  x_{l+1} = x0 * (W x_l + b) + x_l."""

    def __init__(self, low_rank: int = 0, cross_layers: int = 3, **kw):
        super().__init__(cross_layers=cross_layers, name=kw.pop("name", "dcnv2"), **kw)
        dev = kw.get("device")
        d = self.num_dense + self.num_sparse * self.emb_dim
        self.W = nn.ModuleList([nn.Linear(d, d, device=dev) if not low_rank else
                                nn.Sequential(nn.Linear(d, low_rank, bias=False, device=dev), nn.Linear(low_rank, d, device=dev)) for _ in range(cross_layers)])

    def _cross(self, x0):
        x = x0
        for W in self.W:
            x = x0 * W(x) + x
        return x


class MaskNet(CriteoModel):
    """Serial MaskBlocks: instance-guided mask (MLP on the embedding) * LayerNorm(hidden) (masknet/train.py:160-220)."""

    def __init__(self, dnn_hidden_units=(64, 64, 64), **kw):
        super().__init__(name=kw.pop("name", "masknet"), **kw)
        dev = kw.get("device")
        d = self.num_sparse * self.emb_dim
        self.ln_emb = nn.LayerNorm(d, device=dev)
        self.blocks, self.masks = nn.ModuleList(), nn.ModuleList()
        k = d
        for n in dnn_hidden_units:
            self.masks.append(nn.Sequential(nn.Linear(d, 2 * d, device=dev), nn.ReLU(), nn.Linear(2 * d, k, device=dev)))
            self.blocks.append(nn.Sequential(nn.Linear(k, n, device=dev), nn.LayerNorm(n, device=dev), nn.ReLU()))
            k = n
        self.out = mlp((64, 16, 1), k + self.num_dense, last_act=False, device=dev)

    def logits(self, dense, embs):
        v = embs.flatten(1)
        h = self.ln_emb(v)
        for m, b in zip(self.masks, self.blocks):
            h = b(h * m(v))
        return self.out(torch.cat([h, dense], 1)).squeeze(-1)


# --------------------------------------------------------------------------------------------------------------
# Taobao-shaped models
# --------------------------------------------------------------------------------------------------------------
class _SeqBase(nn.Module):
    def __init__(self, emb_dim=16, ev_option=None, device=None, name="seq"):
        super().__init__()
        mk = lambda n: get_embedding_variable(f"{name}/{n}", emb_dim, ev_option=copy.deepcopy(ev_option) if ev_option else None, device=device)
        self.user, self.item, self.cat = mk("user"), mk("item"), mk("cat")
        self.emb_dim, self.device = emb_dim, device

    def _embed(self, b: Dict[str, torch.Tensor]):
        u = self.user.lookup(b["user"])
        q = torch.cat([self.item.lookup(b["item"]), self.cat.lookup(b["cat"])], -1)                   # [B, 2D] target
        hi, hc = b["hist_item"], b["hist_cat"]
        mask = (hi >= 0)
        if hi.device.type == "cpu" and self.item.device.type == "cpu":
            from ..config import PAD_KEY                     # host tables: padding positions are not looked up at all (zero rows, no statistics)
            hi_l, hc_l = torch.where(mask, hi, PAD_KEY), torch.where(mask, hc, PAD_KEY)
        else:
            hi_l, hc_l = hi.clamp_min(0), hc.clamp_min(0)
        k = torch.cat([self.item.lookup(hi_l), self.cat.lookup(hc_l)], -1)                            # [B, L, 2D]
        k = k * mask.unsqueeze(-1).to(k.dtype).to(k.device)
        return u, q, k, mask.to(k.device)

    def _embed_pooled(self, b: Dict[str, torch.Tensor]):
        """(user, target, sum-pooled history [B, 2D]) for models that only consume the pooled behaviour history: the ``[B, L, 2D]``
        history tensor is never built on host tables (``EmbeddingVariable.lookup_pooled``)."""
        u = self.user.lookup(b["user"])
        q = torch.cat([self.item.lookup(b["item"]), self.cat.lookup(b["cat"])], -1)
        hi, hc = b["hist_item"], b["hist_cat"]
        mask = hi >= 0
        pooled = torch.cat([self.item.lookup_pooled(hi, mask), self.cat.lookup_pooled(hc, mask)], -1)
        return u, q, pooled

    def loss(self, b):
        out = self.forward(b)
        return F.binary_cross_entropy_with_logits(out, b["labels"].to(out.device))


def din_attention(q, k, mask, att: nn.Module):
    """DIN attention unit: concat[q, k, q-k, q*k] -> 80 -> 40 -> 1 (sigmoid acts), masked softmax, weighted sum
    (composite autograd path for training, one fused kernel for CUDA inference: ops/attention.py)."""
    from ..ops.attention import din_attention as _impl
    return _impl(q, k, mask, att)


class DIN(_SeqBase):
    def __init__(self, **kw):
        super().__init__(name=kw.pop("name", "din"), **kw)
        D2, dev = 2 * self.emb_dim, self.device
        self.att = nn.Sequential(nn.Linear(4 * D2, 80, device=dev), nn.Sigmoid(), nn.Linear(80, 40, device=dev), nn.Sigmoid(), nn.Linear(40, 1, device=dev))
        self.bn = nn.BatchNorm1d(self.emb_dim + 3 * D2, device=dev)
        self.top = nn.Sequential(nn.Linear(self.emb_dim + 3 * D2, 200, device=dev), nn.PReLU(device=dev), nn.Linear(200, 80, device=dev), nn.PReLU(device=dev),
                                 nn.Linear(80, 1, device=dev))

    def head(self, u, q, k, mask):
        """Dense part on already-looked-up embeddings (user [B, D], target [B, 2D], history [B, L, 2D] zero-padded, mask [B, L]) --
        what :func:`models.rec_engine.din_engine` runs on top of the unique-first sparse pipeline."""
        pooled = k.sum(1)
        att = din_attention(q, k, mask, self.att)
        return self.top(self.bn(torch.cat([u, q, pooled, att], -1))).squeeze(-1)

    def forward(self, b):
        return self.head(*self._embed(b))


class DIEN(_SeqBase):
    """Interest extractor GRU + attention-gated evolution GRU (AUGRU approximated by attention-weighted GRU inputs)."""

    def __init__(self, hidden: int = 32, **kw):
        super().__init__(name=kw.pop("name", "dien"), **kw)
        D2, dev = 2 * self.emb_dim, self.device
        self.gru1 = nn.GRU(D2, hidden, batch_first=True, device=dev)
        self.gru2 = nn.GRU(hidden, hidden, batch_first=True, device=dev)
        self.qproj = nn.Linear(D2, hidden, device=dev)
        self.att = nn.Sequential(nn.Linear(4 * hidden, 80, device=dev), nn.Sigmoid(), nn.Linear(80, 40, device=dev), nn.Sigmoid(), nn.Linear(40, 1, device=dev))
        self.top = nn.Sequential(nn.Linear(self.emb_dim + D2 + hidden + D2, 200, device=dev), nn.PReLU(device=dev), nn.Linear(200, 80, device=dev), nn.PReLU(device=dev),
                                 nn.Linear(80, 1, device=dev))

    def forward(self, b):
        u, q, k, mask = self._embed(b)
        h1, _ = self.gru1(k)
        qh = self.qproj(q).unsqueeze(1).expand_as(h1)
        s = self.att(torch.cat([qh, h1, qh - h1, qh * h1], -1)).squeeze(-1).masked_fill(~mask, -2 ** 31)
        w = torch.softmax(s, -1).unsqueeze(-1)
        h2, _ = self.gru2(h1 * w)
        lens = mask.sum(1).clamp_min(1) - 1
        final = h2[torch.arange(h2.shape[0], device=h2.device), lens]
        return self.top(torch.cat([u, q, final, k.sum(1)], -1)).squeeze(-1)


class BST(_SeqBase):
    """Behaviour Sequence Transformer: one encoder block over [history; target], final [512, 256, 64]."""

    def __init__(self, heads: int = 4, final_hidden_units=(512, 256, 64), max_len: int = 64, **kw):
        super().__init__(name=kw.pop("name", "bst"), **kw)
        D2, dev = 2 * self.emb_dim, self.device
        self.pos = nn.Parameter(torch.zeros(max_len + 1, D2, device=dev))
        self.enc = nn.TransformerEncoderLayer(D2, heads, 4 * D2, dropout=0.0, batch_first=True, device=dev)
        self.final = mlp(final_hidden_units, self.emb_dim + 2 * D2, device=dev)
        self.out = nn.Linear(final_hidden_units[-1], 1, device=dev)

    def forward(self, b):
        u, q, k, mask = self._embed(b)
        x = torch.cat([k, q.unsqueeze(1)], 1)
        x = x + self.pos[: x.shape[1]]
        pad = torch.cat([~mask, torch.zeros(mask.shape[0], 1, dtype=torch.bool, device=mask.device)], 1)
        h = self.enc(x, src_key_padding_mask=pad)
        valid = (~pad).unsqueeze(-1).to(h.dtype)
        pooled = (h * valid).sum(1) / valid.sum(1).clamp_min(1)
        return self.out(self.final(torch.cat([u, q, pooled], -1))).squeeze(-1)


class DSSM(_SeqBase):
    """Two towers [256,128,64,32], cosine similarity."""

    def __init__(self, dnn_hidden_units=(256, 128, 64, 32), **kw):
        super().__init__(name=kw.pop("name", "dssm"), **kw)
        D2, dev = 2 * self.emb_dim, self.device
        self.user_tower = mlp(dnn_hidden_units, self.emb_dim + D2, last_act=False, device=dev)
        self.item_tower = mlp(dnn_hidden_units, D2, last_act=False, device=dev)
        self.scale = nn.Parameter(torch.tensor(5.0, device=dev))

    def forward(self, b):
        u, q, pooled = self._embed_pooled(b)
        ue = self.user_tower(torch.cat([u, pooled], -1))
        ie = self.item_tower(q)
        return F.cosine_similarity(ue, ie, dim=-1) * self.scale


class _MultiTask(_SeqBase):
    tasks = ("ctr", "cvr")

    def _features(self, b):
        u, q, pooled = self._embed_pooled(b)
        return torch.cat([u, q, pooled], -1)

    @property
    def feat_dim(self):
        return self.emb_dim + 4 * self.emb_dim

    def loss(self, b):
        out = self.forward(b)
        y = b["labels"].to(next(iter(out.values())).device)
        y2 = y * (b["item"].to(y.device) % 2 == 0).to(y.dtype)          # synthetic conversion label nested in clicks
        return F.binary_cross_entropy_with_logits(out["ctr"], y) + F.binary_cross_entropy_with_logits(out.get("ctcvr", out["cvr"]), y2)


class ESMM(_MultiTask):
    """pCTCVR = pCTR * pCVR over the entire space (esmm/train.py:66-70 MLP sizes)."""

    def __init__(self, ctr_mlp=(256, 128, 96, 64), cvr_mlp=(256, 128, 96, 64), **kw):
        super().__init__(name=kw.pop("name", "esmm"), **kw)
        dev = self.device
        self.ctr = nn.Sequential(mlp(ctr_mlp, self.feat_dim, device=dev), nn.Linear(ctr_mlp[-1], 1, device=dev))
        self.cvr = nn.Sequential(mlp(cvr_mlp, self.feat_dim, device=dev), nn.Linear(cvr_mlp[-1], 1, device=dev))

    def forward(self, b):
        f = self._features(b)
        ctr, cvr = self.ctr(f).squeeze(-1), self.cvr(f).squeeze(-1)
        p = (torch.sigmoid(ctr) * torch.sigmoid(cvr)).clamp(1e-7, 1 - 1e-7)
        return {"ctr": ctr, "cvr": cvr, "ctcvr": torch.log(p) - torch.log1p(-p)}


class MMoE(_MultiTask):
    def __init__(self, num_experts: int = 3, expert_hidden_units=(256, 192, 128, 64), tower=(256, 192, 128, 64), **kw):
        super().__init__(name=kw.pop("name", "mmoe"), **kw)
        dev = self.device
        self.experts = nn.ModuleList([mlp(expert_hidden_units, self.feat_dim, device=dev) for _ in range(num_experts)])
        self.gates = nn.ModuleDict({t: nn.Linear(self.feat_dim, num_experts, device=dev) for t in self.tasks})
        self.towers = nn.ModuleDict({t: nn.Sequential(mlp(tower, expert_hidden_units[-1], device=dev), nn.Linear(tower[-1], 1, device=dev)) for t in self.tasks})

    def forward(self, b):
        f = self._features(b)
        e = torch.stack([x(f) for x in self.experts], 1)
        return {t: self.towers[t]((torch.softmax(self.gates[t](f), -1).unsqueeze(-1) * e).sum(1)).squeeze(-1) for t in self.tasks}


class DBMTL(_MultiTask):
    """Bottom DNN [1024,512,256] + per-task towers, cvr tower conditioned on the ctr tower (Bayesian relation)."""

    def __init__(self, bottom=(1024, 512, 256), tower=(256, 128, 64, 32), **kw):
        super().__init__(name=kw.pop("name", "dbmtl"), **kw)
        dev = self.device
        self.bottom = mlp(bottom, self.feat_dim, device=dev)
        self.t_ctr = mlp(tower, bottom[-1], device=dev)
        self.t_cvr = mlp(tower, bottom[-1], device=dev)
        self.rel = mlp((32,), 2 * tower[-1], device=dev)
        self.o_ctr, self.o_cvr = nn.Linear(tower[-1], 1, device=dev), nn.Linear(32, 1, device=dev)

    def forward(self, b):
        s = self.bottom(self._features(b))
        a, c = self.t_ctr(s), self.t_cvr(s)
        return {"ctr": self.o_ctr(a).squeeze(-1), "cvr": self.o_cvr(self.rel(torch.cat([a, c], -1))).squeeze(-1)}


class PLE(_MultiTask):
    """Progressive Layered Extraction: per layer shared + task-specific experts with gated fusion (ple/train.py:118-122)."""

    def __init__(self, num_layers: int = 2, shared_expert_num: int = 1, specific_expert_num: int = 2, expert_units=(256, 128, 64), tower=(256, 128, 64), **kw):
        super().__init__(name=kw.pop("name", "ple"), **kw)
        dev = self.device
        self.layers = nn.ModuleList()
        d = self.feat_dim
        for _ in range(num_layers):
            L = nn.ModuleDict({
                "shared": nn.ModuleList([mlp(expert_units, d, device=dev) for _ in range(shared_expert_num)]),
                **{f"spec_{t}": nn.ModuleList([mlp(expert_units, d, device=dev) for _ in range(specific_expert_num)]) for t in self.tasks},
                **{f"gate_{t}": nn.Linear(d, shared_expert_num + specific_expert_num, device=dev) for t in self.tasks},
                "gate_shared": nn.Linear(d, shared_expert_num + specific_expert_num * len(self.tasks), device=dev)})
            self.layers.append(L)
            d = expert_units[-1]
        self.towers = nn.ModuleDict({t: nn.Sequential(mlp(tower, d, device=dev), nn.Linear(tower[-1], 1, device=dev)) for t in self.tasks})

    def forward(self, b):
        f = self._features(b)
        xs = {t: f for t in self.tasks}
        xs["shared"] = f
        for L in self.layers:
            sh = [e(xs["shared"]) for e in L["shared"]]
            sp = {t: [e(xs[t]) for e in L[f"spec_{t}"]] for t in self.tasks}
            nxt = {}
            for t in self.tasks:
                e = torch.stack(sp[t] + sh, 1)
                nxt[t] = (torch.softmax(L[f"gate_{t}"](xs[t]), -1).unsqueeze(-1) * e).sum(1)
            allx = torch.stack([x for t in self.tasks for x in sp[t]] + sh, 1)
            nxt["shared"] = (torch.softmax(L["gate_shared"](xs["shared"]), -1).unsqueeze(-1) * allx).sum(1)
            xs = nxt
        return {t: self.towers[t](xs[t]).squeeze(-1) for t in self.tasks}


class SimpleMultiTask(_MultiTask):
    """Two independent towers [256,196,128,64] on shared embeddings."""

    def __init__(self, hidden=(256, 196, 128, 64), **kw):
        super().__init__(name=kw.pop("name", "simple_multitask"), **kw)
        dev = self.device
        self.towers = nn.ModuleDict({t: nn.Sequential(mlp(hidden, self.feat_dim, device=dev), nn.Linear(hidden[-1], 1, device=dev)) for t in self.tasks})

    def forward(self, b):
        f = self._features(b)
        return {t: self.towers[t](f).squeeze(-1) for t in self.tasks}


class DLRMDCN(CriteoModel):
    """MLPerf DLRM-DCNv2 (modelzoo/mlperf): DLRM bottom MLP on the dense features, low-rank DCNv2 cross layers over
    [bottom | embeddings] as the interaction, top MLP on the crossed vector."""

    def __init__(self, bot=(512, 256), top=(1024, 1024, 512, 256), cross_layers: int = 3, low_rank: int = 512, **kw):
        super().__init__(name=kw.pop("name", "dlrm_dcn"), **kw)
        dev = self.emb.tables[0].device if hasattr(self.emb.tables[0], "device") else None
        D = self.emb_dim
        self.bot = mlp(list(bot) + [D], self.num_dense, device=dev)
        n = D * (self.num_sparse + 1)
        r = min(low_rank, n)
        self.U = nn.ParameterList([nn.Parameter(torch.randn(n, r, device=dev) / n ** 0.5) for _ in range(cross_layers)])
        self.V = nn.ParameterList([nn.Parameter(torch.randn(r, n, device=dev) / r ** 0.5) for _ in range(cross_layers)])
        self.cb = nn.ParameterList([nn.Parameter(torch.zeros(n, device=dev)) for _ in range(cross_layers)])
        self.top = mlp(list(top), n, device=dev)
        self.out = nn.Linear(top[-1], 1, device=dev)

    def logits(self, dense, embs):
        x0 = torch.cat([self.bot(dense).unsqueeze(1), embs], 1).flatten(1)
        x = x0
        for U, V, b in zip(self.U, self.V, self.cb):
            x = x0 * ((x @ U) @ V + b) + x                     # x_{l+1} = x0 * (U V x_l + b) + x_l
        return self.out(self.top(x)).squeeze(-1)


CRITEO_MODELS = {"wdl": WDL, "wide_and_deep": WDL, "deepfm": DeepFM, "dcn": DCN, "dcnv2": DCNv2, "masknet": MaskNet, "dlrm_dcn": DLRMDCN,
                 "mlperf": DLRMDCN}
TAOBAO_MODELS = {"din": DIN, "dien": DIEN, "bst": BST, "dssm": DSSM, "esmm": ESMM, "mmoe": MMoE, "dbmtl": DBMTL, "ple": PLE,
                 "simple_multitask": SimpleMultiTask}


def build_model(name: str, ev_option=None, device=None, group_embedding: bool = False, emb_dim: int = 16, cardinalities=None):
    name = name.lower()
    if name == "dlrm":
        return DLRM(13, cardinalities or [1000] * 26, emb_dim, ev_option=ev_option, device=device)
    if name in CRITEO_MODELS:
        return CRITEO_MODELS[name](emb_dim=emb_dim, ev_option=ev_option, device=device, group_embedding=group_embedding)
    if name in TAOBAO_MODELS:
        return TAOBAO_MODELS[name](emb_dim=emb_dim, ev_option=ev_option, device=device)
    raise KeyError(f"unknown model {name}; available: dlrm, {', '.join(list(CRITEO_MODELS) + list(TAOBAO_MODELS))}")
