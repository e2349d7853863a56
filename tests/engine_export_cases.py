"""Shared pieces of the engine-export tests (tests/test_cuda_emu_engine_export.py, tests/test_gpu_zzzzzzzzz_engine_export.py): engines of
every model the zoo adapters accept at small shapes, seeded batches, and the fp32 oracle an export is compared against.

Oracle: the engine's dense module in fp32 without autocast, in eval mode, over fp32 rows read back from the engine's tables (both tiers
of a tiered table, the HBM copy of a key first).  Keys without a row read the default row ``key mod rows(default)``, padding ids read
zero rows, and bags are pooled in fp32 with their combiner, each over its own valid ids."""
from __future__ import annotations

import copy

import numpy as np
import torch

CARDS = [50, 1000, 7, 300] + [97] * 22
SEQ_CARDS = (300, 1000, 50)                  # user, item, cat
L = 8
CRITEO = ["deepfm", "wdl", "dcn", "dcnv2", "masknet", "dlrm_dcn"]
DIN_FAMILY = ["din", "dien", "bst"]
POOLED = ["dssm", "esmm", "mmoe", "dbmtl", "ple", "simple_multitask"]


# ---- engines ------------------------------------------------------------------------------------------------------------------------
def build(name: str, dev):
    import deeprec_b200 as dr
    from deeprec_b200.models.zoo import build_model
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    return build_model(name, device="cpu" if dev.type == "cpu" else dev)


def make_engine(name: str, dev, B: int, combiner: str = "sum", **kw):
    """FusedRecEngine of zoo model ``name`` through its adapter (criteo_engine / din_engine / pooled_seq_engine)."""
    from deeprec_b200.models.rec_engine import criteo_engine, din_engine, pooled_seq_engine
    device = None if dev.type == "cpu" else dev
    model = build(name, dev)
    kw.setdefault("learning_rate", 0.05)
    if name in CRITEO:
        return criteo_engine(model, B, table_rows=CARDS, device=device, **kw)
    if name in DIN_FAMILY:
        return din_engine(model, B, L, table_rows=SEQ_CARDS, device=device, **kw)
    return pooled_seq_engine(model, B, L, combiner=combiner, table_rows=SEQ_CARDS, device=device, **kw)


def dlrm_dcn_engine(dev, B: int, D: int = 16, **kw):
    from dlrm_dcn_cases import small_config
    from deeprec_b200.models.dlrm_engine import DLRMEngine
    mlp_bot = (32, D)
    return DLRMEngine(small_config(batch_size=B, embedding_dim=D, mlp_bot=mlp_bot, **kw), device=None if dev.type == "cpu" else dev)


def criteo_inputs(B: int, seed: int, unseen: int = 0):
    """(ids [26, B], labels [B], dense [B, 13]); ``unseen`` > 0 moves column 1 of the first ``unseen`` samples to keys never trained."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.stack([torch.randint(0, c, (B,), generator=g) for c in CARDS])
    ids[1, :unseen] += 10 ** 9
    return ids, (torch.rand(B, generator=g) < 0.3).float(), torch.rand(B, 13, generator=g) * 3


def taobao_ids(B: int, seed: int, own_cat_padding: bool):
    """[3 + 2L, B] id columns of din_ids with tail-padded histories (some empty); ``own_cat_padding``: the category history has padding of
    its own on top, so the two history bags count different ids."""
    g = torch.Generator().manual_seed(seed)
    n = torch.randint(0, L + 1, (B,), generator=g)
    n[::5] = 0
    pos = torch.arange(L)[None]
    hi = torch.randint(0, SEQ_CARDS[1], (B, L), generator=g)
    hi[:, ::3] = 7
    hc = hi % SEQ_CARDS[2]
    hi[pos >= n[:, None]] = -1
    hc[pos >= n[:, None]] = -1
    if own_cat_padding:
        hc[(torch.rand(B, L, generator=g) < 0.3)] = -1
    head = torch.stack([torch.randint(0, c, (B,), generator=g) for c in SEQ_CARDS])
    return torch.cat([head, hi.t(), hc.t()], 0).contiguous()


def train(eng, name: str, B: int, steps: int, seed: int):
    """``steps`` training steps on seeded batches; returns the (dense, ids) request of the last one."""
    dev = eng.dev
    for s in range(steps):
        if name in CRITEO or name == "dlrm_dcnv2":
            ids, y, dense = criteo_inputs(B, seed + s)
            if name == "dlrm_dcnv2":
                eng.load_batch(dense.to(dev), ids.to(dev), y.to(dev))
            else:
                eng.load_batch(ids.to(dev), y.to(dev), {"dense": dense.to(dev)})
        else:
            ids = taobao_ids(B, seed + s, name in POOLED)
            y = (torch.rand(B, generator=torch.Generator().manual_seed(seed + s)) < 0.3).float()
            if eng.labels.dim() == 2:
                y = torch.stack([y, y * (ids[1] % 2 == 0).float()], 1)
            dense = torch.zeros(B, 1)
            eng.load_batch(ids.to(dev), y.to(dev))
        eng.train_step()
    return dense, ids


# ---- oracle -------------------------------------------------------------------------------------------------------------------------
def _table_rows(tbl, mgr=None):
    """(sorted keys, fp32 rows [n, dim], default [dvd, dim]) of one engine table, both tiers."""
    s = tbl.snapshot()
    keys, rows = s["keys"], s["rows"][:, : tbl.dim].float()
    if mgr is not None:
        mgr.drain()
        h = mgr.host.snapshot()
        extra = ~torch.isin(h["keys"], keys)
        keys, rows = torch.cat([keys, h["keys"][extra]]), torch.cat([rows, h["rows"][extra][:, : tbl.dim].float()])
    o = torch.argsort(keys)
    return keys[o], rows[o], tbl.default_matrix.detach().float().cpu()


def lookup(tab, ids: torch.Tensor) -> torch.Tensor:
    keys, rows, dm = tab
    ids = ids.cpu()
    out = dm[torch.remainder(ids, dm.shape[0])].clone()
    if keys.numel():
        pos = torch.searchsorted(keys, ids).clamp(max=keys.numel() - 1)
        hit = keys[pos] == ids
        out[hit] = rows[pos[hit]]
    out[ids < 0] = 0.0
    return out


def engine_tables(eng):
    return [_table_rows(eng.tables[t], eng.tiers[t][0] if t in getattr(eng, "tiers", {}) else None) for t in range(eng.T)]


def _pool(x: torch.Tensor, valid: torch.Tensor, comb: str) -> torch.Tensor:
    """x [B, L, D] (padding rows already zero), valid [B, L] -> [B, D]."""
    s = x.sum(1)
    n = valid.sum(1, keepdim=True).float()
    if comb == "sum":
        return s
    return torch.where(n > 0, s / (n if comb == "mean" else n.sqrt()).clamp_min(1.0), torch.zeros_like(s))


@torch.no_grad()
def oracle(eng, name: str, dense: torch.Tensor, ids: torch.Tensor, combiner: str = "sum") -> np.ndarray:
    """Probabilities [B] (multi-task: [B, 2] = ctr, cvr) of the engine's current weights and rows in fp32."""
    if name == "dlrm_dcnv2":
        return _dlrm_dcn_oracle(eng, dense, ids)
    tabs = engine_tables(eng)
    net = copy.deepcopy(eng.net.inner).float().cpu().eval()
    cols = [lookup(tabs[t], ids[c]) for c, t in enumerate([0, 1, 2] + [1] * L + [2] * L if name not in CRITEO else range(26))]
    emb = torch.stack(cols, 1)                                           # [B, C, D]
    if name in CRITEO:
        if name == "wdl":
            lin = [_table_rows(eng.lin_tables[t]) for t in range(eng.T)]
            s = sum(lookup(lin[t], ids[t])[:, 0] for t in range(eng.T))
            logits = net.wide_deep_logits(dense, emb, s[:, None])
        else:
            logits = net.logits(dense, emb)
        return torch.sigmoid(logits).numpy()
    u, q = emb[:, 0], torch.cat([emb[:, 1], emb[:, 2]], -1)
    vi, vc = (ids[3:3 + L] >= 0).t(), (ids[3 + L:] >= 0).t()
    if name in DIN_FAMILY:
        k = torch.cat([emb[:, 3:3 + L], emb[:, 3 + L:]], -1)
        return torch.sigmoid(net.head(u, q, k, vi)).numpy()
    pooled = torch.cat([_pool(emb[:, 3:3 + L], vi, combiner), _pool(emb[:, 3 + L:], vc, combiner)], -1)
    if name == "dssm":
        return torch.sigmoid(net.head(u, q, pooled)).numpy()
    out = net.tower_logits(torch.cat([u, q, pooled], -1))
    return torch.stack([torch.sigmoid(out["ctr"]), torch.sigmoid(out["cvr"])], 1).numpy()


def _dlrm_dcn_oracle(eng, dense, ids):
    from dlrm_dcn_cases import oracle_from_engine
    m = oracle_from_engine(eng).eval()
    for L_, bn in zip(eng.bot, [l for l in m.bot if isinstance(l, torch.nn.BatchNorm1d)]):
        bn.running_mean.copy_(L_.running_mean.cpu()); bn.running_var.copy_(L_.running_var.cpu())
    tabs = engine_tables(eng)
    x0 = torch.cat([m.bot(dense), torch.stack([lookup(tabs[t], ids[t]) for t in range(eng.T)], 1).flatten(1)], 1)
    z = x0
    for v, w in zip(m.cross_v, m.cross_w):
        z = x0 * w(v(z)) + z
    return torch.sigmoid(m.logits(m.top(z)).squeeze(-1)).numpy()


def request(name: str, dense: torch.Tensor, ids: torch.Tensor):
    """(dense, ids) numpy arrays of a Processor request: Taobao models take one dummy dense column."""
    if name in CRITEO or name == "dlrm_dcnv2":
        return dense.numpy().astype(np.float32), ids.numpy()
    return np.zeros((ids.shape[1], 1), np.float32), ids.numpy()


def max_err(got: np.ndarray, ref: np.ndarray) -> float:
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert np.isfinite(got).all()
    return float(np.abs(got - ref).max())

