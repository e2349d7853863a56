"""Cases of the multi-hot bags -- k_sp_pool / k_sp_pool_segsum (csrc/cuda/sparse_pipeline.cu), FusedRecEngine(bags=...) and
models.rec_engine.pooled_seq_engine -- shared by the CUDA-on-CPU emulation tests (test_cuda_emu_pooled_bags.py) and the H100 tests
(test_gpu_pooled_bags.py).

Oracles:
- pool: numpy's float32 sum of the live rows of each bag in column order, times w = 1, 1/n or 1/sqrt(n) (float32, correctly rounded), rounded
  to bf16, bit for bit; size-1 sum bags against k_sp_gather;
- pool_segsum: with sum bags, k_sp_segsum on the bag gradient repeated per column, bit for bit; with mean / sqrtn bags, the fp64 per-key sum of
  dpool * w within the fp32 rounding of the products and of one warp tile's partial sum;
- the engines: a torch replica with nn.Embedding tables copied from the engine's default matrices, pooled with ops.embedding_ops._combine, and
  the model's own loss (the bounds of the DeepFM / WDL engine tests: loss within 3 %, rows within 0.05).
"""
from __future__ import annotations

import copy
import threading

import numpy as np
import torch

D = 16
NO_PERMISSION = 0.375
HOT_KEY = 4242
KCARD = 500
# bag sizes 1, 3 and 100 (and a second 1 / 3); the columns of a bag come from several tables (col_table[c] = c % 4)
BAG_SIZES = [1, 3, 100, 1, 3]
NT = 4


# ---- kernels ----------------------------------------------------------------------------------------------------------------------
def make_tables(dev, owner: int, filter_even: bool):
    """NT dim-16 tables; with ``filter_even`` the even tables admit a key on its 2nd sighting (CounterFilter) and read ``NO_PERMISSION`` until
    then."""
    from deeprec_b200._native import EvConfig
    from deeprec_b200.ops.device_table import DeviceTable, get_context
    ctx = get_context(dev, D, owner=owner)
    tables = []
    for t in range(NT):
        c = EvConfig()
        c.dim, c.num_slots, c.has_scalars = D, 1, 0
        c.init_capacity = 4096
        ff = 2 if filter_even and t % 2 == 0 else 0
        c.filter_type, c.filter_freq = (1, ff) if ff else (0, 0)
        c.bloom_counter_bits = 32
        c.steps_to_live, c.l2_weight_threshold = 0, -1.0
        c.default_value_dim, c.default_value_no_permission = 4096, NO_PERMISSION
        c.record_freq = c.record_version = 1
        c.storage_type = 1
        c.slot_init[0] = 0.1
        g = torch.Generator().manual_seed(17 + t)
        dm = torch.empty(4096, D).normal_(0.0, 0.5, generator=g)
        tables.append(DeviceTable(c, dm, dev, capacity=1 << 14, row_capacity=1 << 13, owner=owner))
    tmap = torch.tensor([t.gid for t in tables], dtype=torch.int32, device=dev)
    return ctx, tables, tmap


def kernel_batch(B: int, seed: int, sizes=BAG_SIZES):
    """ids [C, B]: ~1/9 padding; bag 1 is all padding for every 7th sample; a hot key fills every 4th position of the largest bag; dpool
    [F, B, D] bf16 spanning four decades."""
    g = torch.Generator().manual_seed(seed)
    C, F = sum(sizes), len(sizes)
    ids = torch.randint(0, KCARD, (C, B), generator=g)
    b = torch.arange(B)
    for c in range(C):
        ids[c, (b + c) % 9 == 0] = -1
    off = np.cumsum([0] + list(sizes))
    big = int(np.argmax(sizes))
    ids[off[big]:off[big + 1]:4] = HOT_KEY
    if F > 1 and sizes[1] > 0:
        ids[off[1]:off[2], b % 7 == 0] = -1
    dpool = (torch.randn(F, B, D, generator=g) * 10.0 ** torch.randint(-5, -1, (F, B, 1), generator=g).float()).bfloat16()
    return ids, dpool


def pool_oracle(urow: torch.Tensor, inv: torch.Tensor, sizes, combs):
    """(bf16 [B, F, D], fp32 [F, B]): the float32 sequential sum of each bag's live rows times w, rounded to bf16 once."""
    u = urow.float().cpu().numpy()
    inv = inv.cpu().numpy()
    B = inv.shape[0]
    out = np.zeros((B, len(sizes), u.shape[1]), dtype=np.float32)
    wo = np.zeros((len(sizes), B), dtype=np.float32)
    c0 = 0
    for f, (n, comb) in enumerate(zip(sizes, combs)):
        acc = np.zeros((B, u.shape[1]), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.int64)
        for c in range(c0, c0 + n):
            gs = inv[:, c]
            live = gs >= 0
            acc = (acc + np.where(live[:, None], u[np.maximum(gs, 0)], np.float32(0.0))).astype(np.float32)
            cnt += live
        nf = cnt.astype(np.float32)
        with np.errstate(divide="ignore"):
            w = {"sum": np.ones(B, np.float32), "mean": np.float32(1.0) / nf, "sqrtn": np.float32(1.0) / np.sqrt(nf)}[comb].astype(np.float32)
        w[cnt == 0] = 0.0
        out[:, f] = (acc * w[:, None]).astype(np.float32)
        wo[f] = w
        c0 += n
    return torch.from_numpy(out).bfloat16(), torch.from_numpy(wo)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.cpu().contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def run_kernels_world1(dev, comb: str, B: int, owner: int, graph: bool = False):
    """dedup -> lookup -> pool -> pool_segsum at world 1 (optionally replayed from a CUDA graph) against the oracles; size-1 sum bags against
    gather; sum bags' pool_segsum against segsum on the repeated gradient."""
    from deeprec_b200.parallel.sparse_pipeline import Bags, SparsePipeline
    sizes = BAG_SIZES
    C, F = sum(sizes), len(sizes)
    ids, dpool = kernel_batch(B, seed=60 + len(comb))
    ctx, tables, tmap = make_tables(dev, owner, filter_even=True)
    col_table = [c % NT for c in range(C)]
    sp = SparsePipeline(dev, 0, 1, col_table, NT, B, D)
    ctx.ensure(sp.Btot)
    bags = Bags(dev, [(n, comb) for n in sizes], C)
    ones = Bags(dev, [(1, "sum")] * C, C)
    ids_d, dp_d = ids.to(dev), dpool.to(dev)
    out = torch.full((B, F, D), float("nan"), dtype=torch.bfloat16, device=dev)
    w = torch.full((F, B), float("nan"), dtype=torch.float32, device=dev)
    out1 = torch.full((B, C, D), float("nan"), dtype=torch.bfloat16, device=dev)
    w1 = torch.zeros(C, B, dtype=torch.float32, device=dev)
    gat = torch.full((B, C, D), float("nan"), dtype=torch.bfloat16, device=dev)

    def body():
        sp.dedup(ids_d)
        sp.lookup(ctx, tmap, True)
        sp.pool(out, w, bags)
        sp.pool(out1, w1, ones)
        sp.gather(gat)
        sp.pool_segsum(dp_d, w, bags)

    if graph:
        body()                       # eager first: fresh keys are inserted, so the captured replay below reads the same rows
        torch.cuda.synchronize()
        eager = (out.clone(), w.clone(), sp.ugrad[sp.invT.clamp_min(0).long()].clone())
        sp.reset(); sp.step_end()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                body()
        torch.cuda.current_stream().wait_stream(s)
        out.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
    else:
        body()
    inv, invT = sp.inv.clone(), sp.invT.clone()
    urow, ugrad = sp.urow.clone(), sp.ugrad.clone()
    want, want_w = pool_oracle(urow, inv[:, :C], sizes, [comb] * F)
    assert torch.equal(_bits(w), _bits(want_w)), "pool: w != 1, 1/n or 1/sqrt(n)"
    assert torch.equal(_bits(out), _bits(want)), "pool != float32 sequential bag sum times w"
    assert torch.equal(_bits(out1), _bits(gat)), "size-1 sum bags != gather"
    assert bool((w[1].cpu()[torch.arange(B) % 7 == 0] == 0).all()) and bool((out[torch.arange(B, device=dev) % 7 == 0, 1].float() == 0).all())
    assert not bool(torch.isnan(out.float()).any())
    # the rejected keys of the filtered tables read NO_PERMISSION and count
    live0 = ids[0] >= 0
    assert bool((urow[inv[:, 0][live0.to(inv.device)].long()].float() == NO_PERMISSION).all())
    if graph:
        assert torch.equal(eager[0], out) and torch.equal(eager[1], w) and torch.equal(eager[2], ugrad[invT.clamp_min(0).long()]), "graph replay != eager"
    touched = torch.unique(invT[invT >= 0]).long()
    if comb == "sum":
        sp.ugrad.zero_()
        col_bag = bags.col_bag.long()
        sp.segsum(dp_d[col_bag].contiguous())
        assert torch.equal(sp.ugrad[touched], ugrad[touched]), "pool_segsum (sum bags) != segsum on the repeated bag gradient"
    # fp64 oracle per slot: sum of dpool[bag(c), b] * w[bag(c), b] over the live (c, b) of the slot
    col_bag = np.repeat(np.arange(F), sizes)
    dp = dpool.double().numpy()
    wn = w.double().cpu().numpy()
    it = invT.cpu().numpy()
    tot = np.zeros((sp.Htot, D)); mag = np.zeros((sp.Htot, D)); cnt = np.zeros(sp.Htot)
    for c in range(C):
        live = it[c] >= 0
        term = dp[col_bag[c]][live] * wn[col_bag[c]][live][:, None]
        np.add.at(tot, it[c][live], term)
        np.add.at(mag, it[c][live], np.abs(term))
        np.add.at(cnt, it[c][live], 1)
    got = ugrad.cpu().numpy()[touched.cpu().numpy()].astype(np.float64) * 2.0 ** -40
    tk = touched.cpu().numpy()
    tol = 34 * 2.0 ** -24 * mag[tk] + cnt[tk][:, None] * 2.0 ** -40 + 1e-30
    err = np.abs(got - tot[tk])
    assert (err <= tol).all(), ("pool_segsum != fp64 per-key sum", float((err - tol).max()))
    sp.reset(); sp.step_end()


def _kernel_rank(rank, W, shared, ids_all, dp_all, comb, owner, out, errors):
    try:
        from deeprec_b200 import _native
        from deeprec_b200.parallel.emu_comm import EmuComm
        from deeprec_b200.parallel.sparse_pipeline import Bags, SparsePipeline
        import linear_group_cases as LK
        with _native.cuda_emulation():
            dev = torch.device("cpu")
            comm = EmuComm(shared, rank)
            C, B = ids_all[rank].shape
            ctx, tables, tmap = make_tables(dev, owner + rank, filter_even=False)
            sp = SparsePipeline(dev, rank, W, [c % NT for c in range(C)], NT, B, D, comm=comm)
            ctx.ensure(sp.Btot * W)
            bags = Bags(dev, [(n, comb) for n in BAG_SIZES], C)
            o = torch.zeros(B, bags.F, D, dtype=torch.bfloat16)
            w = torch.zeros(bags.F, B, dtype=torch.float32)
            sp.dedup(ids_all[rank]); sp.lookup(ctx, tmap, True); sp.pool(o, w, bags); sp.pool_segsum(dp_all[rank], w, bags)
            sp.reset(); sp.grad(ctx, tmap)
            out[rank] = (o.clone(), w.clone(), LK._owner_gsum(ctx, tables))
            sp.step_end()
            comm.host_barrier()
    except BaseException as e:                                   # noqa: BLE001 -- surfaced by the main thread
        errors.append((rank, repr(e)))
        try:
            shared.barrier.abort()
        except Exception:
            pass
        raise


def run_kernels_ranks_as_threads(W: int, comb: str, B: int = 96, owner: int = 0):
    """W emulated ranks, each with its own batch: every rank's pool == world 1 on the concatenated batch, bit for bit; every owner's gsum ==
    the fp64 per-key sum of dpool * w within the fp32 rounding of the products and of W fixed-point partials."""
    from deeprec_b200 import _native
    from deeprec_b200.parallel.emu_comm import EmuWorld
    from deeprec_b200.parallel.sparse_pipeline import Bags, SparsePipeline
    C, F = sum(BAG_SIZES), len(BAG_SIZES)
    ids_all, dp_all = [], []
    for r in range(W):
        i, d = kernel_batch(B, seed=700 + 10 * W + r)
        ids_all.append(i); dp_all.append(d)
    with _native.cuda_emulation():
        dev = torch.device("cpu")
        ctx, tables, tmap = make_tables(dev, owner + 100, filter_even=False)
        sp = SparsePipeline(dev, 0, 1, [c % NT for c in range(C)], NT, W * B, D)
        ctx.ensure(sp.Btot)
        bags = Bags(dev, [(n, comb) for n in BAG_SIZES], C)
        ref = torch.zeros(W * B, F, D, dtype=torch.bfloat16)
        ref_w = torch.zeros(F, W * B, dtype=torch.float32)
        sp.dedup(torch.cat(ids_all, 1)); sp.lookup(ctx, tmap, True); sp.pool(ref, ref_w, bags)
        sp.reset(); sp.step_end()
    shared, out, errors = EmuWorld(W), {}, []
    threads = [threading.Thread(target=_kernel_rank, args=(r, W, shared, ids_all, dp_all, comb, owner + 200, out, errors)) for r in range(W)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=800)
    assert not errors and len(out) == W, errors
    for r in range(W):
        assert torch.equal(_bits(out[r][0]), _bits(ref[r * B:(r + 1) * B])), f"rank {r}: pool differs from world 1"
        assert torch.equal(out[r][1], ref_w[:, r * B:(r + 1) * B]), r
    col_bag = np.repeat(np.arange(F), BAG_SIZES)
    want, mag, cnt = {}, {}, {}
    for r in range(W):
        dp, wr = dp_all[r].double(), out[r][1].double()
        for c in range(C):
            for b, k in enumerate(ids_all[r][c].tolist()):
                if k < 0:
                    continue
                key = (c % NT, k)
                term = dp[col_bag[c], b] * wr[col_bag[c], b]
                want[key] = want.get(key, 0.0) + term
                mag[key] = mag.get(key, 0.0) + term.abs()
                cnt[key] = cnt.get(key, 0) + 1
    seen = {}
    for r in range(W):
        for key, row in out[r][2].items():
            assert key not in seen, f"{key} claimed by ranks {seen[key]} and {r}"
            seen[key] = r
            tol = (34 + W) * 2.0 ** -24 * mag[key] + cnt[key] * 2.0 ** -40 + 1e-30
            assert bool(((row - want[key]).abs() <= tol).all()), (key, (row - want[key]).abs().max().item())
    assert set(seen) == set(want), "every key of the batch is claimed by exactly one owner"


# ---- engines ----------------------------------------------------------------------------------------------------------------------
CARDS = (300, 1000, 50)          # user, item, cat
L = 12


def taobao_like(B: int, seed: int):
    """A Taobao-shaped batch dict with variable history lengths (padding -1, some samples with no history) and a hot item."""
    g = torch.Generator().manual_seed(seed)
    hist_len = torch.randint(0, L + 1, (B,), generator=g)
    hist_len[::5] = 0
    pos = torch.arange(L)[None]
    hi = torch.randint(0, CARDS[1], (B, L), generator=g)
    hi[:, ::3] = 7
    hc = hi % CARDS[2]
    hi[pos >= hist_len[:, None]] = -1
    hc[pos >= hist_len[:, None]] = -1
    return dict(user=torch.randint(0, CARDS[0], (B,), generator=g), item=torch.randint(0, CARDS[1], (B,), generator=g),
                cat=torch.randint(0, CARDS[2], (B,), generator=g), hist_item=hi, hist_cat=hc, labels=(torch.rand(B, generator=g) < 0.3).float())


def seq_model(name: str, dev):
    import deeprec_b200 as dr
    from deeprec_b200.models.zoo import build_model
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    return build_model(name, device=dev)


def seq_engine(name: str, dev, B: int, combiner: str = "sum", model=None, **kw):
    from deeprec_b200.models.rec_engine import pooled_seq_engine
    model = model if model is not None else seq_model(name, dev)
    return pooled_seq_engine(model, B, L, combiner=combiner, table_rows=CARDS, device=None if dev.type == "cpu" else dev, **kw)


def engine_inputs(eng, b, dev):
    from deeprec_b200.models.rec_engine import din_ids, taobao_engine_batch
    if eng.labels.dim() == 2:
        ids, y, _ = taobao_engine_batch(b)
    else:
        ids, y = din_ids(b), b["labels"]
    return ids.to(dev), y.to(dev)


class _ReplicaTable(torch.nn.Module):
    """nn.Embedding with the EmbeddingVariable lookup surface the zoo models call; ``lookup_pooled`` pools with ``_combine``."""

    def __init__(self, weight: torch.Tensor, combiner: str):
        super().__init__()
        self.emb = torch.nn.Embedding.from_pretrained(weight.clone(), freeze=False)
        self.combiner = combiner

    def lookup(self, ids):
        return self.emb(ids)

    def lookup_pooled(self, ids, mask):
        from deeprec_b200.ops.embedding_ops import SparseIds, _combine
        sp = SparseIds.from_padded(torch.where(mask, ids, torch.full_like(ids, -1)))
        return _combine(self.emb(sp.values), sp, self.combiner)


def replica_of(eng, dev, combiner: str):
    """The engine's zoo model (dense net deep-copied) with nn.Embedding tables copied from the engine's default matrices."""
    m = copy.deepcopy(eng.net.inner)
    for t, name in enumerate(("user", "item", "cat")):
        dm = eng.tables[t].default_matrix
        setattr(m, name, _ReplicaTable(dm[torch.arange(CARDS[t], device=dm.device) % dm.shape[0]].float().to(dev), combiner))
    return m


def run_engine_vs_replica(name: str, dev, combiner: str = "sum", graph: bool = False, steps: int = 5, B: int = 256):
    """Adagrad on the tables and the dense net, engine against replica: per-step loss, then rows of the user / item tables."""
    eng = seq_engine(name, dev, B, combiner, learning_rate=0.05)
    rep = replica_of(eng, dev, combiner)
    opt = torch.optim.Adagrad(rep.parameters(), lr=0.05, initial_accumulator_value=0.1, eps=0.0)
    le, lr_ = [], []
    for s in range(steps):
        b = taobao_like(B, 100 + s)
        eng.load_batch(*engine_inputs(eng, b, dev))
        if graph and s == 0:
            eng.capture(warmup=1)
        else:
            eng.train_step()
        le.append(eng.loss_value())
        bd = {k: v.to(dev) for k, v in b.items()}
        loss = rep.loss(bd)
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
    for v in (p.values() if isinstance(p, dict) else [p]):
        assert v.shape == (B,) and bool(((v >= 0) & (v <= 1)).all())
    return eng
