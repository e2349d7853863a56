"""Cases of the linear (wide) embedding group -- k_sp_linear_fwd / k_sp_linear_bwd (csrc/cuda/sparse_pipeline.cu) and FusedRecEngine(linear=True)
-- shared by the CUDA-on-CPU emulation tests (test_cuda_emu_linear_group.py) and the H100 tests (test_gpu_linear_group.py).

Oracles:
- linear_fwd: numpy's float32 sum of float(urow[inv[b, c], 0]) over c in column order, bit for bit;
- linear_bwd: numpy's int64 sum of rint(float32(dlogit[b]) * 2^40) per key, bit for bit (elements 1..3 stay zero);
- the engine: a torch replica of Wide & Deep with nn.Embedding tables copied from the engine's default matrices (the DeepFM engine test's
  bounds: loss within 3 %, rows within 0.05), and tests/optim_ref.ftrl_ev for FTRL on the linear group.
"""
from __future__ import annotations

import copy
import threading

import numpy as np
import torch

CARDS = [50, 1000, 7, 300] + [97] * 22
NO_PERMISSION = 0.375
HOT_KEY = 12345


# ---- kernels ----------------------------------------------------------------------------------------------------------------------
def make_tables(dev, ncols: int, owner: int, filter_even: bool):
    """One dim-4 table per id column; with ``filter_even`` the even tables admit a key on its 2nd sighting (CounterFilter) and read
    ``NO_PERMISSION`` until then."""
    from deeprec_b200._native import EvConfig
    from deeprec_b200.ops.device_table import DeviceTable, get_context
    ctx = get_context(dev, 4, owner=owner)
    tables = []
    for t in range(ncols):
        c = EvConfig()
        c.dim, c.num_slots, c.has_scalars = 4, 1, 0
        c.init_capacity = 4096
        ff = 2 if filter_even and t % 2 == 0 else 0
        c.filter_type, c.filter_freq = (1, ff) if ff else (0, 0)
        c.bloom_counter_bits = 32
        c.steps_to_live, c.l2_weight_threshold = 0, -1.0
        c.default_value_dim, c.default_value_no_permission = 4096, NO_PERMISSION
        c.record_freq = c.record_version = 1
        c.storage_type = 1
        c.slot_init[0] = 0.1
        g = torch.Generator().manual_seed(7 + t)
        dm = torch.empty(4096, 4).normal_(0.0, 0.5, generator=g)
        tables.append(DeviceTable(c, dm, dev, capacity=1 << 13, row_capacity=1 << 12, owner=owner))
    tmap = torch.tensor([t.gid for t in tables], dtype=torch.int32, device=dev)
    return ctx, tables, tmap


def kernel_batch(C: int, B: int, seed: int):
    """ids [C, B]: column C-1 (or every other sample of a single column) holds one hot key, ~1/9 of the ids are padding (-1); dlogit [B]
    fp32 spanning six decades."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.stack([torch.randint(0, CARDS[c % len(CARDS)], (B,), generator=g) for c in range(C)])
    if C > 1:
        ids[C - 1] = HOT_KEY
    else:
        ids[0, ::2] = HOT_KEY
    b = torch.arange(B)
    for c in range(C):
        ids[c, (b + c) % 9 == 0] = -1
    dlogit = (torch.randn(B, generator=g) * 10.0 ** torch.randint(-6, 0, (B,), generator=g).float()).float()
    return ids, dlogit


def fwd_oracle(urow: torch.Tensor, inv: torch.Tensor, C: int) -> np.ndarray:
    """float32 sum over the columns in order of float(urow[inv[b, c], 0]); padding adds nothing."""
    u0 = urow[:, 0].float().cpu().numpy()
    inv = inv[:, :C].cpu().numpy()
    acc = np.zeros(inv.shape[0], dtype=np.float32)
    for c in range(C):
        gs = inv[:, c]
        acc = (acc + np.where(gs >= 0, u0[np.maximum(gs, 0)], np.float32(0.0))).astype(np.float32)
    return acc


def bwd_oracle(dlogit: torch.Tensor, invT: torch.Tensor, nslots: int) -> np.ndarray:
    """int64 [nslots]: sum of rint(float32(dlogit[b]) * 2^40) over every live (c, b) of each slot."""
    q = np.rint(dlogit.cpu().numpy().astype(np.float32) * np.float32(2.0 ** 40)).astype(np.int64)
    inv = invT.cpu().numpy()
    out = np.zeros(nslots, dtype=np.int64)
    for c in range(inv.shape[0]):
        live = inv[c] >= 0
        np.add.at(out, inv[c][live], q[live])
    return out


def run_kernels_world1(dev, C: int, B: int, owner: int, graph: bool = False):
    """dedup -> lookup -> linear_fwd -> linear_bwd at world 1 (optionally replayed from a CUDA graph) and the checks of both oracles."""
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
    ids, dlogit = kernel_batch(C, B, seed=40 + C)
    ctx, tables, tmap = make_tables(dev, C, owner, filter_even=True)
    sp = SparsePipeline(dev, 0, 1, list(range(C)), C, B, 4)
    ctx.ensure(sp.Btot)
    ids_d, dl_d = ids.to(dev), dlogit.to(dev)
    out = torch.full((B,), float("nan"), dtype=torch.float32, device=dev)

    def body():
        sp.dedup(ids_d)
        sp.lookup(ctx, tmap, True)
        sp.linear_fwd(out)
        sp.linear_bwd(dl_d)

    if graph:
        body()                       # eager first: fresh keys are inserted, so the captured replay below reads the same rows
        torch.cuda.synchronize()
        eager = (out.clone(), sp.ugrad[sp.invT.clamp_min(0).long()].clone())      # per (c, b): dedup's slot numbering depends on atomic order
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
    got = out.cpu().numpy()
    assert np.array_equal(got.view(np.int32), fwd_oracle(urow, inv, C).view(np.int32)), "linear_fwd != float32 sequential column sum"
    touched = torch.unique(invT[invT >= 0]).cpu()
    want = bwd_oracle(dlogit, invT, sp.Htot)
    ug = ugrad.cpu().numpy()
    assert np.array_equal(ug[touched.numpy(), 0], want[touched.numpy()]), "linear_bwd != int64 sum of the fixed-point terms"
    assert not ug[touched.numpy(), 1:].any(), "elements 1..3 of ugrad must stay zero"
    if graph:
        assert torch.equal(eager[0], out) and torch.equal(eager[1], ugrad[invT.clamp_min(0).long()]), "graph replay != eager"
    # the rows lookup pushed at dim 4 (one lane per row): the tables' rows, NO_PERMISSION for keys a CounterFilter has not admitted
    live = ids >= 0
    for c in range(C):
        k = ids[c][live[c]]
        rows = urow[inv[:, c][live[c].to(inv.device)].long()].float().cpu()
        ref = tables[c].lookup(k.to(dev)).cpu().bfloat16().float()
        assert torch.equal(rows, ref), c
    nperm = [bool((urow[inv[:, c][live[c].to(inv.device)].long(), 0].float() == NO_PERMISSION).all()) for c in range(C)]
    if C > 2:
        assert nperm[0] and not nperm[1], "filtered tables read NO_PERMISSION, unfiltered ones the default rows"
    sp.reset(); sp.step_end()
    return got


def _owner_gsum(ctx, tables):
    """{(table, key): gsum row} of the keys this owner claimed this step."""
    out = {}
    for t, tb in enumerate(tables):
        tag = tb.tag.cpu()
        keys = tb.keys.cpu()
        sel = (tag >= 0).nonzero().flatten()
        rows = ctx.gsum[tag[sel].long().to(ctx.gsum.device)].double().cpu()
        for k, r in zip(keys[sel].tolist(), rows):
            out[(t, k)] = r
    return out


def _kernel_rank(rank, W, shared, ids_all, dl_all, owner, out, errors):
    try:
        from deeprec_b200 import _native
        from deeprec_b200.parallel.emu_comm import EmuComm
        from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
        with _native.cuda_emulation():
            dev = torch.device("cpu")
            comm = EmuComm(shared, rank)
            C, B = ids_all[rank].shape
            ctx, tables, tmap = make_tables(dev, C, owner + rank, filter_even=False)
            sp = SparsePipeline(dev, rank, W, list(range(C)), C, B, 4, comm=comm)
            ctx.ensure(sp.Btot * W)
            fwd = torch.zeros(B, dtype=torch.float32)
            sp.dedup(ids_all[rank]); sp.lookup(ctx, tmap, True); sp.linear_fwd(fwd); sp.linear_bwd(dl_all[rank])
            sp.reset(); sp.grad(ctx, tmap)
            out[rank] = (fwd.clone(), _owner_gsum(ctx, tables))
            sp.step_end()
            comm.host_barrier()
    except BaseException as e:                                   # noqa: BLE001 -- surfaced by the main thread
        errors.append((rank, repr(e)))
        try:
            shared.barrier.abort()
        except Exception:
            pass
        raise


def run_kernels_ranks_as_threads(W: int, C: int = 26, B: int = 333, owner: int = 0):
    """W emulated ranks, each with its own batch: every rank's forward == world 1 on the concatenated batch, bit for bit; every owner's
    gsum == the fp64 per-key sum of dlogit within the fp32 rounding of W fixed-point partials."""
    from deeprec_b200 import _native
    from deeprec_b200.parallel.emu_comm import EmuWorld
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
    ids_all, dl_all = [], []
    for r in range(W):
        i, d = kernel_batch(C, B, seed=500 + 10 * W + r)
        ids_all.append(i); dl_all.append(d)
    with _native.cuda_emulation():
        dev = torch.device("cpu")
        ctx, tables, tmap = make_tables(dev, C, owner + 100, filter_even=False)
        sp = SparsePipeline(dev, 0, 1, list(range(C)), C, W * B, 4)
        ctx.ensure(sp.Btot)
        ref = torch.zeros(W * B, dtype=torch.float32)
        sp.dedup(torch.cat(ids_all, 1)); sp.lookup(ctx, tmap, True); sp.linear_fwd(ref)
        sp.reset(); sp.step_end()
    shared, out, errors = EmuWorld(W), {}, []
    threads = [threading.Thread(target=_kernel_rank, args=(r, W, shared, ids_all, dl_all, owner + 200, out, errors)) for r in range(W)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=800)
    assert not errors and len(out) == W, errors
    for r in range(W):
        assert torch.equal(out[r][0], ref[r * B:(r + 1) * B]), f"rank {r}: linear_fwd differs from world 1"
    # fp64 oracle per (table, key); each rank contributes one exactly-summed fixed-point partial, converted to fp32 and added in fp32
    want, mag, cnt = {}, {}, {}
    for r in range(W):
        for c in range(C):
            for k, d in zip(ids_all[r][c].tolist(), dl_all[r].double().tolist()):
                if k < 0:
                    continue
                want[(c, k)] = want.get((c, k), 0.0) + d
                mag[(c, k)] = mag.get((c, k), 0.0) + abs(d)
                cnt[(c, k)] = cnt.get((c, k), 0) + 1
    seen = {}
    for r in range(W):
        for key, row in out[r][1].items():
            assert key not in seen, f"{key} claimed by ranks {seen[key]} and {r}"
            seen[key] = r
            tol = 2 * (W + 1) * 2.0 ** -24 * mag[key] + cnt[key] * 2.0 ** -40 + 1e-30
            assert abs(row[0].item() - want[key]) <= tol, (key, row[0].item(), want[key], tol)
            assert not row[1:].any(), key
    assert set(seen) == set(want), "every key of the batch is claimed by exactly one owner"


# ---- engine -----------------------------------------------------------------------------------------------------------------------
def engine_batch(B: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    ids = torch.stack([torch.randint(0, c, (B,), generator=g) for c in CARDS])
    return ids, (torch.rand(B, generator=g) < 0.3).float(), {"dense": torch.rand(B, 13, generator=g) * 3}


def wdl_model(dev):
    import deeprec_b200 as dr
    from deeprec_b200.models.zoo import build_model
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    return build_model("wdl", device=dev)


def wdl_engine(dev, B: int, model=None, **kw):
    from deeprec_b200.models.rec_engine import criteo_engine
    model = model if model is not None else wdl_model(dev)
    return criteo_engine(model, B, table_rows=CARDS, device=None if dev.type == "cpu" else dev, **kw)


def replica_of(eng, dev):
    """A torch Wide & Deep with the engine's dense net and nn.Embedding tables copied from its default matrices."""
    net = copy.deepcopy(eng.net.inner)
    deep = torch.nn.ModuleList([torch.nn.Embedding(c, 16, device=dev) for c in CARDS])
    wide = torch.nn.ModuleList([torch.nn.Embedding(c, 4, device=dev) for c in CARDS])
    with torch.no_grad():
        for t in range(len(CARDS)):
            for emb, tb in ((deep[t], eng.tables[t]), (wide[t], eng.lin_tables[t])):
                dm = tb.default_matrix
                emb.weight.copy_(dm[torch.arange(CARDS[t], device=dm.device) % dm.shape[0]].to(dev))
    return net, deep, wide


def replica_loss(net, deep, wide, ids, y, dense):
    embs = torch.stack([deep[t](ids[t]) for t in range(len(CARDS))], 1)
    lin = torch.stack([wide[t](ids[t])[:, 0] for t in range(len(CARDS))], 1).sum(1, keepdim=True)
    return torch.nn.functional.binary_cross_entropy_with_logits(net.wide_deep_logits(dense["dense"], embs, lin).float(), y)


def run_engine_vs_replica(dev, linear_sgd: bool, graph: bool = False, steps: int = 5, B: int = 256):
    """(a) Adagrad on every group; (b) the linear group on SGD at lr 0.2 (two torch optimizers on the replica)."""
    kw = dict(learning_rate=0.05)
    if linear_sgd:
        kw.update(linear_optimizer="sgd", linear_learning_rate=0.2)
    eng = wdl_engine(dev, B, **kw)
    net, deep, wide = replica_of(eng, dev)
    ada = list(net.parameters()) + list(deep.parameters())
    if linear_sgd:
        opts = [torch.optim.Adagrad(ada, lr=0.05, initial_accumulator_value=0.1, eps=0.0), torch.optim.SGD(wide.parameters(), lr=0.2)]
    else:
        opts = [torch.optim.Adagrad(ada + list(wide.parameters()), lr=0.05, initial_accumulator_value=0.1, eps=0.0)]
    le, lr_ = [], []
    for s in range(steps):
        ids, y, dense = engine_batch(B, 100 + s)
        ids, y, dense = ids.to(dev), y.to(dev), {k: v.to(dev) for k, v in dense.items()}
        eng.load_batch(ids, y, dense)
        if graph and s == 0:
            eng.capture(warmup=1)
        else:
            eng.train_step()
        le.append(eng.loss_value())
        loss = replica_loss(net, deep, wide, ids, y, dense)
        for o in opts:
            o.zero_grad()
        loss.backward()
        for o in opts:
            o.step()
        lr_.append(loss.item())
    for a, b in zip(le, lr_):
        assert abs(a - b) < 0.03 * max(1.0, abs(b)), (le, lr_)
    keys = ids[1][:64]
    assert (eng.tables[1].lookup(keys) - deep[1].weight[keys]).abs().max().item() < 0.05
    for t in (0, 1, 3):
        k = ids[t][:64]
        assert (eng.lin_tables[t].lookup(k) - wide[t].weight[k]).abs().max().item() < 0.05, t
    assert eng.tables[0].overflowed() == 0 and eng.lin_tables[1].overflowed() == 0
    p = eng.predict()
    assert p.shape == (B,) and bool(((p >= 0) & (p <= 1)).all())
    return eng


def run_ftrl_one_step(dev, B: int = 256):
    """linear_optimizer="ftrl": after one step every touched linear row == optim_ref.ftrl_ev of its default row and its per-key gradient
    (the fp64 sum of the step's fp32 linear-logit gradients; the replica's gradient agrees with them to bf16 precision)."""
    import optim_ref as R
    eng = wdl_engine(dev, B, learning_rate=0.05, linear_optimizer="ftrl", linear_learning_rate=0.2)
    net, deep, wide = replica_of(eng, dev)
    ids, y, dense = engine_batch(B, 300)
    ids, y, dense = ids.to(dev), y.to(dev), {k: v.to(dev) for k, v in dense.items()}
    eng.load_batch(ids, y, dense)
    eng.train_step()
    dlogit = eng.lin_dlogit.double().cpu()
    # the replica's gradient of the linear logits (fp32 dense net against the engine's bf16 one)
    lin = torch.stack([wide[t](ids[t])[:, 0] for t in range(len(CARDS))], 1).sum(1, keepdim=True).detach().requires_grad_(True)
    embs = torch.stack([deep[t](ids[t]) for t in range(len(CARDS))], 1)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(net.wide_deep_logits(dense["dense"], embs, lin).float(), y)
    loss.backward()
    rg = lin.grad.flatten().double().cpu()
    assert (rg - dlogit).abs().max().item() < 0.02 * rg.abs().max().item() + 1e-6
    idc = ids.cpu()
    for t in (0, 1, 3):
        keys = torch.unique(idc[t])
        g = torch.zeros(keys.numel(), 4, dtype=torch.float64)
        mag = torch.zeros(keys.numel(), dtype=torch.float64)
        pos = torch.searchsorted(keys, idc[t])
        g[:, 0].index_add_(0, pos, dlogit)
        mag.index_add_(0, pos, dlogit.abs())
        cnt = torch.bincount(pos, minlength=keys.numel()).double()
        w0 = eng.lin_tables[t].default_matrix.cpu().double()[keys % 4096]
        ge = R.E(g, torch.zeros_like(g))
        ge.e[:, 0] = 2 * R.U * mag + cnt * 2.0 ** -40          # fixed-point terms, converted to fp32 once
        w, _, _ = R.ftrl_ev(w0, torch.full_like(w0, 0.1), torch.zeros_like(w0), ge, 0.2, 0.0, 0.0, 0.0, -0.5)
        got = eng.lin_tables[t].lookup(keys.to(dev)).double().cpu()
        bad = (got - w.v).abs() > w.tol()
        assert not bool(bad.any()), (t, int(bad.sum()), (got - w.v).abs().max().item())
    return eng
