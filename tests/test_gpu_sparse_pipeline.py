"""GPU: the unique-first sparse pipeline (csrc/cuda/sparse_pipeline.cu) at world_size 1 against plain PyTorch references:
dedup / inverse index vs torch.unique, row push vs table lookup, gradient pre-reduction + pull + Adagrad vs index_add."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk_tables(dev, dims, cards, owner):
    from deeprec_b200._native import EvConfig
    from deeprec_b200.ops.device_table import DeviceTable, get_context
    ctx = get_context(dev, dims, owner=owner)
    tables = []
    for t, card in enumerate(cards):
        c = EvConfig()
        c.dim, c.num_slots, c.has_scalars = dims, 1, 0
        c.init_capacity = card
        c.filter_type, c.filter_freq = 0, 0
        c.bloom_counter_bits = 32
        c.steps_to_live, c.l2_weight_threshold = 0, -1.0
        c.default_value_dim, c.default_value_no_permission = 4096, 0.0
        c.record_freq = c.record_version = 1
        c.storage_type = 1
        c.slot_init[0] = 0.1
        g = torch.Generator().manual_seed(7 + t)
        dm = torch.empty(4096, dims).normal_(0.0, 1.0 / math.sqrt(dims), generator=g)
        tables.append(DeviceTable(c, dm, dev, capacity=1 << 14, row_capacity=1 << 13, owner=owner))
    return ctx, tables


def test_dedup_inverse_and_counts():
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    B, col_table = 1000, [0, 1, 1, 2]                       # columns 1 and 2 share table 1 (sequence-style features)
    sp = SparsePipeline(dev, 0, 1, col_table, 3, B, 16, pad_key=-1)
    ids = torch.stack([torch.randint(0, 40, (B,)), torch.randint(0, 300, (B,)), torch.randint(100, 400, (B,)), torch.randint(0, 5, (B,))]).to(dev)
    ids[1, ::7] = -1                                        # padding
    for rep in range(2):                                    # second round: the reset must have left the scratch clean
        sp.dedup(ids)
        torch.cuda.synchronize()
        scr = sp.scr_buf.tensor(torch.int64, (sp.Htot, 2))
        inv = sp.inv[:, : len(col_table)].t().long()        # [C][B]
        pad = ids == -1
        assert (inv[pad] == -1).all() and (inv[~pad] >= 0).all()
        assert torch.equal(scr[inv[~pad], 0], ids[~pad]), "inv must point at the slot holding the key"
        n_unique = 0
        for t in range(3):
            cols = [c for c, tt in enumerate(col_table) if tt == t]
            k = torch.cat([ids[c][ids[c] != -1] for c in cols])
            u, cnt = torch.unique(k, return_counts=True)
            n_unique += u.numel()
            gs = torch.cat([inv[c][ids[c] != -1] for c in cols])
            # one slot per distinct key of the TABLE (shared across its columns), count = occurrences
            assert torch.unique(gs).numel() == u.numel()
            got = {int(a): int(b) & 0xFFFFFFFF for a, b in zip(scr[torch.unique(gs), 0].tolist(), scr[torch.unique(gs), 1].tolist())}
            assert got == {int(a): int(b) for a, b in zip(u.tolist(), cnt.tolist())}
            assert int(sp.bcnt[t, 0]) == u.numel()
        assert sp.unique_count() == n_unique
        sp.reset(); sp.step_end()
        torch.cuda.synchronize()
        assert int(sp.bcnt.sum()) == 0
        assert int((scr[:, 0] != -(1 << 63)).sum()) == 0, "reset must free every touched scratch slot"


def test_lookup_rows_and_gradient_roundtrip():
    from deeprec_b200._native import OptHyper, ptr
    from deeprec_b200.optim.optimizers import OPT_ADAGRAD
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
    import ctypes as C
    dev = torch.device("cuda", 0)
    torch.manual_seed(1)
    B, D, cards = 512, 16, [37, 5000]
    ctx, tables = _mk_tables(dev, D, cards, owner=991)
    tmap = torch.tensor([t.gid for t in tables], dtype=torch.int32, device=dev)
    sp = SparsePipeline(dev, 0, 1, [0, 1], 2, B, D)
    ctx.ensure(2 * B)
    hp = OptHyper(); hp.kind, hp.lr, hp.init_accum = OPT_ADAGRAD, 0.1, 0.1
    ctx.set_hyper(hp)
    lib = sp.lib
    ids = torch.stack([torch.randint(0, c, (B,)) for c in cards]).to(dev)
    ref = {t: {} for t in range(2)}
    for step in range(3):
        sp.dedup(ids)
        sp.lookup(ctx, tmap, True)
        torch.cuda.synchronize()
        inv = sp.inv[:, :2].t().long()
        for t in range(2):
            rows = sp.urow[inv[t]].float()
            want = tables[t].lookup(ids[t])          # read-only probe of the same table (new keys: default rows)
            assert (rows - want).abs().max().item() < 1e-2, (step, t)
        # gradients: per-sample rows g[c][b] (bf16, feature-major) -> k_sp_segsum pre-reduces them per distinct key (checked vs index_add)
        g = torch.randn(2, B, D, device=dev).bfloat16()
        sp.segsum(g)
        torch.cuda.synchronize()
        got = sp.ugrad_rows()
        want = torch.zeros_like(got).index_add_(0, inv.reshape(-1), g.float().reshape(-1, D))
        touched = torch.unique(inv.reshape(-1))
        assert (got[touched] - want[touched]).abs().max().item() < 1e-4
        g = g.float()
        sp.reset()
        sp.grad(ctx, tmap)
        rc = lib.dr_cuda_sparse_apply(ptr(ctx.structs()), ptr(ctx.ulist), ptr(ctx.nuniq), ctx.ulist.numel(), ptr(ctx.gsum), D, ptr(ctx.hp_dev), 2 * B, 1,
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0
        sp.step_end()
        torch.cuda.synchronize()
        # fp32 oracle: dedup-then-apply Adagrad per distinct key
        for t in range(2):
            u, invu = torch.unique(ids[t], return_inverse=True)
            gsum = torch.zeros(u.numel(), D, device=dev).index_add_(0, invu, g[t])
            for k, gg in zip(u.tolist(), gsum):
                w, a = ref[t].get(k, (tables[t].default_matrix[k % 4096].clone(), torch.full((D,), 0.1, device=dev)))
                a = a + gg * gg
                w = w - 0.1 * gg / a.sqrt()
                ref[t][k] = (w, a)
        ids = torch.stack([torch.randint(0, c, (B,)) for c in cards]).to(dev)
    for t in range(2):
        keys = torch.tensor(sorted(ref[t].keys()), device=dev)
        want = torch.stack([ref[t][int(k)][0] for k in keys.tolist()])
        got = tables[t].lookup(keys)
        assert (got - want).abs().max().item() < 1e-4, t
        freq = tables[t].get_freq(keys)
        assert int(freq.sum()) > 0
        assert tables[t].overflowed() == 0


def test_engine_forward_rows_match_tables():
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    torch.manual_seed(2)
    cards = [50, 1000, 7, 300] + [97] * 22
    eng = DLRMEngine(DLRMConfig(batch_size=512, cardinalities=cards))
    ids = torch.stack([torch.randint(0, c, (512,)) for c in cards]).cuda()
    eng.ids.copy_(ids)
    eng._embedding_forward(True)
    torch.cuda.synchronize()
    inv = eng.sp.inv[:, : eng.T].t().long()
    for t in (0, 1, 2, 25):
        assert (eng.sp.urow[inv[t]].float() - eng.tables[t].lookup(ids[t])).abs().max().item() < 1e-2


@pytest.mark.parametrize("batch", [512, 1000])
def test_fused_interaction_gemm_matches_unfused(batch):
    """k_dlrm_inter_gemm (gather + Gram + pack + Linear + ReLU in one tensor-core kernel) == k_dot_fwd_tc + wgmma GEMM: same Z (bitwise:
    both round the fp32 Gram to bf16), same first top activation up to accumulation order; and the training losses stay together."""
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    cards = [50, 1000, 7, 300] + [97] * 22
    engs = []
    for fuse in (True, False):
        torch.manual_seed(3)
        engs.append(DLRMEngine(DLRMConfig(batch_size=batch, cardinalities=cards, learning_rate=0.05, fuse_interaction_gemm=fuse)))
    assert engs[0].cfg.fuse_interaction_gemm and not engs[1].cfg.fuse_interaction_gemm
    torch.manual_seed(4)
    losses = [[], []]
    for step in range(3):
        dense = torch.rand(batch, 13, device="cuda") * 3
        ids = torch.stack([torch.randint(0, c, (batch,), device="cuda") for c in cards])
        labels = (torch.rand(batch, device="cuda") < 0.3).float()
        for i, e in enumerate(engs):
            e.load_batch(dense, ids, labels)
            e.train_step()
            losses[i].append(e.loss_value())
        torch.cuda.synchronize()
        if step == 0:        # identical parameters and inputs (later steps drift by bf16 rounding of the differently-ordered accumulations)
            za, zb = engs[0].Z.float(), engs[1].Z.float()
            # the bottom-MLP output feeding both paths differs by <= 1 bf16 ulp between two engines (atomic order of the BatchNorm
            # statistics); a 16-term dot product of zero-mean vectors amplifies that to a few ulps of its largest term
            assert ((za - zb).abs() - 2e-2 * zb.abs()).max().item() < 0.1, (step, (za - zb).abs().max().item())
            aa, ab = engs[0].top[0].a.float(), engs[1].top[0].a.float()
            assert (aa - ab).abs().max().item() < 5e-2 * max(1.0, ab.abs().max().item()), (step, (aa - ab).abs().max().item())
    for a, b in zip(*losses):
        assert abs(a - b) < 5e-3, losses
