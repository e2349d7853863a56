"""Cases for the optimizer kernels (csrc/cuda/optimizer_kernels.cu, comm_kernels.cu), written once and run on an H100
(tests/test_gpu_optimizer_edges.py, device "cuda") and on the CUDA-on-CPU emulation (tests/test_cuda_emu_optimizer_edges.py, device "cpu"
inside ``_native.cuda_emulation()``).  Every result is compared with the float64 oracle of tests/optim_ref.py under its per-element bound;
multi-step cases restart the oracle from the kernel's fp32 state after each step."""
from __future__ import annotations

import ctypes as C
import itertools

import torch

import optim_ref as R
from deeprec_b200 import _native
from deeprec_b200._native import EvConfig, OptHyper, ptr, stream_ptr

# name -> (DrOptKind, hyper-parameter overrides)
RULES = {
    "sgd": (R.SGD, {}),
    "adagrad": (R.ADAGRAD, {}),
    "adagraddecay": (R.ADAGRAD_DECAY, {}),
    "adam": (R.ADAM, {"lr": 0.01}),
    "adamasync": (R.ADAM_ASYNC, {"lr": 0.01}),
    "adamw": (R.ADAMW, {"lr": 0.01, "weight_decay": 0.01}),
    "adamasync_rmsprop": (R.ADAM_ASYNC_RMSPROP, {"lr": 0.01, "apply_sparse_rmsprop": 1}),
    "ftrl": (R.FTRL, {"l1": 0.05, "l2": 0.02, "l2_shrinkage": 0.1, "lr_power": -0.5}),
    "ftrl_powf": (R.FTRL, {"l1": 0.05, "l2": 0.02, "l2_shrinkage": 0.1, "lr_power": -0.25}),
}
SPARSE_DIMS = [4, 8, 12, 16, 20, 64, 128, 256, 512]
_OWNER = itertools.count(0x5100)


def _lib():
    return _native.cuda()


def _sync():
    _native.stream_sync()


def make_hyper(rule: str, **over) -> OptHyper:
    kind, hov = RULES[rule]
    hp = OptHyper()
    vals = dict(kind=kind, lr=0.05, beta1=0.9, beta2=0.999, epsilon=1e-8, beta1_power=0.9, beta2_power=0.999, weight_decay=0.0, l1=0.0, l2=0.0,
                l2_shrinkage=0.0, lr_power=-0.5, decay_rate=0.5, decay_baseline=0.1, init_accum=0.1, decay_step=2, global_step=1)
    vals.update(hov)
    vals.update(over)
    for k, v in vals.items():
        setattr(hp, k, v)
    return hp


def hyper_dict(hp: OptHyper) -> dict:
    return {name: getattr(hp, name) for name, _ in OptHyper._fields_}


def read_hyper(hp_dev: torch.Tensor) -> OptHyper:
    _sync()
    return OptHyper.from_buffer_copy(bytes(hp_dev.cpu().numpy().tobytes()))


def write_hyper(hp_dev: torch.Tensor, hp: OptHyper) -> None:
    hp_dev.copy_(torch.frombuffer(bytearray(bytes(hp)), dtype=torch.uint8))


def slot_init(kind: int):
    return [0.1 if kind in (R.ADAGRAD, R.ADAGRAD_DECAY, R.FTRL) else 0.0, 0.0, 0.0, 0.0]


def check(name: str, got: torch.Tensor, ref: R.E) -> None:
    got = got.detach().double().cpu()
    err = (got - ref.v).abs()
    tol = ref.tol()
    bad = ~(err <= tol)
    if bad.any():
        i = int(bad.view(-1).nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements beyond the bound; first at flat index {i}: "
                             f"got {got.view(-1)[i].item()!r}, oracle {ref.v.view(-1)[i].item()!r}, bound {tol.view(-1)[i].item():.3g}")


# ---------------------------------------------------------------------------------------------------------------------------------------
# device tables

def make_table(dev, dim: int, kind: int, filter_freq: int = 0, capacity: int | None = None, seed: int = 0):
    from deeprec_b200.ops.device_table import DeviceTable
    c = EvConfig()
    c.dim, c.num_slots, c.has_scalars = dim, R.NUM_SLOTS[kind], int(kind == R.ADAGRAD_DECAY)
    c.init_capacity = 256
    c.filter_type, c.filter_freq = (1, filter_freq) if filter_freq > 0 else (0, 0)
    c.bloom_counter_bits = 32
    c.l2_weight_threshold = -1.0
    c.default_value_dim = 97
    c.record_freq = c.record_version = 1
    c.storage_type = 1
    for i, v in enumerate(slot_init(kind)):
        c.slot_init[i] = v
    g = torch.Generator().manual_seed(1000 + seed)
    dm = torch.randn(97, dim, generator=g) * 0.3
    return DeviceTable(c, dm, torch.device(dev), capacity=capacity, row_capacity=1024, owner=next(_OWNER))


def table_pos(tb, keys: torch.Tensor) -> torch.Tensor:
    """Slot positions of ``keys`` (-1 when absent) without touching the table."""
    k = keys.to(tb.device, torch.int64).contiguous()
    pos = torch.empty(k.numel(), dtype=torch.int32, device=tb.device)
    n = k.numel()
    assert _lib().dr_cuda_table_lookup(ptr(tb.ctx.structs()), ptr(tb._map), 1, ptr(k), None, n, n, 0, None, ptr(pos), None, None, 0,
                                       stream_ptr()) == 0
    _sync()
    return pos.cpu().long()


def row_state(tb, keys: torch.Tensor):
    """(row index or -1, [n, stride] fp32 row: emb | slots | scalars) of every key; absent / un-admitted keys read as a fresh row would
    start: default_matrix[key % default_value_dim], the slot_init values, zero scalars."""
    pos = table_pos(tb, keys)
    row_of = tb.row_of.cpu().long()
    r = torch.where(pos >= 0, row_of[pos.clamp_min(0)], torch.full_like(pos, -1))
    rows = tb.rows.cpu()[r.clamp_min(0)].clone()
    fresh = torch.zeros(keys.numel(), tb.stride)
    dm = tb.default_matrix.cpu()
    fresh[:, :tb.dim] = dm[keys.cpu() % dm.shape[0]]
    for s in range(tb.num_slots):
        fresh[:, (1 + s) * tb.dim:(2 + s) * tb.dim] = float(tb.cfg.slot_init[s])
    rows[r < 0] = fresh[r < 0]
    return r, rows


def _split(rows: torch.Tensor, dim: int, ns: int):
    w = rows[:, :dim].double()
    s0 = rows[:, dim:2 * dim].double() if ns > 0 else torch.zeros_like(w)
    s1 = rows[:, 2 * dim:3 * dim].double() if ns > 1 else torch.zeros_like(w)
    sc = rows[:, (1 + ns) * dim:(1 + ns) * dim + 4].double()
    return w, s0, s1, sc


def _perturb_slots(tb, rows_idx: torch.Tensor, kind: int, gen: torch.Generator) -> None:
    """Give existing rows non-trivial optimizer state (positive accumulators / second moments, signed first moments / linear)."""
    if rows_idx.numel() == 0 or tb.num_slots == 0:
        return
    D, n = tb.dim, rows_idx.numel()
    rows = tb.rows.cpu()
    pos_slot = torch.rand(n, D, generator=gen) * 2 + 0.05
    signed = torch.randn(n, D, generator=gen) * 0.3
    if kind in (R.ADAGRAD, R.ADAGRAD_DECAY):
        rows[rows_idx, D:2 * D] = pos_slot
    elif kind == R.FTRL:
        rows[rows_idx, D:2 * D] = pos_slot
        rows[rows_idx, 2 * D:3 * D] = signed
    else:   # Adam family: m signed, v positive
        rows[rows_idx, D:2 * D] = signed * 0.1
        rows[rows_idx, 2 * D:3 * D] = pos_slot * 0.01
    tb.rows.copy_(rows.to(tb.rows.device))


# ---------------------------------------------------------------------------------------------------------------------------------------
# dr_cuda_sparse_apply (k_apply)

def sparse_apply_case(dev, rule: str, dim: int, steps: int = 5) -> None:
    """Five steps of ``rule`` on one table of width ``dim`` behind a CounterFilter(2).  Each step touches keys seen before (their slots are
    first set to non-trivial values), keys that appear twice (admitted at first sight: fresh rows from default_matrix / slot_init) and keys
    seen once (not admitted until a second sighting).  dr_cuda_advance_hyper runs between steps; AdagradDecay with decay_step 2 crosses
    two decay boundaries."""
    kind = RULES[rule][0]
    lib = _lib()
    tb = make_table(dev, dim, kind, filter_freq=2, seed=dim)
    ctx = tb.ctx
    ns, D = tb.num_slots, dim
    hp = make_hyper(rule)
    write_hyper(ctx.hp_dev, hp)
    gen = torch.Generator().manual_seed(7 * dim + kind)
    seen = torch.empty(0, dtype=torch.int64)
    for step in range(steps):
        hp = read_hyper(ctx.hp_dev)
        gs = int(hp.global_step)
        old = seen[torch.randperm(seen.numel(), generator=gen)[:12]]
        new = torch.arange(1000 * (step + 1), 1000 * (step + 1) + 16) * 7 + dim
        twice, once = new[:10], new[10:]
        uniq = torch.cat([old, twice, once])
        r_before, _ = row_state(tb, uniq)
        _perturb_slots(tb, r_before[r_before >= 0], kind, gen)
        r_before, before = row_state(tb, uniq)
        ids = torch.cat([old, twice, twice, once])
        _, pos = tb.lookup_train(ids.to(tb.device), gs)
        _sync()
        pos_u = pos.cpu().long()[torch.cat([torch.arange(old.numel() + twice.numel()), torch.arange(ids.numel() - once.numel(), ids.numel())])]
        tags = tb.tag.cpu().long()[pos_u]
        assert (tags >= 0).all()
        scale = 10.0 ** (torch.rand(uniq.numel(), 1, generator=gen) * 3 - 3)      # per-key magnitudes 1e-3 .. 1: FTRL rows on both sides of l1
        g = torch.randn(uniq.numel(), D, generator=gen) * scale
        gsum = ctx.gsum.cpu()
        gsum[tags] = g
        ctx.gsum.copy_(gsum.to(ctx.gsum.device))
        freq_admitted = torch.cat([r_before[:old.numel()] >= 0, torch.ones(twice.numel(), dtype=torch.bool),
                                   torch.zeros(once.numel(), dtype=torch.bool)])
        # a key seen once before and once now reaches the threshold this step
        freq_admitted |= tb.freq.cpu().long()[pos_u] >= 2
        assert lib.dr_cuda_sparse_apply(ptr(ctx.structs()), ptr(ctx.ulist), ptr(ctx.nuniq), ctx.ulist.numel(), ptr(ctx.gsum), D, ptr(ctx.hp_dev),
                                        uniq.numel(), 1, stream_ptr()) == 0
        ctx.pending, ctx.claimed_upper = False, 0
        _sync()
        # bookkeeping of every touched key, admitted or not
        slots_pos = pos_u.to(tb.device)
        assert (tb.version[slots_pos].cpu() == gs).all(), "version != global_step"
        assert (tb.tag[slots_pos].cpu() == -1).all(), "per-step claim not released"
        assert not ctx.gsum.any(), "gsum not re-zeroed"
        assert int(ctx.nuniq.cpu()) == 0
        r_after, after = row_state(tb, uniq)
        assert torch.equal(r_after >= 0, freq_admitted), (r_after, freq_admitted)
        a = freq_admitted
        w0, s00, s10, sc0 = _split(before[a], D, ns)
        w1, s01, s11, sc1 = _split(after[a], D, ns)
        if kind == R.ADAGRAD_DECAY:
            power = sc0[:, 0]
            due = torch.tensor([R.adagrad_decay_due(gs, int(hp.decay_step), float(p)) for p in power], dtype=torch.bool)
            assert torch.equal(sc1[:, 0], power + due.double()), "AdagradDecay power"
            rw, rs0 = [], []
            for d in (False, True):
                m = due == d
                ww, aa = R.adagrad_decay(w0[m], s00[m], g[a][m].double(), hp.lr, d, hp.decay_rate, hp.decay_baseline)
                rw.append((m, ww)); rs0.append((m, aa))
            for nm, got, parts in (("w", w1, rw), ("s0", s01, rs0)):
                for m, ref in parts:
                    check(f"{rule} dim {D} step {step} {nm}", got[m], ref)
        else:
            ref = R.apply(kind, hyper_dict(hp), w0, s00, s10, g[a].double(), dense=False)
            for nm, got, rf, used in (("w", w1, ref[0], True), ("s0", s01, ref[1], ns > 0), ("s1", s11, ref[2], ns > 1)):
                if used:
                    check(f"{rule} dim {D} step {step} {nm}", got, rf)
        seen = torch.unique(torch.cat([seen, uniq]))
        assert lib.dr_cuda_advance_hyper(ptr(ctx.hp_dev), stream_ptr()) == 0
    assert tb.overflowed() == 0


def sparse_overflow_case(dev) -> None:
    """More distinct keys than the claim list holds: the lookup flags the overflow (counter 4 = 2), claims nothing past ulist_cap, and the
    apply updates only the listed keys; the list and gsum past the cap keep their sentinel values."""
    lib = _lib()
    D, cap, n = 16, 8, 13
    tb = make_table(dev, D, R.ADAGRAD)
    ctx = tb.ctx
    write_hyper(ctx.hp_dev, make_hyper("adagrad"))
    keys = (torch.arange(n) * 5 + 3).to(tb.device)
    tb.reserve(n)
    ulist = torch.full((cap + 4,), -7, dtype=torch.int64, device=tb.device)
    gsum = torch.zeros(cap + 4, D, device=tb.device)
    gsum[:cap] = 0.25
    gsum[cap:] = 99.0
    nuniq = torch.zeros(1, dtype=torch.int32, device=tb.device)
    pos = torch.empty(n, dtype=torch.int32, device=tb.device)
    step = torch.ones(1, dtype=torch.int64, device=tb.device)
    assert lib.dr_cuda_table_lookup(ptr(ctx.structs()), ptr(tb._map), 1, ptr(keys), None, n, n, 1, ptr(step), ptr(pos), ptr(ulist), ptr(nuniq), cap,
                                    stream_ptr()) == 0
    _sync()
    assert int(nuniq.cpu()) >= n and int(tb.counters.cpu()[4]) == 2
    assert (ulist.cpu()[cap:] == -7).all()
    assert lib.dr_cuda_sparse_apply(ptr(ctx.structs()), ptr(ulist), ptr(nuniq), cap, ptr(gsum), D, ptr(ctx.hp_dev), n, 1, stream_ptr()) == 0
    _sync()
    assert int(nuniq.cpu()) == 0
    assert not gsum[:cap].any() and (gsum[cap:] == 99.0).all()
    r, _ = row_state(tb, keys.cpu())
    assert int((r >= 0).sum()) == cap and (tb.tag[pos.long()].cpu() == -1).all()


def advance_hyper_case(dev) -> None:
    """k_advance_hyper: global_step + 1 and, for the Adam family, the fp32 running products beta^t, bit for bit."""
    import numpy as np
    lib = _lib()
    for rule in ("adam", "adamw", "adamasync", "adamasync_rmsprop", "adagrad"):
        hp = make_hyper(rule, beta1=0.87, beta2=0.9993, beta1_power=0.87, beta2_power=0.9993, global_step=5)
        hp_dev = torch.zeros(C.sizeof(OptHyper), dtype=torch.uint8, device=dev)
        write_hyper(hp_dev, hp)
        p1, p2 = np.float32(0.87), np.float32(0.9993)
        for t in range(1, 40):
            assert lib.dr_cuda_advance_hyper(ptr(hp_dev), stream_ptr()) == 0
            if rule != "adagrad":
                p1, p2 = np.float32(p1 * np.float32(0.87)), np.float32(p2 * np.float32(0.9993))
        got = read_hyper(hp_dev)
        assert got.global_step == 5 + 39
        assert np.float32(got.beta1_power) == p1 and np.float32(got.beta2_power) == p2, (rule, got.beta1_power, p1, got.beta2_power, p2)


def adagrad_decay_dense_power_case(dev) -> None:
    """The dense AdagradDecay decay power lives next to the hyper-parameters on the device: k_advance_hyper advances it by one whenever
    global_step / decay_step (integer division) exceeded it during the step, as ApplyAdagradDecayOp does with accum_decay_power."""
    lib = _lib()
    hp = make_hyper("adagraddecay", decay_step=3, global_step=0)
    hp_dev = torch.zeros(C.sizeof(OptHyper), dtype=torch.uint8, device=dev)
    write_hyper(hp_dev, hp)
    power = 0
    for gs in range(0, 14):
        got = read_hyper(hp_dev)
        assert got.global_step == gs and got.dense_decay_power == power, (gs, got.dense_decay_power, power)
        if R.adagrad_decay_due(gs, 3, power):
            power += 1
        assert lib.dr_cuda_advance_hyper(ptr(hp_dev), stream_ptr()) == 0


# ---------------------------------------------------------------------------------------------------------------------------------------
# dr_cuda_sparse_accumulate (k_accumulate + the combining cache of table.cuh)

ACCUMULATE_VARIANTS = ["uniform_f32", "offsets_bf16_scale", "row_ids", "flat_in", "hot_keys", "cache_conflicts", "dim512", "big_table"]


def sparse_accumulate_case(dev, variant: str) -> None:
    """gsum[tag[pos_i]] += scale_i * grad(b_i, t_i) over two tables, against a float64 index_add.  Items with pos = -1 are skipped.
    The fp32 sum order is not fixed (combining cache, flushes, red.global.add), so each element of a row that received n items is
    bounded by (n + 1) u sum |scale_i grad_i|."""
    lib = _lib()
    gen = torch.Generator().manual_seed(hash(variant) % 1000)
    D = {"dim512": 512, "cache_conflicts": 64}.get(variant, 16)
    cap = 1 << 18 if variant == "big_table" else None
    tabs = [make_table(dev, D, R.ADAGRAD, capacity=cap, seed=i) for i in range(2)]
    for tb in tabs[1:]:     # the second table joins the first one's step context
        tb.ctx.unregister(tb)
        tb.ctx = tabs[0].ctx
        tb.gid = tb.ctx.register(tb)
        tb._map = torch.tensor([tb.gid], dtype=torch.int32, device=tb.device)
    ctx = tabs[0].ctx
    T = 2
    nkeys = {"hot_keys": 3, "cache_conflicts": 700, "dim512": 40}.get(variant, 50)
    reps = {"hot_keys": 3000, "cache_conflicts": 6, "dim512": 20}.get(variant, 4)
    B = nkeys * reps
    # ids[t, b]: table t, sample b
    base = torch.randint(0, 1 << 30, (T, nkeys), generator=gen)
    ids = base[:, torch.randint(0, nkeys, (B,), generator=gen)]
    ids[:, :nkeys] = base
    pos = torch.empty(T, B, dtype=torch.int64)
    for t, tb in enumerate(tabs):
        _, p = tb.lookup_train(ids[t].to(tb.device), 1)
        _sync()
        pos[t] = p.cpu().long()
    pos[:, ::37] = -1                                        # items the accumulate must skip
    tag = torch.stack([tabs[t].tag.cpu().long()[pos[t].clamp_min(0)] for t in range(T)])
    bf16 = variant == "offsets_bf16_scale"
    flat = variant == "flat_in"
    use_rows = variant == "row_ids"
    use_offsets = variant in ("offsets_bf16_scale", "row_ids")
    # items: table 0 takes n0 of its samples, table 1 all of its samples
    n0 = B - 5 if use_offsets else B
    item_t = torch.cat([torch.zeros(n0, dtype=torch.int64), torch.ones(B, dtype=torch.int64)])
    item_b = torch.cat([torch.arange(n0), torch.arange(B)])
    if use_rows:
        item_b = torch.cat([torch.randperm(B, generator=gen)[:n0], torch.randperm(B, generator=gen)])
    n = item_t.numel()
    item_pos = pos[item_t, item_b]
    item_tag = tag[item_t, item_b]
    grad = torch.randn(B, T, D, generator=gen) * 10.0 ** (torch.rand(B, T, 1, generator=gen) * 4 - 2)
    if bf16:
        grad = grad.bfloat16()
    scale = (torch.rand(n, generator=gen) + 0.5) if variant == "offsets_bf16_scale" else None
    if flat:
        g_in = grad[item_b, item_t].contiguous()
        stride_b = stride_t = 0
    else:
        g_in = grad
        stride_b, stride_t = T * D, D
    offsets = torch.tensor([0, n0], dtype=torch.int64) if use_offsets else None
    row_ids = item_b.to(torch.int32) if use_rows else None
    tmap = torch.tensor([tb.gid for tb in tabs], dtype=torch.int32)
    todev = lambda x: None if x is None else x.to(tabs[0].device).contiguous()
    g_dev, offs_dev, rows_dev, sc_dev = todev(g_in), todev(offsets), todev(row_ids), todev(scale)
    pos_dev, tmap_dev = todev(item_pos.to(torch.int32)), todev(tmap)
    ctx.gsum.zero_()
    rc = lib.dr_cuda_sparse_accumulate(ptr(ctx.structs()), ptr(tmap_dev), T, D, ptr(pos_dev), ptr(offs_dev), n0 if not use_offsets else 0, n,
                                       ptr(g_dev), int(bf16), stride_b, stride_t, int(flat), ptr(rows_dev), ptr(sc_dev), ptr(ctx.gsum), stream_ptr())
    assert rc == 0
    _sync()
    keep = item_pos >= 0
    contrib = grad[item_b, item_t].double() * (scale.double()[:, None] if scale is not None else 1.0)
    nu = int(ctx.nuniq.cpu())
    ref = torch.zeros(nu, D, dtype=torch.float64).index_add_(0, item_tag[keep], contrib[keep])
    mag = torch.zeros(nu, D, dtype=torch.float64).index_add_(0, item_tag[keep], contrib[keep].abs())
    cnt = torch.zeros(nu, dtype=torch.float64).index_add_(0, item_tag[keep], torch.ones(int(keep.sum()), dtype=torch.float64))
    got = ctx.gsum.cpu()
    check(f"accumulate {variant}", got[:nu], R.E(ref, 0.5 * (cnt[:, None] + 1) * R.U * mag))
    assert not got[nu:].any(), "accumulate wrote past the claimed rows"
    if variant == "hot_keys":
        assert cnt.max() > 1000


# ---------------------------------------------------------------------------------------------------------------------------------------
# dr_cuda_dense_apply (k_dense_apply)

DENSE_SIZES = ["1", "255", "257", "grid_stride"]


def _dense_n(size: str, dev) -> int:
    if size != "grid_stride":
        return int(size)
    if str(dev).startswith("cuda"):
        return 3 * torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256 + 13    # > 3 sweeps of the capped grid
    return 3 * 2 * 16 * 256 + 13                                                                  # the emulation's 2 "SMs"


def dense_apply_case(dev, rule: str, size: str, decay_due: bool = False) -> None:
    """One dense update of n elements with grad_scale 0.5 and the bf16 shadow: every element within the oracle bound, the shadow the
    round-to-nearest-even bf16 of the fp32 result bit for bit.  SGD passes null slots.  AdagradDecay runs with the dense decay due or not."""
    lib = _lib()
    kind = RULES[rule][0]
    n = _dense_n(size, dev)
    gen = torch.Generator().manual_seed(n + kind)
    ns = R.NUM_SLOTS[kind]
    w = torch.randn(n, generator=gen) * 0.5
    grad = torch.randn(n, generator=gen) * 10.0 ** (torch.rand(n, generator=gen) * 3 - 2.5)
    s0 = (torch.rand(n, generator=gen) * 2 + 0.05) if kind in (R.ADAGRAD, R.ADAGRAD_DECAY, R.FTRL) else torch.randn(n, generator=gen) * 0.05
    s1 = torch.randn(n, generator=gen) * 0.3 if kind == R.FTRL else torch.rand(n, generator=gen) * 0.02
    hp = make_hyper(rule, global_step=4 if decay_due else 3, decay_step=2)
    if kind == R.ADAGRAD_DECAY:
        hp.dense_decay_power = 1
    hp_dev = torch.zeros(C.sizeof(OptHyper), dtype=torch.uint8, device=dev)
    write_hyper(hp_dev, hp)
    d = lambda x: x.clone().to(dev)
    wd, gd = d(w), d(grad)
    s0d = d(s0) if ns > 0 else None
    s1d = d(s1) if ns > 1 else None
    shadow = torch.zeros(n, dtype=torch.bfloat16, device=dev)
    assert lib.dr_cuda_dense_apply(ptr(wd), ptr(gd), ptr(s0d), ptr(s1d), n, ptr(hp_dev), 0.5, ptr(shadow), stream_ptr()) == 0
    _sync()
    g = R.E(grad.double()) * 0.5
    due = kind == R.ADAGRAD_DECAY and R.adagrad_decay_due(int(hp.global_step), int(hp.decay_step), hp.dense_decay_power)
    assert due == (decay_due and kind == R.ADAGRAD_DECAY)
    ref = R.apply(kind, hyper_dict(hp), w.double(), s0.double(), s1.double(), g, decay_now=due, dense=True)
    check(f"dense {rule} n={n} w", wd, ref[0])
    if ns > 0:
        check(f"dense {rule} n={n} s0", s0d, ref[1])
    if ns > 1:
        check(f"dense {rule} n={n} s1", s1d, ref[2])
    assert torch.equal(shadow.cpu().view(torch.int16), wd.cpu().bfloat16().view(torch.int16)), "bf16 shadow is not RNE(fp32 result)"


# ---------------------------------------------------------------------------------------------------------------------------------------
# DLRMEngine: the update inside the real step

ENGINE_OPTIMIZERS = ["gradientdescent", "adagrad", "adagraddecay", "adam", "adamasync", "adamw", "ftrl"]
ENGINE_CARDS = [50, 1000, 7, 300] + [97] * 22


def engine_batch(B, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, 13, generator=g) * 3, torch.stack([torch.randint(0, c, (B,), generator=g) for c in ENGINE_CARDS]),
            (torch.rand(B, generator=g) < 0.3).float())


def engine_hyper_overrides(eng, opt: str) -> None:
    """Exercise the terms the default engine hyper-parameters leave at zero: FTRL's l1 / l2 / l2_shrinkage, and an AdagradDecay decay due
    at the next step (decay_step 1 at global_step >= 1: the dense accumulators and every row decay)."""
    hp = read_hyper(eng.hp_dev)
    if opt == "ftrl":
        hp.l1, hp.l2, hp.l2_shrinkage = 0.01, 0.01, 0.05
    if opt == "adagraddecay":
        hp.decay_step, hp.decay_rate = 1, 0.5
    write_hyper(eng.hp_dev, hp)
    _sync()


def engine_dense_check(name: str, kind: int, hp: OptHyper, before, after, grad: torch.Tensor) -> None:
    p0, a0, b0 = before
    p1, a1, b1 = after
    due = kind == R.ADAGRAD_DECAY and R.adagrad_decay_due(int(hp.global_step), int(hp.decay_step), hp.dense_decay_power)
    z = torch.zeros_like(p0, dtype=torch.float64)
    ref = R.apply(kind, hyper_dict(hp), p0.double(), a0.double() if a0 is not None else z, b0.double() if b0 is not None else z,
                  grad.double(), decay_now=due, dense=True)
    check(f"{name} dense params", p1, ref[0])
    if a1 is not None:
        check(f"{name} dense s0", a1, ref[1])
    if b1 is not None:
        check(f"{name} dense s1", b1, ref[2])


def engine_update_case(opt: str) -> None:
    """One DLRMEngine step at batch 256 (after one warm-up step): the dense parameters and slots equal the oracle applied to the snapshot
    and the step's gradient (eng.grads); every touched embedding row and its slots equal the oracle applied to the row before the step and
    the key's gradient rebuilt in float64 from demb and the ids."""
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    torch.manual_seed(0)
    cfg = DLRMConfig(batch_size=256, cardinalities=ENGINE_CARDS, optimizer=opt, learning_rate=0.05)
    eng = DLRMEngine(cfg)
    eng.load_batch(*engine_batch(256, 1))
    eng.train_step()
    engine_hyper_overrides(eng, opt)
    hp = read_hyper(eng.hp_dev)
    kind = eng.kind
    snap = lambda: tuple(None if x is None else x.detach().cpu().clone() for x in (eng.params, eng.s0, eng.s1))
    before = snap()
    dense, ids, labels = engine_batch(256, 2)
    tabs = (0, 1, 3, 7)
    rows_before = {}
    for t in tabs:
        keys = torch.unique(ids[t])
        rows_before[t] = (keys,) + row_state(eng.tables[t], keys)
    eng.load_batch(dense.to(eng.dev), ids.to(eng.dev), labels.to(eng.dev))
    eng.train_step()
    _sync()
    engine_dense_check(opt, kind, hp, before, snap(), eng.grads.cpu())
    demb = eng.demb.cpu().double()                           # [T, B, D] per-sample gradient rows of this step
    for t in tabs:
        keys, r0, rows0 = rows_before[t]
        tb = eng.tables[t]
        inv = torch.searchsorted(keys, ids[t])
        g = torch.zeros(keys.numel(), eng.D, dtype=torch.float64).index_add_(0, inv, demb[t])
        mag = torch.zeros_like(g).index_add_(0, inv, demb[t].abs())
        cnt = torch.zeros(keys.numel(), dtype=torch.float64).index_add_(0, inv, torch.ones(ids.shape[1], dtype=torch.float64))
        ge = R.E(g, (cnt[:, None] + 1) * R.U * mag + cnt[:, None] * 2.0 ** -32)
        r1, rows1 = row_state(tb, keys)
        assert (r1 >= 0).all()
        w0, s00, s10, sc0 = _split(rows0, eng.D, tb.num_slots)
        w1, s01, s11, sc1 = _split(rows1, eng.D, tb.num_slots)
        if kind == R.ADAGRAD_DECAY:
            due = torch.tensor([R.adagrad_decay_due(int(hp.global_step), int(hp.decay_step), float(p)) for p in sc0[:, 0]])
            assert due.all() and torch.equal(sc1[:, 0], sc0[:, 0] + 1)
            ref = R.adagrad_decay(w0, s00, ge, hp.lr, True, hp.decay_rate, hp.decay_baseline) + (None,)
        else:
            ref = R.apply(kind, hyper_dict(hp), w0, s00, s10, ge, dense=False)
        check(f"{opt} table {t} rows", w1, ref[0])
        if tb.num_slots > 0:
            check(f"{opt} table {t} slot 0", s01, ref[1])
        if tb.num_slots > 1:
            check(f"{opt} table {t} slot 1", s11, ref[2])


# ---------------------------------------------------------------------------------------------------------------------------------------
# fused dense all-reduce + update (dr_comm_allreduce_apply, k_allreduce_apply), ranks as threads on the emulation

def _run_ranks(W, fn):
    import threading
    from deeprec_b200.parallel.emu_comm import EmuWorld
    with _native.cuda_emulation():
        pass
    shared, out, errors = EmuWorld(W), {}, []

    def body(r):
        try:
            with _native.cuda_emulation():
                out[r] = fn(r, shared)
        except BaseException as e:                            # noqa: BLE001
            errors.append((r, repr(e)))
            shared.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,)) for r in range(W)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=1200)
    assert not errors and len(out) == W, errors
    return out


def fused_allreduce_case(rule: str, W: int) -> None:
    """Every rank pulls all ranks' gradients in rank order and applies the dense rule in the same pass: the reduced gradient must equal the
    fp32 sum taken in rank order bit for bit, and every rank's parameters and slots the oracle applied to that sum."""
    from deeprec_b200.parallel.emu_comm import EmuComm
    from deeprec_b200.parallel.sparse_pipeline import Peers
    kind = RULES[rule][0]
    n = 4 * 97
    gen = torch.Generator().manual_seed(W * 10 + kind)
    grads = [torch.randn(n, generator=gen) * 10.0 ** (torch.rand(n, generator=gen) * 3 - 2.5) for _ in range(W)]
    w = torch.randn(n, generator=gen) * 0.5
    s0 = (torch.rand(n, generator=gen) * 2 + 0.05) if kind in (R.ADAGRAD, R.ADAGRAD_DECAY, R.FTRL) else torch.randn(n, generator=gen) * 0.05
    s1 = torch.randn(n, generator=gen) * 0.3 if kind == R.FTRL else torch.rand(n, generator=gen) * 0.02
    hp = make_hyper(rule, global_step=4, decay_step=2)
    ns = R.NUM_SLOTS[kind]

    def rank(r, shared):
        lib = _lib()
        fn = lib.dr_comm_allreduce_apply
        fn.argtypes, fn.restype = [C.POINTER(Peers), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p], C.c_int
        comm = EmuComm(shared, r)
        g = comm.alloc_grads(n)
        g.copy_(grads[r])
        wr, s0r, s1r = w.clone(), s0.clone() if ns > 0 else None, s1.clone() if ns > 1 else None
        hp_dev = torch.zeros(C.sizeof(OptHyper), dtype=torch.uint8)
        write_hyper(hp_dev, hp)
        reduced = torch.zeros(n)
        comm.host_barrier()                                   # every rank's gradient is in place
        rc = fn(comm.grads_buf.peers_ref(), W, ptr(wr), ptr(s0r), ptr(s1r), n, ptr(hp_dev), ptr(reduced), None)
        comm.host_barrier()                                   # nobody frees its gradient while a peer still reads it
        return rc, wr, s0r, s1r, reduced

    out = _run_ranks(W, rank)
    gsum = torch.zeros(n)
    for r in range(W):
        gsum = gsum + grads[r]
    due = kind == R.ADAGRAD_DECAY and R.adagrad_decay_due(int(hp.global_step), int(hp.decay_step), hp.dense_decay_power)
    ref = R.apply(kind, hyper_dict(hp), w.double(), s0.double(), s1.double(), gsum.double(), decay_now=due, dense=True)
    for r in range(W):
        rc, wr, s0r, s1r, reduced = out[r]
        assert rc == 0
        assert torch.equal(reduced, gsum), "reduced gradient is not the rank-order fp32 sum"
        check(f"fused {rule} W={W} rank {r} w", wr, ref[0])
        if ns > 0:
            check(f"fused {rule} W={W} rank {r} s0", s0r, ref[1])
        if ns > 1:
            check(f"fused {rule} W={W} rank {r} s1", s1r, ref[2])
        assert torch.equal(wr, out[0][1]), "replicas differ"


def engine_world2_case(opt: str) -> None:
    """DLRMEngine at world 2 with the ranks as threads: after one step the dense parameters and slots of both replicas equal the oracle
    applied to the snapshot and the rank-order fp32 sum of the two ranks' gradients (the fused all-reduce + update)."""
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    from deeprec_b200.parallel.emu_comm import EmuComm
    B = 128

    def rank(r, shared):
        with shared.lock:
            torch.manual_seed(0)
            cfg = DLRMConfig(batch_size=B, cardinalities=ENGINE_CARDS, optimizer=opt, learning_rate=0.05)
        eng = DLRMEngine(cfg, None, r, 2, EmuComm(shared, r))
        eng.load_batch(*engine_batch(B, 100 + r))
        eng.train_step()
        eng.comm.host_barrier()
        engine_hyper_overrides(eng, opt)
        hp = read_hyper(eng.hp_dev)
        before = tuple(None if x is None else x.clone() for x in (eng.params, eng.s0, eng.s1))
        eng.load_batch(*engine_batch(B, 200 + r))
        eng.train_step()
        res = (hp, eng.kind, before, tuple(None if x is None else x.clone() for x in (eng.params, eng.s0, eng.s1)), eng.grads.clone())
        eng.comm.host_barrier()
        return res

    out = _run_ranks(2, rank)
    gsum = out[0][4] + out[1][4]
    for r in range(2):
        hp, kind, before, after, _ = out[r]
        engine_dense_check(f"{opt} world 2 rank {r}", kind, hp, before, after, gsum)
    assert torch.equal(out[0][3][0], out[1][3][0]), "dense replicas diverged"
