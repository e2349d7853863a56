"""Shared cases for the GRU recurrence kernels (csrc/cuda/rnn_kernels.cu), ``nn.fused_gru`` and DIEN on FusedRecEngine, with the float64
oracle they are checked against.

The oracle mirrors the kernels' rounding points: gi is bf16, W_hh enters the products as bf16, the state h is fp32 and enters the product
h W_hh^T rounded to bf16; in the backward dgh = [da_r, da_z, da_n r] enters dgh W_hh rounded to bf16 and the carry dh is fp32.  Everything
else is float64.

Bounds (u = 2^-24, the fp32 unit roundoff; b = 2^-8, the bf16 one):
  * one forward step, started from the kernel's own fp32 state y[t-1]: both sides use the same bf16 operands, so they differ only by the
    fp32 accumulation of the mma (at most (H + 1) u sum|terms| on gh), fp32 rounding of the gate arithmetic and __expf (ex2.approx,
    relative error below 2^-21 for the arguments a GRU sees, |x| < 64).  sigmoid' <= 1/4, tanh' <= 1 and |h|, |n|, z, r <= 1, so
    |y[t] - step(y[t-1])| <= 2^-16 (1 + max|gh|) covers all of it with margin (STEP_TOL);
  * the free-running forward against the oracle run from h_0 = 0: where the two fp32 states straddle a bf16 rounding boundary the operand
    of one component differs by one bf16 ulp, which moves gh by <= b |h_k| |W_nk|; the GRU contracts (z, 1 - z <= 1) so these do not grow,
    and 2^-7 absolute covers L = 50 steps at the weight scales of nn.GRU's default init (FREE_TOL);
  * the backward from the kernel's forward: the kernel rounds dgi to bf16 (b/2 relative) and the carry product sees bf16(dgh) (b/2
    relative per term, a flip of one ulp where the two sides straddle a boundary); the backward is linear in dy and the carry contracts by
    z < 1 per step, so the error of every dgi row is below 2^-5 of the largest |dgi| of the tensor (BWD_REL);
  * dW_hh, db_hh: the split-K GEMM adds bf16 products in fp32 (exact products, (rows) u relative on the sum); the operands differ from the
    oracle's by the dgh error above, so |dW - dW_ref| <= 2^-5 sum|dgh_ref| |h| + 2^-20 elementwise (and the same for db with |h| = 1).
"""
from __future__ import annotations

import copy

import torch

STEP_TOL = 2.0 ** -16
FREE_TOL = 2.0 ** -7
BWD_REL = 2.0 ** -5


def bf16(t: torch.Tensor) -> torch.Tensor:
    """Round to bf16 (nearest even) and back to float64."""
    return t.float().to(torch.bfloat16).double()


def f32(t: torch.Tensor) -> torch.Tensor:
    return t.float().double()


def make_lengths(kind: str, B: int, L: int, seed: int = 0) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    if kind == "full":
        return torch.full((B,), L, dtype=torch.int32)
    if kind == "one":
        return torch.ones(B, dtype=torch.int32)
    if kind == "zero":
        return torch.zeros(B, dtype=torch.int32)
    return torch.randint(0, L + 1, (B,), generator=g, dtype=torch.int32)


def make_case(B: int, L: int, H: int, seed: int, dev):
    """gi bf16 [B L, 3H], W_hh fp32 [3H, H], b_hh fp32 [3H] at nn.GRU's init scale (U(-1/sqrt(H), 1/sqrt(H))), dy fp32 [B, L, H]."""
    g = torch.Generator().manual_seed(seed)
    k = H ** -0.5
    gi = (torch.rand(B * L, 3 * H, generator=g) * 2 - 1).to(torch.bfloat16)
    w = (torch.rand(3 * H, H, generator=g) * 2 - 1) * k
    b = (torch.rand(3 * H, generator=g) * 2 - 1) * k
    dy = torch.randn(B, L, H, generator=g)
    return gi.to(dev), w.to(dev), b.to(dev), dy.to(dev)


def _gates(gi_t, hprev, wb, b, H):
    """float64 gates of one step from gi_t [B, 3H] (bf16 values), the fp32 state hprev [B, H] (its bf16 rounding is the operand)."""
    gh = bf16(hprev) @ wb.t() + b
    r = torch.sigmoid(gi_t[:, :H] + gh[:, :H])
    z = torch.sigmoid(gi_t[:, H:2 * H] + gh[:, H:2 * H])
    n = torch.tanh(gi_t[:, 2 * H:] + r * gh[:, 2 * H:])
    return r, z, n, gh


def oracle_step(gi, w, b, y, lengths, B, L, H):
    """One forward step from the kernel's own state: want[b, t] = step(y[b, t - 1]) for t < len[b], 0 past it, and max|gh| per row."""
    gid, wb, bd = gi.double().view(B, L, 3 * H), bf16(w), b.double()
    prev = torch.cat([torch.zeros(B, 1, H, dtype=torch.float64, device=y.device), y.double()[:, :-1]], 1)
    r, z, n, gh = _gates(gid.reshape(B * L, 3 * H), prev.reshape(B * L, H), wb, bd, H)
    h = (1 - z) * n + z * prev.reshape(B * L, H)
    live = (torch.arange(L, device=y.device)[None] < lengths.to(y.device).long()[:, None]).reshape(B * L, 1)
    return (h * live).view(B, L, H), gh.abs().amax(1).view(B, L, 1)


def oracle_forward(gi, w, b, lengths, B, L, H):
    """Free-running float64 forward from h_0 = 0 (fp32 state, bf16 operand)."""
    gid, wb, bd = gi.double().view(B, L, 3 * H), bf16(w), b.double()
    lens = lengths.to(gi.device).long()
    h = torch.zeros(B, H, dtype=torch.float64, device=gi.device)
    ys = []
    for t in range(L):
        r, z, n, _ = _gates(gid[:, t], h, wb, bd, H)
        live = (t < lens)[:, None]
        h = torch.where(live, f32((1 - z) * n + z * h), h)
        ys.append(h * live)
    return torch.stack(ys, 1)


def oracle_backward(gi, w, b, lengths, y, dy, B, L, H):
    """float64 backward through time from the kernel's forward y (gates recomputed from its fp32 states): dgi [B L, 3H], dW_hh, db_hh, and
    the magnitudes sum|dgh| |h_{t-1}| (for dW) and sum|dgh| (for db) the bounds scale with."""
    gid, wb, bd = gi.double().view(B, L, 3 * H), bf16(w), b.double()
    lens = lengths.to(gi.device).long()
    yd = y.double()
    dyd = dy.double()
    dh = torch.zeros(B, H, dtype=torch.float64, device=gi.device)
    dgi = torch.zeros(B, L, 3 * H, dtype=torch.float64, device=gi.device)
    dW = torch.zeros(3 * H, H, dtype=torch.float64, device=gi.device)
    dWmag = torch.zeros_like(dW)
    db = torch.zeros(3 * H, dtype=torch.float64, device=gi.device)
    dbmag = torch.zeros_like(db)
    for t in range(L - 1, -1, -1):
        live = (t < lens)[:, None]
        hprev = yd[:, t - 1] if t > 0 else torch.zeros(B, H, dtype=torch.float64, device=gi.device)
        r, z, n, gh = _gates(gid[:, t], hprev, wb, bd, H)
        d = torch.where(live, dh + dyd[:, t], torch.zeros_like(dh))
        da_n = d * (1 - z) * (1 - n * n)
        da_z = d * (hprev - n) * z * (1 - z)
        da_r = da_n * gh[:, 2 * H:] * r * (1 - r)
        dgi[:, t] = torch.cat([da_r, da_z, da_n], 1)
        dgh = bf16(torch.cat([da_r, da_z, da_n * r], 1))
        hb = bf16(hprev)
        dW += dgh.t() @ hb
        dWmag += dgh.abs().t() @ hb.abs()
        db += dgh.sum(0)
        dbmag += dgh.abs().sum(0)
        dh = f32(dgh @ wb + z * d)
    return dgi.view(B * L, 3 * H), dW, db, dWmag, dbmag


def run_kernels(B, L, H, lengths, seed, dev, inputs=None):
    """The two C entry points on NaN-filled output buffers; returns the inputs (made here unless given, with ``lengths`` on the device) and
    y, dgi, dW_hh, db_hh."""
    from deeprec_b200 import _native
    from deeprec_b200._native import ptr, stream_ptr
    lib = _native.cuda()
    gi, w, b, dy = inputs if inputs is not None else make_case(B, L, H, seed, dev)
    ln = lengths.to(dev)
    nan = lambda *s, dt=torch.float32: torch.full(s, float("nan"), dtype=dt, device=dev)
    y = nan(B, L, H)
    assert lib.dr_cuda_gru_fwd(ptr(gi), ptr(w), ptr(b), ptr(ln), B, L, H, ptr(y), stream_ptr()) == 0
    dgi, dgh, hp = nan(B * L, 3 * H, dt=torch.bfloat16), nan(B * L, 3 * H, dt=torch.bfloat16), nan(B * L, H, dt=torch.bfloat16)
    dW, db = torch.zeros(3 * H, H, device=dev), torch.zeros(3 * H, device=dev)
    assert lib.dr_cuda_gru_bwd(ptr(gi), ptr(w), ptr(b), ptr(ln), ptr(y), ptr(dy), B, L, H, ptr(dgi), ptr(dgh), ptr(hp), ptr(dW), ptr(db),
                               stream_ptr()) == 0
    return (gi, w, b, dy), (y, dgi, dW, db)


def check_kernels(B, L, H, kind, dev, seed=0):
    lengths = make_lengths(kind, B, L, seed + B)
    (gi, w, b, dy), (y, dgi, dW, db) = run_kernels(B, L, H, lengths, seed + 7 * B + L, dev)
    torch.cuda.synchronize()
    live = (torch.arange(L)[None] < lengths.long()[:, None]).to(dev)                 # [B, L]
    # past the length: exactly zero (the buffers were NaN)
    assert bool((y[~live] == 0).all()), "y past the length is not exactly 0"
    assert bool((dgi.view(B, L, 3 * H)[~live] == 0).all()), "dgi past the length is not exactly 0"
    assert not bool(torch.isnan(y).any()) and not bool(torch.isnan(dgi.float()).any())
    # one step from the kernel's own state
    want, ghmax = oracle_step(gi, w, b, y, lengths, B, L, H)
    err = (y.double() - want).abs()
    assert bool((err <= STEP_TOL * (1 + ghmax)).all()), ("forward step", float(err.max()))
    # free-running
    ref = oracle_forward(gi, w, b, lengths, B, L, H)
    assert float((y.double() - ref).abs().max()) <= FREE_TOL, ("free-running forward", float((y.double() - ref).abs().max()))
    # backward
    dgi_ref, dW_ref, db_ref, dWmag, dbmag = oracle_backward(gi, w, b, lengths, y, dy, B, L, H)
    scale = float(dgi_ref.abs().max())
    e = float((dgi.double() - dgi_ref).abs().max())
    assert e <= BWD_REL * scale + 1e-30, ("dgi", e, scale)
    assert bool(((dW.double() - dW_ref).abs() <= BWD_REL * dWmag + 2.0 ** -20).all()), ("dW_hh", float((dW.double() - dW_ref).abs().max()))
    assert bool(((db.double() - db_ref).abs() <= BWD_REL * dbmag + 2.0 ** -20).all()), ("db_hh", float((db.double() - db_ref).abs().max()))


# ---- the op ---------------------------------------------------------------------------------------------------------------------------
def op_vs_module(B, L, I, H, dev, seed=0):
    """fused_gru (bf16 projection and recurrence) against fp32 nn.GRU autograd on the valid positions: outputs, dx, and the four parameter
    gradients, each within 2^-5 of the largest magnitude of its reference (bf16 operands through L steps)."""
    from deeprec_b200.nn import fused_gru
    torch.manual_seed(seed)
    gru = torch.nn.GRU(I, H, batch_first=True, device=dev)
    ref = copy.deepcopy(gru)
    lengths = make_lengths("random", B, L, seed)
    live = (torch.arange(L)[None] < lengths.long()[:, None]).to(dev)
    x = torch.randn(B, L, I, device=dev)
    R = torch.randn(B, L, H, device=dev) * live.unsqueeze(-1)
    x1 = x.clone().requires_grad_(True)
    y = fused_gru(x1, gru, lengths.to(dev))
    (y * R).sum().backward()
    x2 = x.clone().requires_grad_(True)
    y2, _ = ref(x2)
    (y2 * R).sum().backward()
    assert bool((y[~live] == 0).all())
    def close(a, b, what):
        err, mag = float((a.detach().float() - b.detach().float()).abs().max()), float(b.detach().float().abs().max())
        assert err <= 2.0 ** -5 * mag + 1e-6, (what, err, mag)
    close(y[live], y2[live], "y")
    close(x1.grad[live], x2.grad[live], "dx")
    for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"):
        close(getattr(gru, n).grad, getattr(ref, n).grad, n)
        assert getattr(gru, n).grad.dtype == torch.float32


# ---- DIEN on the engine ---------------------------------------------------------------------------------------------------------------
def dien_engine(dev, B, model=None, **kw):
    import pooled_bag_cases as K
    from deeprec_b200.models.rec_engine import din_engine
    model = model if model is not None else K.seq_model("dien", dev)
    return din_engine(model, B, K.L, table_rows=K.CARDS, device=None if dev.type == "cpu" else dev, **kw)


def _seq_replica(eng, dev):
    """pooled_bag_cases.replica_of with tables that also serve DIEN's per-position lookup on host tensors (padding ids -> zero rows)."""
    import pooled_bag_cases as K
    from deeprec_b200.config import PAD_KEY

    class SeqTable(K._ReplicaTable):
        device = property(lambda self: self.emb.weight.device)

        def lookup(self, ids):
            ok = (ids >= 0) & (ids != PAD_KEY)
            return self.emb(torch.where(ok, ids, torch.zeros_like(ids))) * ok.unsqueeze(-1)
    rep = K.replica_of(eng, dev, "sum")
    for name in ("user", "item", "cat"):
        getattr(rep, name).__class__ = SeqTable
    return rep


def run_dien_vs_replica(dev, graph: bool = False, steps: int = 6, B: int = 256):
    """Adagrad on the tables and the dense net, DIEN engine against the zoo model with nn.Embedding tables and nn.GRU: per-step loss, then
    rows of the user / item tables.  taobao_like has tail padding and empty histories."""
    import pooled_bag_cases as K
    from deeprec_b200.models.rec_engine import din_ids
    eng = dien_engine(dev, B, learning_rate=0.05)
    rep = _seq_replica(eng, dev)
    opt = torch.optim.Adagrad(rep.parameters(), lr=0.05, initial_accumulator_value=0.1, eps=0.0)
    le, lr_ = [], []
    for s in range(steps):
        b = K.taobao_like(B, 100 + s)
        eng.load_batch(din_ids(b).to(dev), b["labels"].to(dev))
        if graph and s == 0:
            eng.capture(warmup=1)
        else:
            eng.train_step()
        le.append(eng.loss_value())
        loss = rep.loss({k: v.to(dev) for k, v in b.items()})
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
    assert p.shape == (B,) and bool(((p >= 0) & (p <= 1)).all())
    return eng


def train_dien(dev, graph: bool, steps: int = 6, B: int = 1024, **kw):
    """Parameters, last loss and every table row after ``steps`` DIEN engine steps."""
    import pooled_bag_cases as K
    from deeprec_b200.models.rec_engine import din_ids
    eng = dien_engine(dev, B, learning_rate=0.05, **kw)
    losses = []
    for s in range(steps):
        b = K.taobao_like(B, 1300 + s)
        eng.load_batch(din_ids(b).to(dev), b["labels"].to(dev))
        if graph and s == 0:
            eng.capture(warmup=1)
        else:
            eng.train_step()
        losses.append(eng.loss_value())
    probe = [torch.arange(c, device=eng.dev) for c in K.CARDS]
    return eng.params.clone(), losses, [eng.tables[t].lookup(probe[t]).clone() for t in range(3)]
