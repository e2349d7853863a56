"""DIN attention unit on csrc/cuda/din_att_kernels.cu: a float64 oracle of both modes and the cases the GPU tests run.

The oracle takes the kernels' rounding points: bf16 operands X = [bf16(k) | bf16(q * k)] (0 at masked positions), bf16([Wk | Wp]) with
Wk = Wb - Wc, bf16(W2), bf16(h1) as the second layer's input, and in the backward bf16(dz2) and bf16(dz1) as the operands of dh1, dX and the
weight gradients.  Everything else is float64.  What is left between kernel and oracle is fp32 accumulation and the odd intermediate that
rounds to the neighbouring bf16 value, so each tensor is held to TOL of its largest magnitude (a planted bug moves it by far more).
"""
from __future__ import annotations

import ctypes as C

import torch

TOL = 2.0 ** -6            # normwise: max |kernel - oracle| <= TOL * max |oracle| (+ ABS)
ABS = 1e-6


def bf16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(torch.float64)


def make_mask(B: int, L: int, seed: int) -> torch.Tensor:
    """row r: kind (r + seed) % 4 -- all valid, tail padding, scattered padding, no valid position."""
    g = torch.Generator().manual_seed(seed)
    m = torch.ones(B, L, dtype=torch.bool)
    for r in range(B):
        kind = (r + seed) % 4
        if kind == 1:
            m[r, int(torch.randint(1, L + 1, (1,), generator=g)):] = False
        elif kind == 2:
            m[r] = torch.rand(L, generator=g) < 0.6
            m[r, int(torch.randint(0, L, (1,), generator=g))] = True
        elif kind == 3:
            m[r] = False
    return m


def make_case(B, L, D, H1, H2, seed, dev, k_dtype=torch.bfloat16, mask=None):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, D, generator=g) * 0.7
    k = torch.randn(B, L, D, generator=g) * 0.7
    mask = make_mask(B, L, seed) if mask is None else mask
    k = torch.where(mask.unsqueeze(-1), k, torch.full_like(k, 3e4))       # whatever k holds at masked positions must not matter
    W1 = torch.randn(H1, 4 * D, generator=g) * (1.5 / (4 * D) ** 0.5)
    b1 = torch.randn(H1, generator=g) * 0.2
    W2 = torch.randn(H2, H1, generator=g) * (2.0 / H1 ** 0.5)
    b2 = torch.randn(H2, generator=g) * 0.2
    w3 = torch.randn(H2, generator=g) * (4.0 / H2 ** 0.5)
    b3 = torch.randn(1, generator=g)
    t = dict(q=q, k=k.to(k_dtype), mask=mask, W1=W1, b1=b1, W2=W2, b2=b2, w3=w3, b3=b3)
    return {n: v.to(dev) for n, v in t.items()}


def _split(W1, D):
    Wa, Wb, Wc, Wd = W1[:, :D], W1[:, D:2 * D], W1[:, 2 * D:3 * D], W1[:, 3 * D:]
    Wq = Wa.double() + Wc.double()
    Wk = (Wb - Wc).float()                 # fp32 difference, as the kernels stage it
    return Wq, bf16(Wk), bf16(Wd)


def oracle(c, mode: int, gout=None):
    """Float64 forward (out [B, D] or w [B, L]) and, with gout, every gradient: dict."""
    q, k, m = c["q"].double(), c["k"].double(), c["mask"]
    B, L, D = k.shape
    Wq, Wk, Wp = _split(c["W1"], D)
    W2b, b1, b2, w3 = bf16(c["W2"]), c["b1"].double(), c["b2"].double(), c["w3"].double()
    mf = m.unsqueeze(-1).double()
    Xk = bf16(c["k"].float()) * mf
    Xp = bf16((c["q"].float().unsqueeze(1) * c["k"].float())) * mf
    hq = q @ Wq.t() + b1
    z1 = Xk @ Wk.t() + Xp @ Wp.t() + hq.unsqueeze(1)
    h1 = torch.sigmoid(z1)
    h1b = bf16(h1)
    h2 = torch.sigmoid(h1b @ W2b.t() + b2)
    s = h2 @ w3
    any_ = m.any(-1, keepdim=True)
    s = s.masked_fill(~m, float("-inf"))
    w = torch.softmax(torch.where(any_, s, torch.zeros_like(s)), -1)
    w = torch.where(m, w, torch.zeros_like(w))
    kz = torch.where(m.unsqueeze(-1), k, torch.zeros_like(k))
    if mode == 0:
        w = w * any_
        out = (w.unsqueeze(-1) * kz).sum(1)
    else:
        out = torch.where(any_, w, torch.full_like(w, 1.0 / L))
    r = {"out": out}
    if gout is None:
        return r
    g = gout.double()
    gt = (kz @ g.unsqueeze(-1)).squeeze(-1) if mode == 0 else g
    cs = (w * gt).sum(-1, keepdim=True)
    ds = torch.where(m & any_, w * (gt - cs), torch.zeros_like(w))
    dz2 = ds.unsqueeze(-1) * w3 * h2 * (1 - h2)
    dz2b = bf16(dz2)
    dz1 = (dz2b @ W2b) * h1 * (1 - h1) * mf
    dz1b = bf16(dz1)
    dXk, dXp = dz1b @ Wk, dz1b @ Wp
    dk = (dXk + q.unsqueeze(1) * dXp) * mf
    if mode == 0:
        dk = dk + w.unsqueeze(-1) * g.unsqueeze(1)
    dhq = dz1.sum(1)
    r["dq"] = dhq @ Wq + (kz * dXp).sum(1)
    r["dk"] = dk
    dWk = torch.einsum("blh,bld->hd", dz1b, Xk)
    dWp = torch.einsum("blh,bld->hd", dz1b, Xp)
    dWq = dhq.t() @ q
    r["dW1"] = torch.cat([dWq, dWk, dWq - dWk, dWp], 1)
    r["db1"] = dhq.sum(0)
    r["dW2"] = torch.einsum("blj,blh->jh", dz2b, h1b)
    r["db2"] = dz2.sum((0, 1))
    r["dw3"] = (ds.unsqueeze(-1) * h2).sum((0, 1))
    r["db3"] = torch.zeros(1, dtype=torch.float64, device=q.device)
    return r


def _p(t):
    return C.c_void_p(t.data_ptr())


def run_kernels(c, mode: int, gout=None):
    """The two entry points on case c, outputs NaN-filled before the call: (rc_fwd, out, rc_bwd, grads dict)."""
    from deeprec_b200 import _native
    from deeprec_b200._native import stream_ptr
    lib = _native.cuda()
    q, k, m = c["q"].float().contiguous(), c["k"].contiguous(), c["mask"].contiguous()
    B, L, D = k.shape
    H1, H2 = c["W1"].shape[0], c["W2"].shape[0]
    kb = int(k.dtype == torch.bfloat16)
    W = [c[n].float().contiguous() for n in ("W1", "b1", "W2", "b2", "w3")]
    out = torch.full((B, D) if mode == 0 else (B, L), float("nan"), device=q.device)
    rc = lib.dr_cuda_din_att_fwd(_p(q), _p(k), kb, _p(m), B, L, D, _p(W[0]), _p(W[1]), H1, _p(W[2]), _p(W[3]), H2, _p(W[4]), mode, _p(out),
                                 stream_ptr())
    if gout is None:
        return rc, out, None, None
    nan = lambda *s, dt=torch.float32: torch.full(s, float("nan"), dtype=dt, device=q.device)
    gr = {"dq": nan(B, D), "dk": nan(B, L, D, dt=k.dtype), "dW1": nan(H1, 4 * D), "db1": nan(H1), "dW2": nan(H2, H1), "db2": nan(H2),
          "dw3": nan(H2), "db3": nan(1)}
    scratch = torch.empty(B * L * (2 * D + 2 * H1 + H2), dtype=torch.bfloat16, device=q.device)
    gf = gout.float().contiguous()
    rc2 = lib.dr_cuda_din_att_bwd(_p(q), _p(k), kb, _p(m), _p(gf), B, L, D, _p(W[0]), _p(W[1]), H1, _p(W[2]), _p(W[3]), H2, _p(W[4]), mode,
                                  *[_p(gr[n]) for n in ("dq", "dk", "dW1", "db1", "dW2", "db2", "dw3", "db3")], _p(scratch), stream_ptr())
    return rc, out, rc2, gr


def make_gout(c, mode: int, seed: int):
    B, L, D = c["k"].shape
    g = torch.Generator().manual_seed(seed + 7)
    return (torch.randn(B, D, generator=g) if mode == 0 else torch.randn(B, L, generator=g)).to(c["q"].device)


def close(got, ref, what):
    got, ref = got.double(), ref.double()
    assert not torch.isnan(got).any(), f"{what}: NaN"
    err = (got - ref).abs().max().item()
    bound = TOL * ref.abs().max().item() + ABS
    assert err <= bound, f"{what}: max error {err:.3e} > {bound:.3e}"


def check_case(B, L, D, H1, H2, mode, seed, dev, k_dtype=torch.bfloat16):
    c = make_case(B, L, D, H1, H2, seed, dev, k_dtype)
    gout = make_gout(c, mode, seed)
    rc, out, rc2, gr = run_kernels(c, mode, gout)
    assert rc == 0 and rc2 == 0, (rc, rc2)
    ref = oracle(c, mode, gout)
    close(out, ref["out"], "out")
    for n in ("dq", "dk", "dW1", "db1", "dW2", "db2", "dw3"):
        close(gr[n], ref[n], n)
    # exact values: dk = 0 at masked positions, empty rows, db3 = 0
    m = c["mask"]
    assert bool((gr["dk"][~m] == 0).all())
    assert float(gr["db3"][0]) == 0.0
    empty = ~m.any(-1)
    if bool(empty.any()):
        if mode == 0:
            assert bool((out[empty] == 0).all())
        else:
            assert bool((out[empty] == torch.tensor(1.0 / L, dtype=torch.float32)).all())
        assert bool((gr["dq"][empty] == 0).all()) and bool((gr["dk"][empty] == 0).all())
    return c, gout, gr


def empty_rows_add_nothing(dev, mode):
    """Appending samples with no valid position changes no parameter gradient by a single bit."""
    B, L, D, H1, H2 = 8, 20, 32, 80, 40
    c = make_case(B, L, D, H1, H2, 5, dev, mask=torch.ones(B, L, dtype=torch.bool))
    gout = make_gout(c, mode, 5)
    *_, g1 = run_kernels(c, mode, gout)
    c2 = dict(c)
    c2["q"] = torch.cat([c["q"], c["q"][:4] * 3])
    c2["k"] = torch.cat([c["k"], c["k"][:4] * 5])
    c2["mask"] = torch.cat([c["mask"], torch.zeros(4, L, dtype=torch.bool, device=dev)])
    gout2 = torch.cat([gout, gout[:4] * 9])
    *_, g2 = run_kernels(c2, mode, gout2)
    for n in ("dW1", "db1", "dW2", "db2", "dw3"):
        assert torch.equal(g1[n], g2[n]), n
    assert bool((g2["dq"][B:] == 0).all()) and bool((g2["dk"][B:] == 0).all())


# ---- engines --------------------------------------------------------------------------------------------------------------------------
def seq_engine(name, dev, B, **kw):
    import gru_cases as G
    import pooled_bag_cases as K
    return G.dien_engine(dev, B, model=K.seq_model(name, dev), **kw)


def run_vs_replica(name, dev, graph: bool = False, steps: int = 6, B: int = 256):
    """gru_cases.run_dien_vs_replica for DIN or DIEN: the engine (fused attention) against the zoo model on nn.Embedding tables, whose
    head runs the attention unit in torch."""
    import gru_cases as G
    import pooled_bag_cases as K
    from deeprec_b200.models.rec_engine import din_ids
    eng = seq_engine(name, dev, B, learning_rate=0.05)
    rep = G._seq_replica(eng, dev)
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


def train(name, dev, graph: bool, steps: int = 5, B: int = 1024):
    import pooled_bag_cases as K
    from deeprec_b200.models.rec_engine import din_ids
    eng = seq_engine(name, dev, B, learning_rate=0.05)
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
