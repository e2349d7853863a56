"""nn.fused_din_attention off the GPU is today's torch expression, bit for bit: DIN's ops.attention.din_attention (sum) and DIEN's inline
softmax (weights), forward and every gradient; and the zoo heads with ``attention=fused_din_attention`` equal the heads without it."""
import pytest
import torch

from deeprec_b200.nn import fused_din_attention


def _unit(D, seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(4 * D, 80), torch.nn.Sigmoid(), torch.nn.Linear(80, 40), torch.nn.Sigmoid(), torch.nn.Linear(40, 1))


def _inputs(B=6, L=9, D=32, seed=1):
    g = torch.Generator().manual_seed(seed)
    q, k = torch.randn(B, D, generator=g), torch.randn(B, L, D, generator=g)
    mask = torch.rand(B, L, generator=g) < 0.7
    mask[0] = True
    mask[1] = False
    mask[2, 4:] = False
    return q, k, mask


def _grads(fn, q, k, mask, att):
    att.zero_grad(set_to_none=True)
    q, k = q.clone().requires_grad_(), k.clone().requires_grad_()
    out = fn(q, k, mask, att)
    (out * torch.linspace(-1, 1, out.shape[-1])).sum().backward()
    return [out.detach(), q.grad, k.grad] + [p.grad for p in att.parameters()]


def _dien_weights(q, k, mask, att):
    qe = q.unsqueeze(1).expand_as(k)
    s = att(torch.cat([qe, k, qe - k, qe * k], -1)).squeeze(-1).masked_fill(~mask, -2 ** 31)
    return torch.softmax(s, -1)


@pytest.mark.parametrize("weights", (False, True))
def test_cpu_path_is_todays_expression(weights):
    from deeprec_b200.ops.attention import din_attention
    att = _unit(32)
    q, k, mask = _inputs()
    ref = _dien_weights if weights else din_attention
    got = _grads(lambda *a: fused_din_attention(*a, weights=weights), q, k, mask, att)
    exp = _grads(ref, q, k, mask, att)
    for a, b in zip(got, exp):
        assert torch.equal(a, b)


def test_unsupported_unit_raises():
    q, k, mask = _inputs()
    with pytest.raises(ValueError, match="fused_din_attention"):
        fused_din_attention(q, k, mask, torch.nn.Sequential(torch.nn.Linear(128, 1)))
    with pytest.raises(ValueError, match="fused_din_attention"):
        fused_din_attention(q, k[..., :16], mask, _unit(32))


def _seq_inputs(model, B=5, L=7, seed=3):
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(B, model.emb_dim, generator=g)
    q = torch.randn(B, 2 * model.emb_dim, generator=g)
    mask = torch.zeros(B, L, dtype=torch.bool)
    for b, n in enumerate((7, 3, 0, 5, 1)[:B]):
        mask[b, :n] = True
    k = torch.randn(B, L, 2 * model.emb_dim, generator=g) * mask.unsqueeze(-1)
    return u, q, k, mask


@pytest.mark.parametrize("name", ("din", "dien"))
def test_zoo_heads_with_the_op_equal_the_heads_without(name):
    import deeprec_b200 as dr
    from deeprec_b200.models.zoo import build_model
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    model = build_model(name, device="cpu")
    model.train()
    u, q, k, mask = _seq_inputs(model)
    outs = []
    for attention in (None, fused_din_attention):
        torch.manual_seed(1)
        model.zero_grad(set_to_none=True)
        kk = k.clone().requires_grad_()
        y = model.head(u, q, kk, mask) if attention is None else model.head(u, q, kk, mask, attention=attention)
        y.sum().backward()
        outs.append([y.detach(), kk.grad] + [p.grad for p in model.parameters() if p.grad is not None])
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert len(outs[0]) == len(outs[1])
