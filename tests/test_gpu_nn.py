"""deeprec_b200.nn layers (wgmma GEMM chain, fused interactions) against plain fp32 PyTorch."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return (a.float() - b.float()).abs().max().item() / (b.float().abs().max().item() + 1e-6)


def _rel_fro(a, b):
    """relative Frobenius error: robust to the isolated ReLU-mask flips bf16 rounding causes at pre-activations ~ 0"""
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def _r(t):
    """bf16 rounding as a differentiable op (gradient rounded the same way): emulates the kernels' storage precision in fp32 math"""
    return t.bfloat16().float()


@pytest.mark.parametrize("M,in_dim,sizes,last_act", [(4096, 429, (1024, 256, 32), True), (1000, 64, (512, 256), True), (777, 13, (64, 16, 1), False),
                                                      (2048, 96, (80,), False), (513, 40, (200, 80, 2), False)])
def test_fused_mlp_matches_fp32(M, in_dim, sizes, last_act):
    from deeprec_b200.nn import FusedMLP
    torch.manual_seed(0)
    m = FusedMLP(in_dim, sizes, last_act=last_act, device="cuda")
    for b in m.biases:
        torch.nn.init.normal_(b, std=0.1)
    x = torch.randn(M, in_dim, device="cuda", requires_grad=True)
    y = m(x)
    assert y.shape == (M, sizes[-1]) and y.dtype == torch.float32
    # fp32 reference of the same chain with bf16-rounded storage (inputs, weights, activations): only the accumulation differs
    xr = x.detach().clone().requires_grad_(True)
    h = _r(xr)
    Ws = [w.detach().clone().requires_grad_(True) for w in m.weights]
    bs = [b.detach().clone().requires_grad_(True) for b in m.biases]
    for i, (w, b) in enumerate(zip(Ws, bs)):
        h = torch.nn.functional.linear(h, _r(w), b)
        if i + 1 < len(Ws) or last_act:
            h = torch.relu(h)
        h = _r(h)
    assert _rel(y, h) < 2e-2
    g = torch.randn_like(h) * 0.1
    y.backward(g); h.backward(g)
    assert _rel_fro(x.grad, xr.grad) < 3e-2, _rel_fro(x.grad, xr.grad)
    for w, wr in zip(m.weights, Ws):
        assert _rel_fro(w.grad, wr.grad) < 3e-2, _rel_fro(w.grad, wr.grad)
    for b, br in zip(m.biases, bs):
        assert _rel_fro(b.grad, br.grad) < 3e-2, _rel_fro(b.grad, br.grad)


def test_fused_mlp_trains():
    from deeprec_b200.nn import FusedMLP
    torch.manual_seed(1)
    m = torch.nn.Sequential(FusedMLP(32, (128, 64)), torch.nn.Linear(64, 1)).cuda()
    opt = torch.optim.Adam(m.parameters(), 1e-2)
    x = torch.randn(2048, 32, device="cuda"); y = (x[:, :4].sum(1, keepdim=True) > 0).float()
    first = None
    for _ in range(60):
        loss = torch.nn.functional.binary_cross_entropy_with_logits(m(x), y)
        first = first or loss.item()
        opt.zero_grad(); loss.backward(); opt.step()
    assert loss.item() < 0.5 * first


def test_interaction_functions():
    from deeprec_b200.models.dlrm import dot_interaction as ref_dot
    from deeprec_b200.nn import dot_interaction, fm_interaction
    torch.manual_seed(2)
    B, T, D = 1537, 26, 16
    x = torch.randn(B, D, device="cuda", requires_grad=True); e = (torch.randn(B, T, D, device="cuda") * 0.5).requires_grad_(True)
    xr, er = x.detach().clone().requires_grad_(True), e.detach().clone().requires_grad_(True)
    z, zr = dot_interaction(x, e), ref_dot(xr, er)
    assert z.shape == zr.shape and _rel(z, zr) < 3e-2
    g = torch.randn_like(zr) * 0.1
    z.backward(g); zr.backward(g)
    assert _rel(x.grad, xr.grad) < 4e-2 and _rel(e.grad, er.grad) < 4e-2
    e2 = (torch.randn(B, 10, D, device="cuda") * 0.5).requires_grad_(True); e2r = e2.detach().clone().requires_grad_(True)
    f, fr = fm_interaction(e2), 0.5 * (e2r.sum(1) ** 2 - (e2r ** 2).sum(1))
    assert _rel(f, fr) < 3e-2
    g = torch.randn_like(fr) * 0.1
    f.backward(g); fr.backward(g)
    assert _rel(e2.grad, e2r.grad) < 4e-2


@pytest.mark.parametrize("name", ["deepfm", "wdl", "dcn", "dlrm"])
def test_zoo_models_run_on_fused_kernels(name):
    """Criteo-shaped zoo models on cuda: MLPs are FusedMLP/FusedLinear nodes, embeddings are device tables."""
    import deeprec_b200 as dr
    from deeprec_b200.models.zoo import build_model
    from deeprec_b200.nn import FusedMLP
    torch.manual_seed(3)
    opt_ev = dr.EmbeddingVariableOption(storage_option=dr.StorageOption(dr.StorageType.HBM))
    m = build_model(name, ev_option=opt_ev, device="cuda", group_embedding=True)
    assert any(isinstance(x, FusedMLP) for x in m.modules()) or name == "dlrm"
    B = 512
    dense = torch.randn(B, 13, device="cuda"); ids = torch.randint(0, 1000, (26, B), device="cuda"); y = (torch.rand(B, device="cuda") < 0.3).float()
    opt = dr.optim.AdagradOptimizer(m, lr=0.05)
    losses = []
    for _ in range(8):
        loss = m.loss(dense, ids, y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(l == l for l in losses) and losses[-1] < losses[0]
