"""Fused DIN attention kernel vs the composite fp32 PyTorch reference."""
import os
import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,L,D,H1,H2", [(257, 50, 32, 80, 40), (64, 7, 16, 36, 20), (1000, 100, 32, 80, 40), (3, 1, 8, 8, 8)])
def test_din_attention_kernel_matches_reference(B, L, D, H1, H2):
    from deeprec_b200.ops import attention as A
    torch.manual_seed(0)
    att = nn.Sequential(nn.Linear(4 * D, H1), nn.Sigmoid(), nn.Linear(H1, H2), nn.Sigmoid(), nn.Linear(H2, 1)).cuda()
    q = torch.randn(B, D, device="cuda"); k = torch.randn(B, L, D, device="cuda")
    lens = torch.randint(0, L + 1, (B,), device="cuda"); lens[0] = 0; lens[-1] = L
    mask = torch.arange(L, device="cuda").unsqueeze(0) < lens.unsqueeze(1)
    k = k * mask.unsqueeze(-1)
    with torch.no_grad():
        ref = A.din_attention_reference(q, k, mask, att)
        got = A.din_attention(q, k, mask, att)
    assert got.shape == ref.shape and torch.all(got[0] == 0)
    assert torch.allclose(got, ref, atol=2e-4, rtol=1e-3), (got - ref).abs().max()


def test_din_model_inference_uses_the_kernel_and_matches_training_path():
    import deeprec_b200 as dr
    from deeprec_b200.data import taobao_batch
    from deeprec_b200.models.zoo import build_model
    torch.manual_seed(1)
    m = build_model("din", ev_option=dr.EmbeddingVariableOption(storage_option=dr.StorageOption(dr.StorageType.HBM)), device="cuda")
    b = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in taobao_batch(256, max_len=20, n_users=1000, n_items=2000, n_cats=50, seed=0).items()}
    m.eval()
    out_grad_path = m(b).detach()                       # autograd enabled -> composite implementation
    with torch.no_grad():
        out_kernel = m(b)                               # no grad -> fused kernel
    assert torch.allclose(out_kernel, out_grad_path, atol=1e-3, rtol=1e-3), (out_kernel - out_grad_path).abs().max()
