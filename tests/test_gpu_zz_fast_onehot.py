"""One-hot group lookup fast path (DEEPREC_FAST_ONEHOT=1) == the generic bag-building path, forward and after training steps."""
import os
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_fast_onehot_group_lookup_matches_generic(monkeypatch):
    import deeprec_b200 as dr
    from deeprec_b200.models.zoo import build_model

    def run(flag):
        monkeypatch.setenv("DEEPREC_FAST_ONEHOT", flag)
        dr.embedding_variable.clear_registry()
        torch.manual_seed(3)
        m = build_model("deepfm", ev_option=dr.EmbeddingVariableOption(storage_option=dr.StorageOption(dr.StorageType.HBM)), device="cuda", group_embedding=True)
        opt = dr.optim.AdagradOptimizer(m, lr=0.05)
        g = torch.Generator().manual_seed(5)
        losses = []
        for _ in range(6):
            dense = torch.randn(512, 13, generator=g).cuda(); ids = torch.randint(0, 1000, (26, 512), generator=g).cuda(); y = (torch.rand(512, generator=g) < 0.3).float().cuda()
            loss = m.loss(dense, ids, y); opt.zero_grad(); loss.backward(); opt.step(); losses.append(loss.item())
        with torch.no_grad():
            emb = m.emb(ids).clone()
        return losses, emb

    l0, e0 = run("0")
    l1, e1 = run("1")
    assert all(abs(a - b) < 2e-3 for a, b in zip(l0, l1)), (l0, l1)
    assert torch.allclose(e0, e1, atol=1e-3)
