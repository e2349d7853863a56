"""Shared pieces of the DLRM-DCNv2 engine tests (tests/test_cuda_emu_dlrm_dcn_engine.py, tests/test_gpu_zzzzzzzz_dlrm_dcn.py): the fp32
``DLRM(interaction_op="dcnv2")`` oracle loaded from an engine's weights, the pairing of the engine's flat parameters with the oracle's, and
seeded Criteo-shaped batches."""
import torch

CARDS = [50, 1000, 7, 300] + [97] * 22


def small_config(**kw):
    """D = 16, rank 32, 2 cross layers, B = 256.  The top MLP ends in 256 because the fused head kernel takes K in {256, 512, 1024}."""
    from deeprec_b200.models.dlrm_engine import DLRMConfig
    base = dict(batch_size=256, cardinalities=CARDS, embedding_dim=16, mlp_bot=(32, 16), mlp_top=(64, 256), interaction_op="dcnv2", dcn_num_layers=2,
                dcn_low_rank_dim=32, optimizer="adagrad", learning_rate=0.05)
    base.update(kw)
    return DLRMConfig(**base)


def batch(B, seed, cards=CARDS):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, 13, generator=g) * 3, torch.stack([torch.randint(0, c, (B,), generator=g) for c in cards]),
            (torch.rand(B, generator=g) < 0.3).float())


def oracle_from_engine(eng, device="cpu"):
    from deeprec_b200.models.dlrm import DLRM
    cfg = eng.cfg
    m = DLRM(cfg.num_dense, cfg.cardinalities, cfg.embedding_dim, cfg.mlp_bot, cfg.mlp_top, interaction_op="dcnv2", use_ev=False, device=device,
             bn_eps=cfg.bn_eps, bn_momentum=cfg.bn_momentum, dcn_num_layers=cfg.dcn_num_layers, dcn_low_rank_dim=cfg.dcn_low_rank_dim)
    with torch.no_grad():
        for name, e, o in param_pairs(eng, m):
            o.copy_(e.to(device))
        for t, emb in enumerate(m.tables):
            dm = eng.tables[t].default_matrix
            emb.weight.copy_(dm[torch.arange(emb.num_embeddings, device=dm.device) % dm.shape[0]].to(device))
    return m


def param_pairs(eng, m, grads=False):
    """(name, engine view shaped like the oracle tensor, oracle tensor) for every dense parameter; grads=True: the engine's gradients."""
    src = eng.g if grads else eng.p
    lin_bot = [l for l in m.bot if isinstance(l, torch.nn.Linear)]
    bns = [l for l in m.bot if isinstance(l, torch.nn.BatchNorm1d)]
    lin_top = [l for l in m.top if isinstance(l, torch.nn.Linear)]
    out = []
    for L, lin in zip(eng.bot + eng.top, lin_bot + lin_top):
        out.append((L.name + "/kernel", src(L.name + "/kernel").view(L.N, L.Kp)[:, : L.K], lin.weight))
        out.append((L.name + "/bias", src(L.name + "/bias"), lin.bias))
    for L, bn in zip(eng.bot, bns):
        out.append((L.name + "/bn_gamma", src(L.name + "/bn_gamma"), bn.weight))
        out.append((L.name + "/bn_beta", src(L.name + "/bn_beta"), bn.bias))
    for (V, W), v, w in zip(eng.cross, m.cross_v, m.cross_w):
        out.append((V.name + "/kernel", src(V.name + "/kernel").view(V.N, V.Kp)[:, : V.K], v.weight))
        out.append((W.name + "/kernel", src(W.name + "/kernel").view(W.N, W.Kp)[:, : W.K], w.weight))
        out.append((W.name + "/bias", src(W.name + "/bias"), w.bias))
    out.append(("logits/kernel", src("logits/kernel").view(1, -1), m.logits.weight))
    out.append(("logits/bias", src("logits/bias")[:1], m.logits.bias))
    return out


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def bn_stats(eng, m):
    bns = [l for l in m.bot if isinstance(l, torch.nn.BatchNorm1d)]
    return [(L.running_mean, bn.running_mean, L.running_var, bn.running_var) for L, bn in zip(eng.bot, bns)]
