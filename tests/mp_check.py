"""Multi-GPU correctness script (run under torchrun): the fused unique-first P2P pipeline must agree with the NCCL
re-creation of the reference (SOK) dataflow, and the P2P all-reduce with ncclAllReduce.  Mirrors the reference's SOK unit
tests, which compare the multi-GPU embedding against a single-device model
(addons/sparse_operation_kit/legacy/unit_test/test_scripts/tf1/test_dense_emb_demo.py)."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gathered_rows(eng, t, probe, dev):
    """Rows / frequencies of `probe` keys of table t, whichever rank owns them (sum over ranks of the present entries)."""
    rows = torch.zeros(probe.numel(), eng.D, device=dev)
    freq = torch.zeros(probe.numel(), device=dev)
    cnt = torch.zeros(probe.numel(), device=dev)
    if t in eng.tables:
        f = eng.tables[t].get_freq(probe).float().to(dev)
        present = (f > 0).float()
        rows = eng.tables[t].lookup(probe).to(dev) * present[:, None]
        freq, cnt = f, present
    for x in (rows, freq, cnt):
        dist.all_reduce(x)
    return rows, freq, cnt


def main(optimizer: str = "adagrad"):
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    from deeprec_b200.data.synthetic import criteo_batch
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    from deeprec_b200.parallel.nccl_baseline import NcclComm
    from deeprec_b200.parallel.p2p import P2PComm

    p2p = P2PComm(rank, world, dev)
    # ---- 1. one-shot P2P all-reduce vs NCCL
    g = p2p.alloc_grads(1 << 16)
    torch.manual_seed(rank)
    g.copy_(torch.randn(1 << 16, device=dev))
    ref = g.clone()
    dist.all_reduce(ref)
    out = torch.empty_like(ref)
    p2p.allreduce(out)
    torch.cuda.synchronize()
    err = (out - ref).abs().max().item()
    assert err < 1e-4, f"p2p allreduce mismatch {err}"
    dist.barrier()

    # ---- 2. DLRM engine: unique-first P2P pipeline vs NCCL (SOK) dataflow, same seeds / batches
    cards = [50, 1000, 7, 300] + [97] * 21 + [200000]
    cfg = DLRMConfig(batch_size=2048, cardinalities=cards, optimizer=optimizer, learning_rate=0.05)
    nsteps = 5
    batches = [criteo_batch(cfg.batch_size, 13, cards, seed=100 * rank + s) for s in range(nsteps)]
    results = {}
    probe = torch.arange(0, 300, device=dev)
    for name in ("p2p", "nccl"):
        comm = P2PComm(rank, world, dev) if name == "p2p" else NcclComm(rank, world, dev)
        eng = DLRMEngine(cfg, dev, rank, world, comm)
        losses = []
        for i, (d, ids, y) in enumerate(batches):
            eng.load_batch(d.to(dev), ids.to(dev), y.to(dev))
            if name == "p2p" and i == 1:
                eng.capture()                     # eager step + capture of the whole P2P step (flag waits included) into a CUDA graph
            else:
                eng.train_step()
            losses.append(eng.loss_value())
        torch.cuda.synchronize()
        rows = {t: gathered_rows(eng, t, probe, dev) for t in (0, 1, 3, 25)}
        total = torch.tensor([float(sum(tb.size() for tb in eng.tables.values()))], device=dev)
        dist.all_reduce(total)
        ovf = sum(tb.overflowed() for tb in eng.tables.values())
        results[name] = (losses, eng.params.clone(), rows, int(total.item()), ovf)
        dist.barrier()
    (l1, p1, r1, n1, o1), (l2, p2, r2, n2, o2) = results["p2p"], results["nccl"]
    assert o1 == 0 and o2 == 0, (o1, o2)
    for a, b in zip(l1, l2):
        assert abs(a - b) < 2e-3 * max(1.0, abs(b)), (l1, l2)
    assert (p1 - p2).abs().max().item() < 2e-3, (p1 - p2).abs().max().item()
    assert n1 == n2, ("distinct keys", n1, n2)
    for t in r1:
        (ra, fa, ca), (rb, fb, cb) = r1[t], r2[t]
        assert torch.equal(ca, cb) and float(ca.max()) <= 1.0, f"table {t}: key ownership differs"
        assert torch.equal(fa, fb), f"table {t}: frequencies differ (occurrence counts must survive the dedup)"
        assert (ra - rb).abs().max().item() < 2e-3, (t, (ra - rb).abs().max().item())
    # dense replicas stay bitwise identical across ranks (fixed summation order)
    ref = p1.clone()
    dist.broadcast(ref, 0)
    assert torch.equal(ref, p1), "dense parameters diverged across ranks"
    if rank == 0:
        print(f"MP_CHECK_OK world={world} optimizer={optimizer} losses={['%.4f' % x for x in l1]} distinct_keys={n1}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main(*sys.argv[1:2])
