"""torchrun --nproc-per-node 2 tests/mp_linear_group.py: FusedRecEngine(linear=True) (Wide & Deep) at world 2 over NVLink peer memory.  Run by
test_gpu_linear_group.py::test_wdl_engine_world2."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import linear_group_cases as K  # noqa: E402


def main():
    rank, W = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    from deeprec_b200.checkpoint.engine_ckpt import sp_owner
    from deeprec_b200.parallel.p2p import P2PComm
    comm = P2PComm(rank, W, dev)
    B = 1024
    eng = K.wdl_engine(dev, B, learning_rate=0.05, linear_optimizer="ftrl", linear_learning_rate=0.2, rank=rank, world_size=W, comm=comm)
    losses = []
    for s in range(6):
        ids, y, dense = K.engine_batch(B, 1300 + 10 * s + rank)
        eng.load_batch(ids.to(dev), y.to(dev), {k: v.to(dev) for k, v in dense.items()})
        if s == 0:
            eng.capture(warmup=1)
        else:
            eng.train_step()
        losses.append(eng.loss_value())
        if s == 3:
            p = eng.predict()
            assert p.shape == (B,) and bool(((p >= 0) & (p <= 1)).all())
    torch.cuda.synchronize()
    params = [torch.empty_like(eng.params) for _ in range(W)]
    dist.all_gather(params, eng.params)
    assert torch.equal(params[0], params[1]), "dense replicas diverged"
    lt = torch.tensor(losses, device=dev)
    lts = [torch.empty_like(lt) for _ in range(W)]
    dist.all_gather(lts, lt)
    assert torch.equal(lts[0], lts[1]), "global loss differs between ranks"
    for t in range(26):
        keys = torch.arange(K.CARDS[t], device=dev)
        f = eng.lin_tables[t].get_freq(keys).to(dev)
        fs = [torch.empty_like(f) for _ in range(W)]
        dist.all_gather(fs, f)
        freq = torch.stack(fs)
        assert int(((freq > 0).sum(0) > 1).sum()) == 0, t
        mine = (sp_owner(keys.cpu(), W) == rank).to(dev)
        assert bool((f[~mine] == 0).all()), t
    dist.barrier()
    if rank == 0:
        print("linear group mp ok", losses)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
