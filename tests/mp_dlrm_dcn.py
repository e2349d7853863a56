"""Two-GPU DLRM-DCNv2 check (run under torchrun): DLRMEngine(interaction_op="dcnv2") over P2PComm on the two halves of each global batch
against one GPU on the whole batch (computed by rank 0 before the distributed run starts).  Prints MP_DCN_OK on success."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    from dlrm_dcn_cases import batch, small_config
    from deeprec_b200.models.dlrm_engine import DLRMEngine
    from deeprec_b200.parallel.p2p import P2PComm
    steps, GB = 3, 512
    ref = None
    if rank == 0:
        one = DLRMEngine(small_config(batch_size=GB), dev)
        ref = []
        for s in range(steps):
            d, ids, y = batch(GB, 700 + s)
            one.load_batch(d.to(dev), ids.to(dev), y.to(dev)); one.train_step(); ref.append(one.loss_value())
        ref = (ref, one.params.cpu())
        del one
    dist.init_process_group("nccl", device_id=dev)
    B = GB // world
    eng = DLRMEngine(small_config(batch_size=B), dev, rank, world, P2PComm(rank, world, dev))
    losses = []
    for s in range(steps):
        d, ids, y = batch(GB, 700 + s)
        sl = slice(rank * B, rank * B + B)
        eng.load_batch(d[sl].to(dev), ids[:, sl].contiguous().to(dev), y[sl].to(dev)); eng.train_step(); losses.append(eng.loss_value())
    params = eng.params.clone()
    other = params.clone()
    dist.broadcast(other, 0)
    assert torch.equal(params, other), "dense replicas diverged"
    if rank == 0:
        # BatchNorm normalises with each rank's own batch statistics, and the batch sums are ordered differently: close, not bitwise
        for a, b in zip(losses, ref[0]):
            assert abs(a - b) < 1e-3, (losses, ref[0])
        assert (params.cpu() - ref[1]).abs().max().item() < 5e-3
        print("MP_DCN_OK")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
