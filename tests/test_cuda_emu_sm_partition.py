"""DLRMConfig.sparse_sms on the CUDA-on-CPU emulation: the emulated step is eager on one stream, so the SM partition is never made and the
step computes the same bits with or without it."""
import pytest
import torch

from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(900)]
CARDS = [50, 1000, 7, 300] + [97] * 22


def _step(sparse_sms):
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    g = torch.Generator().manual_seed(3)
    B = 128
    dense, ids, y = torch.rand(B, 13, generator=g), torch.stack([torch.randint(0, c, (B,), generator=g) for c in CARDS]), (torch.rand(B, generator=g) < 0.3).float()
    with _native.cuda_emulation():
        eng = DLRMEngine(DLRMConfig(batch_size=B, cardinalities=CARDS, sparse_sms=sparse_sms))
        eng.load_batch(dense, ids, y)
        eng.train_step()
        assert eng.partition_sms is None
        return eng.params.clone(), eng.prob.clone()


def test_sparse_sms_is_a_no_op_on_the_emulation():
    p0, q0 = _step(0)
    p1, q1 = _step(16)
    assert torch.equal(p0, p1) and torch.equal(q0, q1)
