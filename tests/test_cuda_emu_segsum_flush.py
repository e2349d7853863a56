"""k_sp_segsum bit for bit against the numpy model of its semantics (tests/segsum_cases.py) on the CUDA-on-CPU emulation: the CPU twin of
test_gpu_segsum_flush.py, at emulation sizes."""
import pytest
import torch

from deeprec_b200 import _native
from segsum_cases import cases, check

pytestmark = [pytest.mark.timeout(900)]


@pytest.mark.parametrize("name,ids,demb", cases(small=True), ids=[c[0] for c in cases(small=True)])
def test_segsum_matches_the_model_bit_for_bit(name, ids, demb):
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
    C, B = ids.shape
    with _native.cuda_emulation():
        sp = SparsePipeline(torch.device("cpu"), 0, 1, list(range(C)), C, B, demb.shape[2])
        check(sp, ids, demb)
