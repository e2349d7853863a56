"""GPU: k_sp_segsum bit for bit against the numpy model of its semantics (tests/segsum_cases.py) -- one key, distinct keys, a power-law
stream with padding, a key hot across blocks, saturation at +-2^22, dims 8 / 16 / 64 / 128, B not a multiple of 32 or 256 -- on a grid
sized to every SM and on one sized to an 8-SM partition (the per-key sums must not depend on the grid)."""
import pytest
import torch

from segsum_cases import cases, check

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,ids,demb", cases(small=False), ids=[c[0] for c in cases(small=False)])
@pytest.mark.parametrize("grid_sms", [0, 8])
def test_segsum_matches_the_model_bit_for_bit(name, ids, demb, grid_sms):
    from deeprec_b200 import _native
    from deeprec_b200.parallel.sparse_pipeline import SparsePipeline
    dev = torch.device("cuda", 0)
    C, B = ids.shape
    sp = SparsePipeline(dev, 0, 1, list(range(C)), C, B, demb.shape[2])
    lib = _native.cuda()
    lib.dr_cuda_set_sparse_sms(grid_sms)
    try:
        check(sp, ids.to(dev), demb.to(dev), torch.cuda.synchronize)
    finally:
        lib.dr_cuda_set_sparse_sms(0)
