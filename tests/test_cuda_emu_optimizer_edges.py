"""The optimizer kernels on the CUDA-on-CPU emulation against the float64 oracle (tests/optim_ref.py): the sparse row update at every lane
width, the gradient accumulation and its combining cache, the dense update, the fused all-reduce + update with 2 and 3 ranks as threads, and
the update inside a DLRMEngine step for every optimizer at world 1 and 2.  The same cases (tests/optim_cases.py) run on an H100 in
tests/test_gpu_optimizer_edges.py."""
import pytest

import optim_cases as K
from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(1500)]


@pytest.mark.parametrize("dim", K.SPARSE_DIMS)
@pytest.mark.parametrize("rule", list(K.RULES))
def test_sparse_apply_matches_oracle(rule, dim):
    with _native.cuda_emulation():
        K.sparse_apply_case("cpu", rule, dim)


def test_sparse_apply_claim_overflow():
    with _native.cuda_emulation():
        K.sparse_overflow_case("cpu")


def test_advance_hyper_beta_powers():
    with _native.cuda_emulation():
        K.advance_hyper_case("cpu")


def test_adagrad_decay_dense_power_advances_on_device():
    with _native.cuda_emulation():
        K.adagrad_decay_dense_power_case("cpu")


@pytest.mark.parametrize("variant", K.ACCUMULATE_VARIANTS)
def test_sparse_accumulate_matches_index_add(variant):
    with _native.cuda_emulation():
        K.sparse_accumulate_case("cpu", variant)


@pytest.mark.parametrize("size", K.DENSE_SIZES)
@pytest.mark.parametrize("rule", list(K.RULES))
def test_dense_apply_matches_oracle(rule, size):
    with _native.cuda_emulation():
        K.dense_apply_case("cpu", rule, size)


@pytest.mark.parametrize("due", [False, True])
def test_dense_adagrad_decay(due):
    with _native.cuda_emulation():
        K.dense_apply_case("cpu", "adagraddecay", "257", decay_due=due)


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("rule", list(K.RULES))
def test_fused_allreduce_apply_matches_oracle(rule, W):
    K.fused_allreduce_case(rule, W)


@pytest.mark.parametrize("opt", K.ENGINE_OPTIMIZERS)
def test_engine_update_matches_oracle(opt):
    with _native.cuda_emulation():
        K.engine_update_case(opt)


@pytest.mark.parametrize("opt", ["adagrad", "adagraddecay", "adam", "ftrl"])
def test_engine_world2_dense_update_matches_oracle(opt):
    K.engine_world2_case(opt)


@pytest.mark.parametrize("lr_power", [-0.5, -0.25])
def test_framework_dense_ftrl_matches_apply_ftrl_v2(lr_power):
    """FtrlOptimizer on a plain dense parameter (torch ops, no kernel) follows ApplyFtrlV2: the shrinkage gradient enters `linear`, the
    raw gradient the accumulator."""
    import torch
    import optim_ref as R
    from deeprec_b200.optim import FtrlOptimizer, GlobalStep
    g = torch.Generator().manual_seed(3)
    p = torch.nn.Parameter(torch.randn(4096, generator=g) * 0.5)
    opt = FtrlOptimizer([p], None, lr=0.05, learning_rate_power=lr_power, initial_accumulator_value=0.1, l1_regularization_strength=0.05,
                        l2_regularization_strength=0.02, l2_shrinkage_regularization_strength=0.1, global_step=GlobalStep())
    for step in range(3):
        st = opt.state[p]
        w0 = p.detach().clone()
        a0 = st["accum"].clone() if st else torch.full_like(w0, 0.1)
        l0 = st["linear"].clone() if st else torch.zeros_like(w0)
        p.grad = torch.randn(4096, generator=g) * 10.0 ** (torch.rand(4096, generator=g) * 3 - 2.5)
        opt.step()
        ref = R.ftrl_dense(w0.double(), a0.double(), l0.double(), p.grad.double(), 0.05, 0.05, 0.02, 0.1, lr_power)
        K.check(f"step {step} w", p.detach(), ref[0])
        K.check(f"step {step} accum", opt.state[p]["accum"], ref[1])
        K.check(f"step {step} linear", opt.state[p]["linear"], ref[2])
