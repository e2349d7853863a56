"""The optimizer kernels on an H100 against the float64 oracle (tests/optim_ref.py); the same cases (tests/optim_cases.py) run on the CUDA-on-
CPU emulation in tests/test_cuda_emu_optimizer_edges.py.  The fused multi-GPU all-reduce + update is checked per optimizer by
tests/test_gpu_multi.py (tests/mp_check.py) on boxes with two or more GPUs."""
import pytest

import optim_cases as K

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dim", K.SPARSE_DIMS)
@pytest.mark.parametrize("rule", list(K.RULES))
def test_sparse_apply_matches_oracle(rule, dim):
    K.sparse_apply_case("cuda", rule, dim)


def test_sparse_apply_claim_overflow():
    K.sparse_overflow_case("cuda")


def test_advance_hyper_beta_powers():
    K.advance_hyper_case("cuda")


def test_adagrad_decay_dense_power_advances_on_device():
    K.adagrad_decay_dense_power_case("cuda")


@pytest.mark.parametrize("variant", K.ACCUMULATE_VARIANTS)
def test_sparse_accumulate_matches_index_add(variant):
    K.sparse_accumulate_case("cuda", variant)


@pytest.mark.parametrize("size", K.DENSE_SIZES)
@pytest.mark.parametrize("rule", list(K.RULES))
def test_dense_apply_matches_oracle(rule, size):
    K.dense_apply_case("cuda", rule, size)


@pytest.mark.parametrize("due", [False, True])
def test_dense_adagrad_decay(due):
    K.dense_apply_case("cuda", "adagraddecay", "257", decay_due=due)


@pytest.mark.parametrize("opt", K.ENGINE_OPTIMIZERS)
def test_engine_update_matches_oracle(opt):
    K.engine_update_case(opt)
