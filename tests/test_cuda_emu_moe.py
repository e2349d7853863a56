"""MMoE / PLE expert mixtures on the CPU tier: the grouped GEMM stand-ins and the mixture kernels (csrc/cuda/moe_kernels.cu) on the CUDA-on-CPU
emulation against per-group calls and float64, the ops' gradients, the models with ``moe=`` against the plain modules, and engines with two
micro-batches against one batch.  GPU twin: tests/test_gpu_zzzzzzzzzzz_moe.py."""
import pytest
import torch

import moe_cases as K
import pooled_bag_cases as PB
from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(1500)]


@pytest.mark.parametrize("G,M,N,K_", [(1, 1, 64, 80), (3, 129, 64, 136), (5, 127, 192, 80)])
def test_grouped_gemm_stand_in_matches_per_group_calls(G, M, N, K_):
    with _native.cuda_emulation():
        for bias, relu, mask, stats in ((True, True, False, False), (False, False, True, True), (True, False, False, True)):
            K.grouped_tn_case("cpu", G, M, N, K_, bias, relu, mask, stats, seed=G + M)
        K.grouped_dw_case("cpu", G, M, N, K_, seed=G)


def test_grouped_gemm_stand_in_refusals():
    with _native.cuda_emulation():
        K.grouped_refusals("cpu")


@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("select", [K.MMOE_MAP, K.PLE_MAP, ([0, 1], [2, 3, 4, 5, 6, 7, 8, 9]), ([0, 1, 2, 3, 4, 5, 6, 7],)])
def test_mixture_kernels_against_float64(select, H):
    with _native.cuda_emulation():
        a = K.mix_case("cpu", 37, H, select, saturate=True)
        b = K.mix_case("cpu", 37, H, select, saturate=True)
    for u, v in zip(a, b):
        for x, y in zip(u if isinstance(u, list) else [u], v if isinstance(v, list) else [v]):
            assert torch.equal(x, y)


def test_mixture_refusals():
    with _native.cuda_emulation():
        K.mix_refusals("cpu")


@pytest.mark.parametrize("G,shared", [(3, True), (4, False), (13, True), (13, False)])
def test_expert_op_gradients_against_float64(G, shared):
    with _native.cuda_emulation():
        K.expert_grad_case("cpu", 256, G, 20, (24, 16), shared=shared)


@pytest.mark.parametrize("name", ["mmoe", "ple"])
def test_model_with_moe_ops_matches_the_modules(name):
    with _native.cuda_emulation():
        K.model_case(name, torch.device("cpu"), M=16)
    K.model_case(name, torch.device("cpu"), M=16)                     # off the emulation the ops are the torch expression


@pytest.mark.parametrize("name", ["mmoe", "ple"])
def test_two_micro_batches_match_one_batch(name):
    # engine against its torch replica and the export on both Processors, on these fused paths: test_cuda_emu_pooled_bags.py and
    # test_cuda_emu_engine_export.py (their mmoe / ple cases)
    dev = torch.device("cpu")
    with _native.cuda_emulation():
        a = PB.seq_engine(name, dev, 16, learning_rate=0.05)
        b = PB.seq_engine(name, dev, 16, learning_rate=0.05, micro_batch_num=2)
        bt = PB.taobao_like(16, 300)
        for e in (a, b):
            e.load_batch(*PB.engine_inputs(e, bt, dev))
            e.train_step()
        assert abs(a.loss_value() - b.loss_value()) < 0.03 * max(1.0, abs(a.loss_value()))
        for (n, p), q in zip(a.net.inner.named_parameters(), b.net.inner.parameters()):
            assert float((p - q).abs().max()) < 0.05, n
