"""MMoE / PLE expert mixtures on the H100: the grouped wgmma GEMMs against per-group calls (bit for bit) and float64, the mixture kernels
against float64 and bitwise repeatable, the ops' gradients, the models with ``moe=`` against the plain modules, engines against their torch
replica (eager and replayed, bitwise repeatable), a falling loss, the export on the GPU Processor and the train CLI.
CPU twin: tests/test_cuda_emu_moe.py."""
import copy
import os
import subprocess
import sys

import pytest
import torch

import moe_cases as K
import pooled_bag_cases as PB

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)


@pytest.mark.parametrize("K_", [80, 136])
@pytest.mark.parametrize("N", [64, 192, 256])
@pytest.mark.parametrize("M", [1, 127, 129, 4099])
@pytest.mark.parametrize("G", [1, 3, 5, K.MAX_GROUPS])
def test_grouped_gemms_match_per_group_calls_and_float64(G, M, N, K_):
    for bias, relu, mask, stats in ((True, True, False, False), (False, False, True, True), (True, False, False, True), (False, True, True, False)):
        K.grouped_tn_case("cuda", G, M, N, K_, bias, relu, mask, stats, seed=G + M + N)
    K.grouped_dw_case("cuda", G, M, N, K_, seed=G + M)


def test_grouped_gemm_refusals():
    K.grouped_refusals("cuda")


@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("select", [K.MMOE_MAP, K.PLE_MAP, ([0, 1], [2, 3, 4, 5, 6, 7, 8, 9]), ([0, 1, 2, 3, 4, 5, 6, 7],)])
@pytest.mark.parametrize("M", [1, 300, 65536])
def test_mixture_kernels_against_float64_and_repeatable(M, select, H):
    a = K.mix_case("cuda", M, H, select, saturate=True)
    b = K.mix_case("cuda", M, H, select, saturate=True)
    for u, v in zip(a, b):
        for x, y in zip(u if isinstance(u, list) else [u], v if isinstance(v, list) else [v]):
            assert torch.equal(x, y)


def test_mixture_refusals():
    K.mix_refusals("cuda")


@pytest.mark.parametrize("G,shared", [(3, True), (4, False), (5, False), (13, True), (13, False)])
def test_expert_op_gradients_against_float64_and_repeatable(G, shared):
    a = K.expert_grad_case("cuda", 1024, G, 80, (256, 192, 128, 64), shared=shared)
    b = K.expert_grad_case("cuda", 1024, G, 80, (256, 192, 128, 64), shared=shared)
    assert torch.equal(a[0], b[0]) and all(torch.equal(x, y) for x, y in zip(a[1], b[1]))


@pytest.mark.parametrize("name", ["mmoe", "ple"])
def test_model_with_moe_ops_matches_the_modules(name):
    K.model_case(name, DEV, M=512)


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("name", ["mmoe", "ple"])
def test_engine_matches_its_torch_replica(name, graph):
    PB.run_engine_vs_replica(name, DEV, graph=graph, steps=5, B=512)


def _params(eng):
    return {k: v.detach().clone() for k, v in eng.net.inner.state_dict().items()}


@pytest.mark.parametrize("name", ["mmoe", "ple"])
def test_engines_are_bitwise_repeatable_eager_and_replayed(name):
    B = 1024
    batches = [PB.taobao_like(B, 50 + s) for s in range(3)]
    outs = []
    for graph in (False, False, True, True):                          # capture(): three eager warm-up steps that train, then replays
        eng = PB.seq_engine(name, DEV, B, learning_rate=0.05)
        for i, b in enumerate(batches):
            eng.load_batch(*PB.engine_inputs(eng, b, DEV))
            if i == 0:
                if graph:
                    eng.capture()
                else:
                    for _ in range(3):
                        eng.train_step()
            else:
                eng.train_step()
        torch.cuda.synchronize()
        outs.append(_params(eng))
    for other in outs[1:]:
        for k in outs[0]:
            assert torch.equal(outs[0][k], other[k]), k


@pytest.mark.parametrize("name", ["mmoe", "ple"])
def test_engine_learns_a_signal(name):
    eng = PB.seq_engine(name, DEV, 1024, learning_rate=0.05)
    losses = []
    for s in range(30):
        b = PB.taobao_like(1024, 1000 + s)
        b["labels"] = (b["item"] % 3 == 0).float()                    # a learnable signal: the item id decides the click
        eng.load_batch(*PB.engine_inputs(eng, b, DEV))
        eng.train_step()
        losses.append(eng.loss_value())
    assert sum(losses[-5:]) / 5 < 0.92 * sum(losses[:5]) / 5, losses


@pytest.mark.parametrize("name", ["mmoe", "ple"])
def test_engine_export_on_the_gpu_processor(tmp_path, name):
    import engine_export_cases as E
    from deeprec_b200.serving import Processor, export_engine_program
    eng = E.make_engine(name, DEV, 512)
    dense, ids = E.train(eng, name, 512, 3, 10)
    ref = E.oracle(eng, name, dense, ids)
    export_engine_program(eng, str(tmp_path / "v"), root=str(tmp_path))
    p = Processor(str(tmp_path / "v"), {"session_num": 2, "max_batch": 256, "model_update_interval_ms": 0}, device="cuda")
    try:
        assert E.max_err(p.predict(*E.request(name, dense, ids)), ref) < 3e-2
    finally:
        p.close()


@pytest.mark.parametrize("name", ["mmoe", "ple"])
def test_train_cli_smoke(name):
    r = subprocess.run([sys.executable, "-m", "deeprec_b200.models.train", "--model", name, "--engine", "--steps", "4", "--batch_size", "1024",
                        "--log_every", "1"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "nan" not in (r.stdout + r.stderr).lower()
