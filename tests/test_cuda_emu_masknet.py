"""MaskNet (zoo.MaskBlockNet, nn.FusedMaskBlock) on the CPU tier: the model against a float64 transcription of the reference, the MaskBlock
kernels on the CUDA-on-CPU emulation against float64, the engine against a torch replica, and the export served by both Processors.
GPU twin: tests/test_gpu_zzzzzzzzzz_masknet.py."""
import os

import pytest
import torch

import masknet_cases as K
from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(1500)]


@pytest.mark.parametrize("mode", ["parallel", "serial"])
def test_model_matches_the_reference_in_float64(mode):
    m = K.build(f"masknet_{mode}").double()
    widths = [(b.fc1.weight.shape, b.fc2.weight.shape, b.fc3.weight.shape) for b in m.blocks]
    assert len(widths) == 5 and widths[0] == ((429, 429), (429, 429), (64, 429))
    if mode == "serial":
        assert all(w == ((64, 429), (64, 64), (64, 64)) for w in widths[1:])
    g = torch.Generator().manual_seed(3)
    dense, embs = torch.rand(32, 13, generator=g).double(), torch.randn(32, 26, 16, generator=g).double()
    got = m.logits(dense, embs)
    assert torch.allclose(got, K.reference_logits(m, dense, embs), rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("N", K.SIMT_N)
@pytest.mark.parametrize("M", K.SIMT_M)
def test_ln_relu_bwd_against_float64(M, N):
    with _native.cuda_emulation():
        K.ln_relu_bwd_case("cpu", M, N)


@pytest.mark.parametrize("N", K.SIMT_N)
@pytest.mark.parametrize("M", K.SIMT_M)
def test_bn_apply_mul_and_backward_against_float64(M, N):
    with _native.cuda_emulation():
        K.bn_mul_case("cpu", M, N)


@pytest.mark.parametrize("M,N,K_,bias,relu,pad", [(1, 16, 8, True, True, 0), (37, 64, 432, False, True, 8), (130, 128, 40, True, False, 0),
                                                  (9, 48, 520, False, False, 16)])
def test_gemm_ln_stand_in_against_float64(M, N, K_, bias, relu, pad):
    with _native.cuda_emulation():
        K.gemm_ln_case("cpu", M, N, K_, bias, relu, pad)


def test_gemm_ln_stand_in_refusals():
    with _native.cuda_emulation():
        K.gemm_ln_refusals("cpu")


@pytest.mark.parametrize("same", [False, True])
def test_op_gradients_on_the_emulation(same):
    with _native.cuda_emulation():
        K.op_grad_case("cpu", 40, 52, 52 if same else 24, 16, same_input=same)


@pytest.mark.parametrize("mode", ["parallel", "serial"])
def test_engine_on_the_emulation_matches_a_torch_replica(mode):
    B = 32
    batches = [K.batch(B, 100 + s) for s in range(3)]
    with _native.cuda_emulation():
        eng = K.make_engine(f"masknet_{mode}", B, num_blocks=2)          # two blocks: x shared by both (parallel), 429 -> 64 wide (serial)
        start = {k: v.detach().clone() for k, v in eng.net.inner.state_dict().items()}
        tables = K.replica_tables(eng)
        le = []
        for ids, y, dense in batches:
            eng.load_batch(ids, y, dense)
            eng.train_step()
            le.append(eng.loss_value())
    import copy
    ref_net = copy.deepcopy(eng.net.inner)
    ref_net.load_state_dict(start)
    lr_, net = K.replica_step_losses(ref_net, tables, batches)
    for a, b in zip(le, lr_):
        assert abs(a - b) < 0.03 * max(1.0, abs(b)), (le, lr_)
    for (n, p), q in zip(eng.net.inner.named_parameters(), net.parameters()):          # as the DeepFM replica bounds its embedding rows
        assert (p.detach().float() - q.detach()).abs().max().item() < 0.05, n


@pytest.mark.parametrize("mode", ["parallel", "serial"])
def test_engine_export_serves_on_both_processors(tmp_path, mode):
    import engine_export_cases as E
    from deeprec_b200.serving import Processor, export_engine_program
    B = 32
    with _native.cuda_emulation():
        eng = K.make_engine(f"masknet_{mode}", B, num_blocks=2)
        for s in range(3):
            ids, y, dense = K.batch(B, 10 + s)
            eng.load_batch(ids, y, dense)
            eng.train_step()
        tabs = E.engine_tables(eng)
        emb = torch.stack([E.lookup(tabs[t], ids[t]) for t in range(26)], 1)
        export_engine_program(eng, str(tmp_path / "v"), root=str(tmp_path))
    import copy
    net = copy.deepcopy(eng.net.inner).float().eval()
    ref = torch.sigmoid(net.logits(dense["dense"], emb)).detach().numpy()
    for dev, tol in (("cpu", 1e-4), ("cuda_emu", 3e-2)):
        p = Processor(str(tmp_path / "v"), {"session_num": 1, "max_batch": 24, "model_update_interval_ms": 0}, device=dev)
        try:
            assert E.max_err(p.predict(*E.request("deepfm", dense["dense"], ids)), ref) < tol, dev
        finally:
            p.close()
