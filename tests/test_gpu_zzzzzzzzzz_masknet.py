"""MaskNet on the H100: the LayerNorm GEMM epilogue (dr_cuda_gemm_tn_ln) and the MaskBlock SIMT kernels against float64, the op's gradients,
bitwise repeatability of the op and of engines (eager and graph replay), engine training against its torch replica, the export on the GPU
Processor, and the train CLI.  CPU twin: tests/test_cuda_emu_masknet.py."""
import copy
import os
import subprocess
import sys

import pytest
import torch

import masknet_cases as K

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("K_", [8, 432, 520])
@pytest.mark.parametrize("N", [16, 48, 64, 128])
@pytest.mark.parametrize("M", [1, 127, 129, 4099])
def test_gemm_ln_against_float64(M, N, K_):
    for bias, relu, pad in ((True, True, 0), (False, False, 8), (True, False, 24), (False, True, 0)):
        K.gemm_ln_case("cuda", M, N, K_, bias, relu, pad, seed=M + N + K_)


def test_gemm_ln_refusals():
    K.gemm_ln_refusals("cuda")


@pytest.mark.parametrize("N", K.SIMT_N)
@pytest.mark.parametrize("M", K.SIMT_M + [65536])
def test_simt_kernels_against_float64(M, N):
    K.ln_relu_bwd_case("cuda", M, N)
    K.bn_mul_case("cuda", M, N)


@pytest.mark.parametrize("E,H,same", [(429, 429, True), (429, 64, False)])
def test_op_gradients_and_repeatability(E, H, same):
    a = K.op_grad_case("cuda", 1024, E, H, 64, same_input=same)
    b = K.op_grad_case("cuda", 1024, E, H, 64, same_input=same)
    assert torch.equal(a[0], b[0])
    for n in a[1]:
        assert torch.equal(a[1][n], b[1][n]), n


def test_op_refuses_wide_blocks():
    from deeprec_b200.nn import FusedMaskBlock
    blk = FusedMaskBlock(32, 32, 136).cuda()
    x = torch.randn(8, 32, device="cuda")
    with pytest.raises(ValueError):
        blk(x, x)


def _params(eng):
    return {k: v.detach().clone() for k, v in eng.net.inner.state_dict().items()}


@pytest.mark.parametrize("mode", ["parallel", "serial"])
def test_engines_are_bitwise_repeatable_eager_and_replayed(mode):
    B = 512
    batches = [K.batch(B, 50 + s) for s in range(3)]
    outs = []
    for graph in (False, False, True, True):                          # capture(): three eager warm-up steps that train, then replays
        eng = K.make_engine(f"masknet_{mode}", B, dev=torch.device("cuda", 0))
        for i, (ids, y, dense) in enumerate(batches):
            eng.load_batch(ids.cuda(), y.cuda(), {"dense": dense["dense"].cuda()})
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


@pytest.mark.parametrize("mode", ["parallel", "serial"])
def test_engine_matches_its_torch_replica_and_learns(mode):
    B = 1024
    dev = torch.device("cuda", 0)
    batches = [K.batch(B, 100 + s) for s in range(3)]
    eng = K.make_engine(f"masknet_{mode}", B, dev=dev)
    start = copy.deepcopy(eng.net.inner).cpu()
    tables = K.replica_tables(eng)
    le = []
    for ids, y, dense in batches:
        eng.load_batch(ids.cuda(), y.cuda(), {"dense": dense["dense"].cuda()})
        eng.train_step()
        le.append(eng.loss_value())
    os.environ["DEEPREC_FUSED_NN"] = "0"
    try:
        lr_, _ = K.replica_step_losses(start.float(), tables, batches)
    finally:
        del os.environ["DEEPREC_FUSED_NN"]
    for a, b in zip(le, lr_):
        assert abs(a - b) < 0.03 * max(1.0, abs(b)), (le, lr_)
    # a learnable signal: the loss falls
    eng = K.make_engine(f"masknet_{mode}", B, dev=dev)
    losses = []
    for s in range(30):
        ids, y, dense = K.batch(B, 1000 + s, learnable=True)
        eng.load_batch(ids.cuda(), y.cuda(), {"dense": dense["dense"].cuda()})
        eng.train_step()
        losses.append(eng.loss_value())
    assert sum(losses[-5:]) / 5 < 0.92 * sum(losses[:5]) / 5, losses


@pytest.mark.parametrize("mode", ["parallel", "serial"])
def test_engine_export_on_the_gpu_processor(tmp_path, mode):
    import engine_export_cases as E
    from deeprec_b200.serving import Processor, export_engine_program
    B = 1024
    eng = K.make_engine(f"masknet_{mode}", B, dev=torch.device("cuda", 0))
    for s in range(3):
        ids, y, dense = K.batch(B, 10 + s)
        eng.load_batch(ids.cuda(), y.cuda(), {"dense": dense["dense"].cuda()})
        eng.train_step()
    tabs = E.engine_tables(eng)
    emb = torch.stack([E.lookup(tabs[t], ids[t]) for t in range(26)], 1)
    export_engine_program(eng, str(tmp_path / "v"), root=str(tmp_path))
    net = copy.deepcopy(eng.net.inner).float().cpu().eval()
    ref = torch.sigmoid(net.logits(dense["dense"], emb)).detach().numpy()
    p = Processor(str(tmp_path / "v"), {"session_num": 2, "max_batch": 512, "model_update_interval_ms": 0}, device="cuda")
    try:
        assert E.max_err(p.predict(*E.request("deepfm", dense["dense"], ids)), ref) < 3e-2
    finally:
        p.close()


def test_train_cli_smoke():
    r = subprocess.run([sys.executable, "-m", "deeprec_b200.models.train", "--model", "masknet_parallel", "--engine", "--steps", "4",
                        "--batch_size", "1024", "--log_every", "1"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "nan" not in (r.stdout + r.stderr).lower()
