"""GPU: the multi-head self-attention kernels (csrc/cuda/mha_kernels.cu) against the float64 oracle of tests/mha_cases.py for (heads, dh) =
(4, 8), (2, 16), (1, 32), S = 1, 2, 17, 51, 64, 65, 128, B = 1, 3, 4099 and four key masks, into NaN-filled buffers; nn.fused_encoder_layer
against fp32 nn.TransformerEncoderLayer autograd; unsupported layers and shapes; bit-identical results across runs and graph replay; BST on
FusedRecEngine against a torch replica, eager and captured, bit-identical across engines and graph replay; the training CLI with --model bst
--engine."""
import os
import subprocess
import sys

import pytest
import torch

import mha_cases as M

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("kind", M.MASKS)
@pytest.mark.parametrize("S", [1, 2, 17, 51, 64, 65, 128])
@pytest.mark.parametrize("heads,dh", [(4, 8), (2, 16), (1, 32)])
def test_kernels_match_the_float64_oracle(heads, dh, S, kind):
    for B in (1, 3, 4099):
        M.check_kernels(B, S, heads, dh, kind, DEV)


@pytest.mark.parametrize("B,S,E,heads", [(300, 21, 32, 4), (64, 51, 32, 2), (40, 65, 32, 1), (17, 128, 64, 4)])
def test_fused_encoder_layer_matches_the_module(B, S, E, heads):
    M.layer_vs_module(B, S, E, heads, DEV)


def test_unsupported_layers_and_shapes_raise():
    from deeprec_b200 import _native
    from deeprec_b200._native import ptr, stream_ptr
    from deeprec_b200.nn import fused_encoder_layer
    x = torch.randn(4, 9, 48, device=DEV)
    valid = torch.ones(4, 9, dtype=torch.bool, device=DEV)
    with pytest.raises(ValueError, match="head size 12"):
        fused_encoder_layer(x, M.encoder_layer(48, 4, DEV), valid)
    x = torch.randn(2, 129, 32, device=DEV)
    with pytest.raises(ValueError, match="S = 129"):
        fused_encoder_layer(x, M.encoder_layer(32, 4, DEV), torch.ones(2, 129, dtype=torch.bool, device=DEV))
    x = torch.randn(4, 9, 32, device=DEV)
    valid = torch.ones(4, 9, dtype=torch.bool, device=DEV)
    with pytest.raises(ValueError, match="post-norm"):
        fused_encoder_layer(x, M.encoder_layer(32, 4, DEV, norm_first=True), valid)
    with pytest.raises(ValueError, match="ReLU"):
        fused_encoder_layer(x, M.encoder_layer(32, 4, DEV, activation="gelu"), valid)
    with pytest.raises(ValueError, match="dropout"):
        fused_encoder_layer(x, torch.nn.TransformerEncoderLayer(32, 4, 128, dropout=0.1, batch_first=True, device=DEV), valid)
    lib = _native.cuda()
    for B, S, E, heads in ((4, 9, 48, 4), (2, 129, 32, 4)):
        qkv, do = M.make_case(B, S, heads, E // heads, 0, DEV)
        v = torch.ones(B, S, dtype=torch.uint8, device=DEV)
        o = torch.empty(B * S, E, dtype=torch.bfloat16, device=DEV)
        assert lib.dr_cuda_mha_fwd(ptr(qkv), ptr(v), B, S, E, heads, ptr(o), stream_ptr()) == -2
        assert lib.dr_cuda_mha_bwd(ptr(qkv), ptr(v), ptr(o), ptr(do), B, S, E, heads, ptr(qkv), stream_ptr()) == -2


def test_kernels_are_bit_identical_across_runs_and_graph_replay():
    B, S, heads, dh = 4099, 51, 4, 8
    valid = M.make_valid("random", B, S, 5).to(DEV)
    qkv, do = M.make_case(B, S, heads, dh, 11, DEV)
    a = M.run_kernels(qkv, valid, do, B, S, heads)
    b = M.run_kernels(qkv, valid, do, B, S, heads)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        M.run_kernels(qkv, valid, do, B, S, heads)
        with torch.cuda.graph(g):
            c = M.run_kernels(qkv, valid, do, B, S, heads)
    torch.cuda.current_stream().wait_stream(s)
    for x in c:
        x.fill_(7.0)
    g.replay()                                                           # refills the NaN sentinels, then runs both kernels
    torch.cuda.synchronize()
    for x, y, z in zip(a, b, c):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16)), "two runs differ"
        assert torch.equal(x.view(torch.int16), z.view(torch.int16)), "graph replay differs"


@pytest.mark.parametrize("graph", [False, True])
def test_bst_engine_matches_a_torch_replica(graph):
    M.run_bst_vs_replica(DEV, graph=graph, B=1024, steps=6)


def test_bst_training_is_bit_identical_across_engines_and_graph_replay():
    e1, e2, g1 = M.train_bst(DEV, False), M.train_bst(DEV, False), M.train_bst(DEV, True)
    for other, what in ((e2, "two eager engines differ"), (g1, "graph replay differs from eager steps")):
        assert torch.equal(e1[0], other[0]) and e1[1] == other[1], what
        assert all(torch.equal(x, y) for x, y in zip(e1[2], other[2])), what


def test_train_cli_bst_on_the_engine():
    r = subprocess.run([sys.executable, "-m", "deeprec_b200.models.train", "--model", "bst", "--engine", "--steps", "5", "--batch_size", "4096",
                        "--log_every", "1"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    losses = [float(l.split()[-1]) for l in r.stdout.splitlines() if l.startswith("global_step")]
    assert len(losses) == 5 and all(l == l and abs(l) < 1e6 for l in losses), r.stdout[-2000:]
