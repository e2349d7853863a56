"""GPU: the GRU recurrence kernels (csrc/cuda/rnn_kernels.cu) against the float64 oracle of tests/gru_cases.py for H = 32, 64, L = 1, 2, 20,
50, B = 1, 15, 16, 17, 4099 and full / one / zero / random lengths, into NaN-filled buffers; nn.fused_gru against fp32 nn.GRU autograd; an
unsupported hidden size; bit-identical results across runs and graph replay; DIEN on FusedRecEngine against a torch replica, eager and
captured, bit-identical across engines and graph replay; the training CLI with --model dien --engine."""
import os
import subprocess
import sys

import pytest
import torch

import gru_cases as G

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("kind", ["full", "one", "zero", "random"])
@pytest.mark.parametrize("L", [1, 2, 20, 50])
@pytest.mark.parametrize("H", [32, 64])
def test_kernels_match_the_float64_oracle(H, L, kind):
    for B in (1, 15, 16, 17, 4099):
        G.check_kernels(B, L, H, kind, DEV)


@pytest.mark.parametrize("I,H", [(32, 32), (32, 64), (20, 16)])
def test_fused_gru_matches_nn_gru(I, H):
    G.op_vs_module(300, 20, I, H, DEV)


def test_unsupported_hidden_size_raises():
    from deeprec_b200 import _native
    from deeprec_b200._native import ptr, stream_ptr
    from deeprec_b200.nn import fused_gru
    gru = torch.nn.GRU(32, 36, batch_first=True, device=DEV)              # the reference's DIEN hidden size
    with pytest.raises(ValueError, match="hidden size 36"):
        fused_gru(torch.randn(4, 5, 32, device=DEV), gru, torch.full((4,), 5, device=DEV))
    gi, w, b, _ = G.make_case(4, 5, 32, 0, DEV)
    ln = torch.full((4,), 5, dtype=torch.int32, device=DEV)
    y = torch.empty(4, 5, 36, device=DEV)
    assert _native.cuda().dr_cuda_gru_fwd(ptr(gi), ptr(w), ptr(b), ptr(ln), 4, 5, 36, ptr(y), stream_ptr()) != 0
    with pytest.raises(ValueError, match="single-layer"):
        fused_gru(torch.randn(4, 5, 32, device=DEV), torch.nn.GRU(32, 32, num_layers=2, batch_first=True, device=DEV), ln)


def test_kernels_are_bit_identical_across_runs_and_graph_replay():
    B, L, H = 4099, 50, 32
    lengths = G.make_lengths("random", B, L, 5).to(DEV)
    inputs, a = G.run_kernels(B, L, H, lengths, 11, DEV)
    _, b = G.run_kernels(B, L, H, lengths, 11, DEV, inputs)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        G.run_kernels(B, L, H, lengths, 11, DEV, inputs)                 # warm-up outside capture (workspaces of the dW GEMM / column sums)
        with torch.cuda.graph(g):
            _, c = G.run_kernels(B, L, H, lengths, 11, DEV, inputs)
    torch.cuda.current_stream().wait_stream(s)
    for x in c:
        x.fill_(7.0)
    g.replay()                                                           # refills the NaN sentinels and zeros, then runs both kernels
    torch.cuda.synchronize()
    bits = lambda t: t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)
    for x, y, z in zip(a, b, c):
        assert torch.equal(bits(x), bits(y)), "two runs differ"
        assert torch.equal(bits(x), bits(z)), "graph replay differs"


@pytest.mark.parametrize("graph", [False, True])
def test_dien_engine_matches_a_torch_replica(graph):
    G.run_dien_vs_replica(DEV, graph=graph, B=1024, steps=6)


def test_dien_training_is_bit_identical_across_engines_and_graph_replay():
    e1, e2, g1 = G.train_dien(DEV, False), G.train_dien(DEV, False), G.train_dien(DEV, True)
    for other, what in ((e2, "two eager engines differ"), (g1, "graph replay differs from eager steps")):
        assert torch.equal(e1[0], other[0]) and e1[1] == other[1], what
        assert all(torch.equal(x, y) for x, y in zip(e1[2], other[2])), what


def test_train_cli_dien_on_the_engine():
    r = subprocess.run([sys.executable, "-m", "deeprec_b200.models.train", "--model", "dien", "--engine", "--steps", "5", "--batch_size", "4096",
                        "--log_every", "1"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    losses = [float(l.split()[-1]) for l in r.stdout.splitlines() if l.startswith("global_step")]
    assert len(losses) == 5 and all(l == l and abs(l) < 1e6 for l in losses), r.stdout[-2000:]
