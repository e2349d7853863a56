"""GPU: multi-hot bags -- k_sp_pool / k_sp_pool_segsum against their oracles for sum, mean and sqrtn, eager and replayed from a CUDA graph;
pooled_seq_engine (DSSM sum / mean, ESMM, MMoE) against a torch replica, eager and graph-captured; bit-identical training across two engines
and between graph replay and eager steps; the training CLI for DSSM and ESMM.  Cases: tests/pooled_bag_cases.py."""
import os
import subprocess
import sys

import pytest
import torch

import pooled_bag_cases as K

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMBS = ["sum", "mean", "sqrtn"]


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("comb", COMBS)
def test_pool_kernels(comb, graph):
    K.run_kernels_world1(DEV, comb, 2000, owner=0x8100 + 2 * COMBS.index(comb) + int(graph), graph=graph)


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("name,comb", [("dssm", "sum"), ("dssm", "mean"), ("esmm", "sum"), ("mmoe", "sum")])
def test_engine_matches_a_torch_replica(name, comb, graph):
    K.run_engine_vs_replica(name, DEV, comb, graph=graph, B=1024, steps=6)


def _train(graph: bool, steps: int = 6, B: int = 2048):
    eng = K.seq_engine("esmm", DEV, B, "sqrtn", learning_rate=0.05)
    for s in range(steps):
        eng.load_batch(*K.engine_inputs(eng, K.taobao_like(B, 1100 + s), DEV))
        if graph and s == 0:
            eng.capture(warmup=1)
        else:
            eng.train_step()
    torch.cuda.synchronize()
    probe = [torch.arange(c, device=DEV) for c in K.CARDS]
    return eng.params.clone(), eng.loss.clone(), [eng.tables[t].lookup(probe[t]) for t in range(3)]


def test_training_is_bit_identical_across_engines_and_graph_replay():
    eq = lambda a, b: torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and all(torch.equal(x, y) for x, y in zip(a[2], b[2]))
    e1, e2, g1 = _train(False), _train(False), _train(True)
    assert eq(e1, e2), "two eager engines differ"
    assert eq(e1, g1), "graph replay differs from eager steps"


@pytest.mark.parametrize("model", ["dssm", "esmm"])
def test_train_cli_on_the_engine(model):
    r = subprocess.run([sys.executable, "-m", "deeprec_b200.models.train", "--model", model, "--engine", "--steps", "5", "--batch_size", "4096",
                        "--log_every", "1"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    losses = [float(l.split()[-1]) for l in r.stdout.splitlines() if l.startswith("global_step")]
    assert len(losses) == 5 and all(l == l and abs(l) < 1e6 for l in losses), r.stdout[-2000:]
