"""GPU: the linear (wide) embedding group -- k_sp_linear_fwd / k_sp_linear_bwd against their numpy oracles bit for bit, eager and replayed from
a CUDA graph; FusedRecEngine(linear=True) (Wide & Deep) against a torch replica, eager and graph-captured; bit-identical training across two
engines and between graph replay and eager steps; the WDL training CLI; world 2 (needs two GPUs).  Cases: tests/linear_group_cases.py."""
import os
import subprocess
import sys

import pytest
import torch

import linear_group_cases as K

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("C", [26, 1])
def test_linear_kernels_bit_for_bit(C, graph):
    K.run_kernels_world1(DEV, C, 1000, owner=0x6100 + 2 * C + int(graph), graph=graph)


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("linear_sgd", [False, True], ids=["adagrad", "linear_sgd"])
def test_wdl_engine_matches_a_torch_replica(linear_sgd, graph):
    K.run_engine_vs_replica(DEV, linear_sgd, graph=graph, B=1024, steps=6)


def test_wdl_engine_ftrl_on_the_linear_group():
    K.run_ftrl_one_step(DEV, B=1024)


def _train(graph: bool, steps: int = 6, B: int = 2048):
    eng = K.wdl_engine(DEV, B, learning_rate=0.05, linear_optimizer="ftrl", linear_learning_rate=0.2)
    for s in range(steps):
        ids, y, dense = K.engine_batch(B, 1100 + s)
        eng.load_batch(ids.to(DEV), y.to(DEV), {k: v.to(DEV) for k, v in dense.items()})
        if graph and s == 0:
            eng.capture(warmup=1)
        else:
            eng.train_step()
    torch.cuda.synchronize()
    probe = [torch.arange(c, device=DEV) for c in K.CARDS]
    return (eng.params.clone(), eng.loss.clone(), [eng.lin_tables[t].lookup(probe[t]) for t in range(26)],
            [eng.tables[t].lookup(probe[t]) for t in range(26)])


def _equal(a, b):
    return torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and all(torch.equal(x, y) for x, y in zip(a[2] + a[3], b[2] + b[3]))


def test_wdl_training_is_bit_identical_across_engines_and_graph_replay():
    e1, e2, g1 = _train(False), _train(False), _train(True)
    assert _equal(e1, e2), "two eager engines differ"
    assert _equal(e1, g1), "graph replay differs from eager steps"


def test_wdl_train_cli_on_the_engine():
    r = subprocess.run([sys.executable, "-m", "deeprec_b200.models.train", "--model", "wdl", "--engine", "--steps", "5", "--batch_size", "4096",
                        "--log_every", "1"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    losses = [float(l.split()[-1]) for l in r.stdout.splitlines() if l.startswith("global_step")]
    assert losses and all(l == l and abs(l) < 1e6 for l in losses), r.stdout[-2000:]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_wdl_engine_world2():
    """Two processes over NVLink peer memory (torchrun): identical dense replicas, every linear key on one owner, train -> predict -> train."""
    script = os.path.join(ROOT, "tests", "mp_linear_group.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29561",
                        script], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "linear group mp ok" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
