"""Multi-GPU tests: launched as torchrun subprocesses when the box has >= 2 GPUs."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(n, optimizer="adagrad"):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tests", "mp_check.py"), optimizer]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "MP_CHECK_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("optimizer", ["adagrad", "adam", "ftrl"])
def test_p2p_matches_nccl_2gpu(optimizer):
    """The fused P2P / NVLS all-reduce + dense update against the NCCL arm's all-reduce + dr_cuda_dense_apply, per optimizer."""
    _run(2, optimizer)


@pytest.mark.skipif(torch.cuda.device_count() < 8, reason="needs 8 GPUs")
def test_p2p_matches_nccl_8gpu():
    _run(8)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_checkpoint_restores_under_another_world_size(tmp_path):
    """A checkpoint written by 2 ranks (hash(key) % 2 shards) restores into a 1-rank engine: every key lands on its new owner with its
    row, optimizer slot, frequency; the dense block comes back bit-exact (N -> M re-sharding, embedding_var_restore.cc)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29534",
           os.path.join(ROOT, "tests", "mp_ckpt.py"), str(tmp_path)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "MP_CKPT_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    exp = torch.load(os.path.join(str(tmp_path), "expect.pt"))
    cards = [50, 1000, 7, 300] + [97] * 21 + [200000]
    eng = DLRMEngine(DLRMConfig(batch_size=1024, cardinalities=cards, learning_rate=0.05))
    assert eng.restore(os.path.join(str(tmp_path), "dlrm")) == exp["step"] == 3
    assert torch.equal(eng.params.cpu(), exp["params"])
    probe = torch.arange(0, 300, device="cuda")
    for t, (rows, freq, cnt) in exp["rows"].items():
        f = eng.tables[t].get_freq(probe).float().cpu()
        assert torch.equal(f, freq), t
        got = eng.tables[t].lookup(probe).cpu() * (f > 0).float()[:, None]
        assert torch.allclose(got, rows, atol=1e-6), t


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_tiered_tables_under_model_parallelism_2gpu():
    """FusedRecEngine(tiered=...) at world 2: every rank keeps a 1024-row HBM cache over its own DRAM tier for the keys it owns; the owners find
    their keys in both ranks' next batches over peer memory (tier_kernels.cu: k_tier_miss_list_mp).  Same losses / rows as single-tier tables.
    CPU twin with ranks as threads: tests/test_cuda_emu_tier.py::test_owner_side_promotion_with_ranks_as_threads."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29535",
           os.path.join(ROOT, "tests", "mp_tier.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "MP_TIER_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
