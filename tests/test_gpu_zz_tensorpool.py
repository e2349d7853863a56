"""GPU TensorPool as PyTorch's CUDA allocator (subprocess: the allocator must be installed before the first CUDA allocation)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

SCRIPT = r"""
import torch
from deeprec_b200.utils import memory
memory.enable_gpu_tensorpool()
lin = torch.nn.Linear(512, 512).cuda()
x = torch.randn(4096, 512, device="cuda")
ref = None
for step in range(8):
    y = torch.relu(lin(x)); z = (y * 2).sum(); z.backward()
    torch.cuda.synchronize()
    ref = ref if ref is not None else float(z)
    assert abs(float(z) - ref) < 1e-3 * abs(ref)
    del y, z
    memory.gpu_tensorpool_step()
s = memory.gpu_tensorpool_stats()
assert s["phase"] == 1 and s["pool_hits"] > 0 and s["pool_bytes"] > 0, s
print("TENSORPOOL_OK", s)
"""


def test_gpu_tensorpool_allocator():
    r = subprocess.run([sys.executable, "-c", SCRIPT], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "TENSORPOOL_OK" in r.stdout, r.stdout + r.stderr
