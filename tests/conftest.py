import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with `pytest -m gpu`")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no GPU in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


_MULTIPROCESS_TESTS = ("test_ps_cpu.py", "test_collective_cpu.py", "test_sok_elastic_cpu.py", "test_health.py", "test_examples.py",
                       "test_work_queue_shared_between_processes")


@pytest.fixture(autouse=True)
def _few_threads_for_multiprocess_tests(request, monkeypatch):
    """Tests that spawn several worker processes (PS roles, gloo ranks, example scripts): give every child 2 OpenMP threads instead of one
    per core each -- N processes x all cores of spin-waiting OpenMP workers on a small shared box is what made them time out
    (torchrun sets OMP_NUM_THREADS=1 for the same reason).  Children inherit the environment at spawn time."""
    node = request.node.nodeid
    if any(tag in node for tag in _MULTIPROCESS_TESTS):
        monkeypatch.setenv("OMP_NUM_THREADS", "2")
        monkeypatch.setenv("DEEPREC_HOST_THREADS", "2")
    yield
