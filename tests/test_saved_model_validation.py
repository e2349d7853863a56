"""Both native Processors refuse the same malformed saved models (csrc/common/saved_model.h): truncated or ragged tensors, a ModelConfig nested
past the JSON reader's depth limit and a delta whose rows do not match its keys.  Every case runs on the CPU runtime and on the GPU runtime
compiled for the host (``cuda_emu``).  The malformed bundles are valid exports rewritten with ``checkpoint.saver``."""
import os
import shutil
import time

import numpy as np
import pytest
import torch

import deeprec_b200 as dr
from deeprec_b200.checkpoint.saver import BundleReader, BundleWriter
from deeprec_b200.data import criteo_batch
from deeprec_b200.models.dlrm import DLRM
from deeprec_b200.models.zoo import build_model
from deeprec_b200.serving import Processor, export_delta_module, export_saved_model_module, export_saved_model_program

pytestmark = [pytest.mark.timeout(900)]

CARDS = [50, 1000, 7, 300]
DEVICES = ["cpu", "cuda_emu"]
TOL = {"cpu": 1e-5, "cuda_emu": 3e-2}       # the GPU runtime keeps bf16 activations between the layers
JSON_DEPTH_LIMIT = 64                       # drjson::JParser


def _dlrm(cards=CARDS):
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    return DLRM(13, cards, 16, mlp_bot=(64, 16), mlp_top=(512, 256), device="cpu")    # top MLP of the zoo DLRM: a shape the GPU kernels cover


def _train(model, steps, seed):
    opt = dr.optim.AdagradOptimizer(model, lr=0.05)
    for s in range(steps):
        d, ids, y = criteo_batch(64, 13, CARDS, seed=seed + s)
        loss = model.loss(d, ids, y); opt.zero_grad(); loss.backward(); opt.step()


def _ref(model, d, ids):
    model.eval()
    with torch.no_grad():
        p = torch.sigmoid(model(d, ids)).numpy().copy()
    model.train()
    return p


def _rewrite(prefix, edit):
    """Rewrite the bundle at ``prefix``: ``edit(name, tensor)`` returns the tensor to store."""
    r = BundleReader(prefix)
    tensors = {n: r.read(n) for n in r.entries}
    r.close()
    w = BundleWriter(prefix)
    for n, t in tensors.items():
        w.add(n, edit(n, t))
    w.close()


def _variables(export_dir):
    return os.path.join(export_dir, "variables", "variables")


@pytest.fixture(scope="module")
def dlrm_export(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("dlrm"))
    model = _dlrm()
    _train(model, 3, 0)
    export_saved_model_module(model, os.path.join(root, "v1"), version=1, root=root)
    return os.path.join(root, "v1")


@pytest.fixture(scope="module")
def program_export(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("program"))
    dr.embedding_variable.clear_registry()
    torch.manual_seed(0)
    model = build_model("deepfm", device="cpu", cardinalities=CARDS)
    export_saved_model_program(model, os.path.join(root, "v1"), version=1, root=root)
    return os.path.join(root, "v1")


def _first_linear_kernel(name, t):
    return name.startswith("prog/") and name.endswith("/kernel")


# name -> (export, which tensor, how it is damaged)
MALFORMED = {
    "truncated_table_values": ("dlrm", lambda n, t: n == "table/1-values", lambda t: t[:-1]),
    "default_not_a_multiple_of_D": ("dlrm", lambda n, t: n == "table/0-default", lambda t: t.reshape(-1)[:-3]),
    "short_moving_variance": ("dlrm", lambda n, t: n == "bn/mlp_bot_1/moving_variance", lambda t: t[:-1]),
    "linear_kernel_of_the_wrong_length": ("program", _first_linear_kernel, lambda t: t.reshape(-1)[:-1]),
}


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("case", sorted(MALFORMED))
def test_initialization_refuses_a_malformed_export(tmp_path, dlrm_export, program_export, case, device):
    which, match, damage = MALFORMED[case]
    src = dlrm_export if which == "dlrm" else program_export
    # the untouched export loads on this runtime
    Processor(src, {"session_num": 1, "max_batch": 16, "model_update_interval_ms": 0}, device=device).close()
    bad = str(tmp_path / "bad")
    shutil.copytree(src, bad)
    hits = []

    def edit(name, t):
        if match(name, t) and not hits:
            hits.append(name)
            return damage(t).contiguous()
        return t
    _rewrite(_variables(bad), edit)
    assert hits, case
    with pytest.raises(RuntimeError):
        Processor(bad, {"session_num": 1, "max_batch": 16, "model_update_interval_ms": 0}, device=device)


@pytest.mark.parametrize("device", DEVICES)
def test_model_config_nesting_is_limited(dlrm_export, device):
    def cfg(depth):            # the config object is level 1, its "nested" value levels 2 .. depth
        nested = []
        for _ in range(depth - 2):
            nested = [nested]
        return {"session_num": 1, "max_batch": 16, "model_update_interval_ms": 0, "nested": nested}
    Processor(dlrm_export, cfg(JSON_DEPTH_LIMIT), device=device).close()
    with pytest.raises(RuntimeError):
        Processor(dlrm_export, cfg(JSON_DEPTH_LIMIT + 1), device=device)


@pytest.mark.parametrize("device", DEVICES)
def test_delta_with_short_values_is_not_applied(tmp_path, device):
    root = str(tmp_path)
    model = _dlrm()
    _train(model, 3, 0)
    export_saved_model_module(model, os.path.join(root, "v1"), version=6, root=root)
    d, ids, _ = criteo_batch(32, 13, CARDS, seed=77)
    ref = _ref(model, d, ids)
    _train(model, 3, 100)
    assert np.abs(_ref(model, d, ids) - ref).max() > 1e-3           # the delta would change the predictions
    prefix = export_delta_module(model, root, base_version=6, version=9)
    _rewrite(prefix, lambda n, t: t[:-1].contiguous() if n.endswith("-sparse_incr_values") else t)
    proc = Processor(os.path.join(root, "v1"), {"session_num": 1, "max_batch": 32, "checkpoint_dir": root, "model_update_interval_ms": 50}, device=device)
    try:
        time.sleep(1.5)                                              # ~30 polls of the version file
        info = proc.model_info()
        assert info["delta_version"] == -1 and info["delta_updates"] == 0 and info["model_version"] == 6
        assert np.abs(proc.predict(d.numpy(), ids.numpy()) - ref).max() < TOL[device]
    finally:
        proc.close()


def test_gpu_runtime_rejects_a_full_version_with_more_tables(tmp_path):
    """The GPU runtime's sessions are sized for the architecture they started with: a full version with another table is refused and the
    old version keeps answering (the CPU runtime grows its sessions instead: test_cpu_serving.py)."""
    root = str(tmp_path)
    model = _dlrm()
    export_saved_model_module(model, os.path.join(root, "v1"), version=1, root=root)
    d, ids, _ = criteo_batch(32, 13, CARDS, seed=5)
    ref = _ref(model, d, ids)
    proc = Processor(os.path.join(root, "v1"), {"session_num": 1, "max_batch": 32, "checkpoint_dir": root, "model_update_interval_ms": 50},
                     device="cuda_emu")
    try:
        wider = _dlrm(CARDS + [20])
        export_saved_model_module(wider, os.path.join(root, "v2"), version=2, root=root)
        time.sleep(1.5)
        info = proc.model_info()
        assert info["model_version"] == 1 and info["full_updates"] == 0
        assert np.abs(proc.predict(d.numpy(), ids.numpy()) - ref).max() < TOL["cuda_emu"]
    finally:
        proc.close()
