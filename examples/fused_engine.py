"""FusedRecEngine: any dense net over the unique-first sparse pipeline, the whole training step as one CUDA graph on an H100 -- shown here on the
CUDA-on-CPU emulation of the same kernels (``_native.cuda_emulation()``), so it runs anywhere.  Multi-tier tables (HBM cache over host DRAM),
auto micro-batch, full + incremental training checkpoints.  On a GPU: drop the ``with`` line, build the model on ``cuda`` and call
``eng.capture()`` after the first batch; with torchrun + ``parallel.p2p.P2PComm`` the same code runs model-parallel on 1-8 GPUs."""
import contextlib
import os
import tempfile

import torch

import _path  # noqa: F401  (repository root on sys.path)
import deeprec_b200 as dr
from deeprec_b200 import _native
from deeprec_b200.data import criteo_batch
from deeprec_b200.models.rec_engine import criteo_engine
from deeprec_b200.models.zoo import build_model

on_gpu = torch.cuda.is_available()
CARDS = [50, 4000, 7, 300] + [97] * 22
B = 2048 if on_gpu else 128

with (contextlib.nullcontext() if on_gpu else _native.cuda_emulation()):
    torch.manual_seed(0)
    model = build_model("deepfm", device="cuda" if on_gpu else "cpu")
    eng = criteo_engine(model, B, table_rows=CARDS, optimizer="adagrad", learning_rate=0.05,
                        tiered={1: dict(cache_rows=128, strategy=0)},          # table 1: <= 128 rows in the HBM tier (LFU), the rest in host DRAM
                        micro_batch_num=2)                                     # dense net over 2 slices per step, one optimizer step

    def batch(s):
        d, ids, y = criteo_batch(B, 13, CARDS, seed=s)
        dev = eng.dev
        return ids.to(dev), y.to(dev), {"dense": d.to(dev)}

    ckpt = os.path.join(tempfile.mkdtemp(), "deepfm")
    eng.prefetch(batch(0)[0])                                                  # multi-tier: the NEXT batch's ids, one step ahead
    for s in range(8):
        eng.load_batch(*batch(s))
        eng.train_step()
        eng.prefetch(batch(s + 1)[0])
        if s == 3:
            eng.save(ckpt)                                                     # full checkpoint (both tiers of table 1)
        if s in (0, 7):
            print(f"step {s}: loss {eng.loss_value():.4f}")
    eng.save(ckpt, incremental=True)                                           # only the rows touched since step 3 + the dense block
    st = eng.tiers[1][0].stats()
    print(f"table 1: {st['hbm_rows']} rows in the HBM tier, {st['dram_rows']} in DRAM, hit rate {st['hit_rate']:.2f}, "
          f"{st['promoted_rows']} promoted / {st['demoted_rows']} demoted")

    dr.embedding_variable.clear_registry()
    fresh = criteo_engine(build_model("deepfm", device="cuda" if on_gpu else "cpu"), B, table_rows=CARDS, learning_rate=0.05,
                          tiered={1: dict(cache_rows=128, strategy=0)})
    step = fresh.restore(ckpt)                                                 # last full + the incremental chain; any world size
    print("restored at step", step, "| dense parameters identical:", bool(torch.equal(fresh.params, eng.params)))
