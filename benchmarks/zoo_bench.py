#!/usr/bin/env python
"""Model-zoo training throughput on one GPU (BASELINE.json configs 3 and 4):

  --model deepfm   Criteo-shaped synthetic data, 26 EmbeddingVariables through ONE fused GroupEmbedding lookup, FM kernel + FusedMLP
  --model din      Taobao-shaped synthetic data; the user-behaviour (item) table draws ids from a 1B-row id space and lives in
                   multi-tier storage (--hbm_rows rows of HBM cache over host DRAM, optional SSD tier) with CounterFilter admission and
                   GlobalStep eviction enabled
Any other zoo model name works too.  Timing: CUDA events around K steps after W warm-up steps; the input H2D copy of every step
is inside the timed region.  Prints one JSON line.

Multi-GPU (BASELINE.json config #3, DeepFM on 8 GPUs): launch with torchrun; the Criteo models then run through ``CollectiveStrategy``
-- tables model-parallel (table t on rank t % world, ids / rows exchanged with NCCL collectives), dense net data-parallel with a
bucketed gradient all-reduce -- i.e. the generic framework path (the fused NVLink kernels are the DLRM engine's, bench.py).  The value
is the whole-job samples/s, timed on the device, max over ranks.  ``--device cpu`` (gloo) is a functional dry run.

  torchrun --nnodes 1 --nproc-per-node 8 --master-addr 127.0.0.1 benchmarks/zoo_bench.py --model deepfm
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import deeprec_b200 as dr  # noqa: E402
from deeprec_b200.data import criteo_batch, taobao_batch  # noqa: E402
from deeprec_b200.models.zoo import CRITEO_MODELS, build_model  # noqa: E402


def engine_main(a):
    """BASELINE configs #3 (DeepFM) and #4 (DIN, 1B-id behaviour table with admission) on the fused engine, 1-8 GPUs; DIEN and BST on the
    same id layout; DSSM and the multi-task models (ESMM, MMoE, DBMTL, PLE, SimpleMultiTask) over pooled history bags."""
    import torch.distributed as dist
    from deeprec_b200.models.rec_engine import POOLED_SEQ_MODELS, criteo_engine, din_engine, din_ids, pooled_seq_engine, taobao_engine_batch
    world, rank, lr = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    from deeprec_b200.utils.affinity import bind_to_gpu_numa
    bound = bind_to_gpu_numa(lr)                                    # host threads (pinned buffers, OpenMP pool) next to the GPU
    if bound:
        torch.set_num_threads(max(1, min(torch.get_num_threads(), len(bound))))
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    comm = None
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
        from deeprec_b200.parallel.p2p import P2PComm
        comm = P2PComm(rank, world, dev)
    name = a.model.lower()
    torch.manual_seed(0)
    model = build_model(name, device=dev)
    n = a.warmup + a.steps + 3
    if name in CRITEO_MODELS:
        cards = [1_000_000] * 26
        eng = criteo_engine(model, a.batch, table_rows=cards, optimizer=a.optimizer, device=dev, rank=rank, world_size=world, comm=comm)
        host = []
        for s in range(n):
            d, ids, y = criteo_batch(a.batch, 13, cards, seed=s * world + rank)
            host.append((ids.pin_memory(), y.pin_memory(), {"dense": d.pin_memory()}))
        extra = {}
    elif name in POOLED_SEQ_MODELS:             # DSSM / multi-task: the behaviour history pooled into bags (sum) inside the sparse pipeline
        eng = pooled_seq_engine(model, a.batch, 50, table_rows=(10_000_000, min(a.id_space, 200_000_000), 10_000), optimizer=a.optimizer,
                                device=dev, rank=rank, world_size=world, comm=comm)
        host = []
        for s in range(n):
            b = taobao_batch(a.batch, 50, 10_000_000, a.id_space, 10_000, seed=s * world + rank)
            ids, y, _ = taobao_engine_batch(b) if eng.labels.dim() == 2 else (din_ids(b), b["labels"], None)
            host.append((ids.pin_memory(), y.pin_memory(), None))
        extra = {"item_id_space": a.id_space, "bags": "sum"}
    elif name not in ("din", "dien", "bst"):
        raise SystemExit(f"--engine: no fused-engine adapter for {name}")
    else:                                       # DIN; DIEN with both GRUs on the fused recurrence kernels; BST with its encoder block on the fused attention kernels
        eng = din_engine(model, a.batch, 50, table_rows=(10_000_000, min(a.id_space, 200_000_000), 10_000), optimizer=a.optimizer,
                         filter_freq=a.filter_freq, steps_to_live=100000, device=dev, rank=rank, world_size=world, comm=comm,
                         tiered={1: {"cache_rows": a.tier_rows, "strategy": 0}} if a.tier_rows > 0 else None)      # table 1 = the 1B-id behaviour (item) table
        host = []
        for s in range(n):
            b = taobao_batch(a.batch, 50, 10_000_000, a.id_space, 10_000, seed=s * world + rank)
            host.append((din_ids(b).pin_memory(), b["labels"].pin_memory(), None))
        extra = {"item_id_space": a.id_space, "filter_freq": a.filter_freq}
    put = lambda b: eng.load_batch(b[0].to(dev, non_blocking=True), b[1].to(dev, non_blocking=True),
                                   {k: v.to(dev, non_blocking=True) for k, v in b[2].items()} if b[2] else None)
    tiered = bool(getattr(eng, "tiers", None))
    ahead = (lambda j: eng.prefetch(host[j][0].to(dev, non_blocking=True))) if tiered else (lambda j: None)   # multi-tier: the NEXT batch's ids, one step ahead
    put(host[0]); eng.capture()
    ahead(3)
    for i in range(a.warmup):
        put(host[3 + i]); eng.train_step(); ahead(3 + i + 1)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        put(host[3 + a.warmup + i])                     # H2D of every step's inputs inside the timed region (pinned -> device)
        eng.train_step()
        if i + 1 < a.steps:
            ahead(3 + a.warmup + i + 1)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    t = torch.tensor([ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t[0])
    keys = torch.tensor([float(sum(tb.size() for tb in eng.tables.values()))], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(keys)
    loss = eng.loss_value()
    if tiered:
        st = eng.tiers[1][0].stats()
        extra["multi_tier"] = {"hbm_cache_rows_per_rank": a.tier_rows, **{k: st[k] for k in ("hit_rate", "promoted_rows", "demoted_rows", "h2d_bytes", "d2h_bytes", "hbm_rows", "dram_rows")}}
    if rank == 0:
        print(json.dumps({"metric": f"{name} training samples/s ({world} GPU, FusedRecEngine: unique-first sparse pipeline + CUDA graph, H2D inside the timed region)",
                          "value": a.batch * world / ms * 1e3, "unit": "samples/s", "n_gpus": world, "ms_per_step": ms, "batch": a.batch,
                          "global_batch": a.batch * world, "steps": a.steps, "warmup": a.warmup, "final_loss": loss, "keys_in_tables": int(keys.item()),
                          "parallelism": f"mp{world}(emb, hash(key)%{world}, P2P unique-first)+dp{world}(dense)", "dtype": "bf16 GEMMs / fp32 master weights",
                          "data": "synthetic", "launches_per_step": eng.launches_per_step, **extra}))
    if world > 1:
        dist.barrier(); dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="deepfm", help="a zoo model (models/zoo.py), e.g. deepfm, dcn, masknet_parallel, masknet_serial, din")
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--optimizer", default="adagrad")
    ap.add_argument("--hbm_rows", type=int, default=1 << 20, help="DIN: HBM cache rows of the multi-tier item table")
    ap.add_argument("--id_space", type=int, default=1_000_000_000, help="DIN: size of the item id space")
    ap.add_argument("--ssd", action="store_true", help="DIN: add the SSD tier below DRAM (HBM_DRAM_SSDHASH)")
    ap.add_argument("--filter_freq", type=int, default=2)
    ap.add_argument("--device", default="cuda", choices=["cuda", "cpu"])
    ap.add_argument("--tier_rows", type=int, default=0, help="--engine, DIN: HBM cache rows PER RANK of the behaviour table over a host DRAM tier (0 = single tier); works at 1-8 GPUs")
    ap.add_argument("--engine", action="store_true", help="FusedRecEngine: unique-first sparse pipeline + one CUDA graph per step (1-8 GPUs, NVLink P2P)")
    a = ap.parse_args()
    if a.engine:
        return engine_main(a)
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    strategy = None
    if world > 1:
        from deeprec_b200.parallel import CollectiveStrategy
        strategy = CollectiveStrategy(backend="nccl" if a.device == "cuda" else "gloo")
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0"))) if a.device == "cuda" else torch.device("cpu")
    cuda = dev.type == "cuda"
    name = a.model.lower()
    criteo = name in CRITEO_MODELS or name == "dlrm"
    if criteo:
        opt_ev = dr.EmbeddingVariableOption(storage_option=dr.StorageOption(dr.StorageType.HBM if cuda else dr.StorageType.DRAM))
        model = build_model(name, ev_option=opt_ev, device=dev, group_embedding=True)
        cards = [1_000_000] * 26
        gen = lambda s: criteo_batch(a.batch, 13, cards, seed=s * world + rank)
    else:
        row_bytes = 4 * 16 * 2
        if not cuda or world > 1:
            raise SystemExit("the multi-tier DIN configuration is single-GPU (HBM cache over host DRAM)")
        st = dr.StorageType.HBM_DRAM_SSDHASH if a.ssd else dr.StorageType.HBM_DRAM
        opt_ev = dr.EmbeddingVariableOption(storage_option=dr.StorageOption(dr.StorageType.HBM))
        model = build_model(name, ev_option=opt_ev, device=dev)
        # re-create the behaviour table as a multi-tier, filtered, evicting EmbeddingVariable
        big = dr.EmbeddingVariableOption(filter_option=dr.CounterFilter(a.filter_freq), evict_option=dr.GlobalStepEvict(100000),
                                         storage_option=dr.StorageOption(st, storage_size=(a.hbm_rows * row_bytes, 8 << 30),
                                                                         cache_strategy=dr.CacheStrategy.LFU))
        model.item = dr.get_embedding_variable(f"{name}/item_multitier", 16, ev_option=big, device=dev)
        gen = lambda s: taobao_batch(a.batch, 50, 10_000_000, a.id_space, 10_000, seed=s)
    opt = dr.optim.make_optimizer(a.optimizer, model, lr=0.01)
    dense_params = [p for g in opt.param_groups for p in g["params"]]
    if strategy is not None:
        strategy.broadcast_parameters(model)

    def to_dev(b):
        if not cuda:
            return b
        if isinstance(b, dict):
            return {k: v.pin_memory().to(dev, non_blocking=True) for k, v in b.items()}
        return tuple(t.pin_memory().to(dev, non_blocking=True) for t in b)

    def step(b):
        b = to_dev(b)
        if strategy is not None:
            with strategy.scope(), strategy.embedding_scope():          # group lookups inside are model-parallel
                loss = model.loss(*b)
        else:
            loss = model.loss(b) if isinstance(b, dict) else model.loss(*b)
        opt.zero_grad(); loss.backward()
        if strategy is not None:
            strategy.allreduce_gradients(dense_params, average=True)
        opt.step()
        return loss

    import torch.distributed as dist
    batches = [gen(s) for s in range(a.warmup + a.steps)]
    for i in range(a.warmup):
        step(batches[i])
    if strategy is not None:
        dist.barrier()
    if cuda:
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    t0 = time.perf_counter()
    for i in range(a.steps):
        loss = step(batches[a.warmup + i])
    if cuda:
        e1.record()
        torch.cuda.synchronize()
    wall_ms = (time.perf_counter() - t0) * 1e3 / a.steps
    ms = e0.elapsed_time(e1) / a.steps if cuda else wall_ms
    if strategy is not None:                      # max over ranks
        t = torch.tensor([ms], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t[0])
    out = {"metric": f"{name} training samples/s ({world} GPU{'s' if world > 1 else ''}, framework API, H2D inside the timed region)",
           "value": a.batch * world / ms * 1e3, "unit": "samples/s", "n_gpus": world, "parallelism": f"mp{world}(emb,table-wise,NCCL)+dp{world}(dense)" if world > 1 else "single",
           "ms_per_step": ms, "wall_ms_per_step": wall_ms, "batch": a.batch, "global_batch": a.batch * world, "steps": a.steps, "warmup": a.warmup,
           "final_loss": float(loss.item()), "dtype": "bf16 GEMMs / fp32 master weights" if cuda else "fp32 (cpu dry run)", "data": "synthetic"}
    if not criteo:
        t = model.item.table
        out["multi_tier"] = {k: (float(v) if not isinstance(v, dict) else v) for k, v in t.cache_stats().items()}
        out["item_table"] = {"admitted_rows": int(model.item.total_count()), "id_space": a.id_space, "hbm_rows": a.hbm_rows}
    if rank == 0:
        print(json.dumps(out))
    if strategy is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
