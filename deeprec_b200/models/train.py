"""``python -m deeprec_b200.models.train --model dlrm ...``: the modelzoo train.py flag surface (modelzoo/mlperf/README.md:40-74):
--ev --ev_filter {counter,cbf} --ev_elimination {l2,gstep} --emb_fusion --op_fusion --smartstaged --optimizer {adam,adamasync,
adagraddecay,adagrad,gradientdescent,ftrl} --bf16 --incremental_ckpt --workqueue --parquet_dataset --group_embedding
--adaptive_emb --dynamic_ev --micro_batch --timeline --steps --batch_size --learning_rate --checkpoint.
Synthetic Criteo / Taobao data (no datasets offline); ``--engine`` runs DLRM through the fused GPU engine."""
from __future__ import annotations

import argparse
import sys
import os
import time

import torch

import deeprec_b200 as dr
from deeprec_b200.data import criteo_batch, smart_stage, taobao_batch
from deeprec_b200.models.zoo import TAOBAO_MODELS, build_model
from deeprec_b200.optim import make_optimizer
from deeprec_b200.utils import Trainer


def get_arg_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="dlrm")
    p.add_argument("--steps", type=int, default=100)
    p.add_argument("--batch_size", type=int, default=2048)
    p.add_argument("--learning_rate", type=float, default=0.01)
    p.add_argument("--optimizer", default="adagrad", choices=["adam", "adamasync", "adagraddecay", "adagrad", "gradientdescent", "ftrl", "adamw"])
    p.add_argument("--ev", action="store_true", default=True)
    p.add_argument("--ev_filter", default=None, choices=[None, "counter", "cbf"])
    p.add_argument("--ev_elimination", default=None, choices=[None, "l2", "gstep"])
    p.add_argument("--emb_fusion", action="store_true")
    p.add_argument("--op_fusion", action="store_true")
    p.add_argument("--group_embedding", action="store_true")
    p.add_argument("--smartstaged", action="store_true")
    p.add_argument("--bf16", action="store_true")
    p.add_argument("--incremental_ckpt", type=float, default=0, help="seconds between incremental checkpoints")
    p.add_argument("--checkpoint", default=None)
    p.add_argument("--save_steps", type=int, default=0)
    p.add_argument("--workqueue", action="store_true")
    p.add_argument("--micro_batch", type=int, default=1)
    p.add_argument("--output_dir", default=None, help="TensorBoard event files (loss, global_step/sec, EmbeddingVariable sizes) are written here")
    p.add_argument("--no_eval", action="store_true", help="skip the evaluation pass (ACC / AUC on held-out synthetic batches) after training")
    p.add_argument("--eval_steps", type=int, default=10)
    p.add_argument("--parquet_dataset", default=None, help="glob of Criteo-shaped parquet files (label, I1..I13, C1..C26); default: synthetic data")
    p.add_argument("--multihash", action="store_true", help="Q-R multi-hash embeddings instead of EmbeddingVariables")
    p.add_argument("--adaptive_emb", action="store_true", help="adaptive embedding: static hashed table for cold ids, EV for hot ids")
    p.add_argument("--dynamic_ev", action="store_true", help="accepted for parity (the modelzoo marks dynamic-dimension EV as not enabled)")
    p.add_argument("--protocol", default="local", choices=["local", "grpc", "grpc++", "star_server"],
                   help="grpc / grpc++ / star_server select the asynchronous parameter-server mode (deeprec_b200.parallel.ps); run the "
                        "roles with `python -m deeprec_b200.parallel.ps_train`")
    p.add_argument("--timeline", type=int, default=0)
    p.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
    p.add_argument("--engine", action="store_true", help="fused sm_90a engines: DLRM (models/dlrm_engine.py); WDL / DeepFM / DCN / DCNv2 / MaskNet / DIN through FusedRecEngine (models/rec_engine.py)")
    p.add_argument("--log_every", type=int, default=20)
    p.add_argument("--watchdog", type=float, default=0, help="seconds without a finished step before the job dumps stacks and exits 86")
    return p


def ev_option_from_args(a) -> dr.EmbeddingVariableOption:
    flt = dr.CounterFilter(2) if a.ev_filter == "counter" else dr.CBFFilter(2, 1 << 20, 0.01) if a.ev_filter == "cbf" else None
    ev = dr.L2WeightEvict(1e-4) if a.ev_elimination == "l2" else dr.GlobalStepEvict(4000) if a.ev_elimination == "gstep" else None
    st = dr.StorageOption(dr.StorageType.HBM if a.device.startswith("cuda") else dr.StorageType.DRAM)
    return dr.EmbeddingVariableOption(filter_option=flt, evict_option=ev, storage_option=st)


def main(argv=None) -> int:
    a = get_arg_parser().parse_args(argv)
    dev = torch.device(a.device)
    name = a.model.lower()
    if a.engine and name == "dlrm":
        from deeprec_b200.models.dlrm_engine import CRITEO_KAGGLE_CARDINALITIES, DLRMConfig, DLRMEngine
        eng = DLRMEngine(DLRMConfig(batch_size=a.batch_size, cardinalities=CRITEO_KAGGLE_CARDINALITIES, optimizer=a.optimizer, learning_rate=a.learning_rate))
        t0 = time.time()
        for s in range(a.steps):
            d, ids, y = criteo_batch(a.batch_size, 13, CRITEO_KAGGLE_CARDINALITIES, seed=s)
            eng.load_batch(d.to(dev), ids.to(dev), y.to(dev)); eng.train_step()
            if s == 2:
                eng.capture()
            if a.log_every and s % a.log_every == 0:
                print(f"global_step {s} loss {eng.loss_value():.5f}")
        print(f"{a.steps * a.batch_size / (time.time() - t0):.0f} samples/s")
        return 0
    if a.engine:
        # every other Criteo-style model (and DIN) through FusedRecEngine: the same unique-first sparse pipeline + one CUDA graph per step
        # under the model's own dense net (models/rec_engine.py; 1..8 GPUs when launched with torchrun / parallel.launch)
        from deeprec_b200.models import zoo
        from deeprec_b200.models.rec_engine import criteo_engine, din_engine, din_ids
        if name not in zoo.CRITEO_MODELS and name != "din":
            raise SystemExit(f"--engine: no fused-engine adapter for {name} (dlrm, {', '.join(sorted(zoo.CRITEO_MODELS))}, din)")
        import torch.distributed as dist
        world, rank, lrank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(lrank)
        dev = torch.device("cuda", lrank)
        comm = None
        if world > 1:
            dist.init_process_group("nccl", device_id=dev)
            from deeprec_b200.parallel.p2p import P2PComm
            comm = P2PComm(rank, world, dev)
        torch.manual_seed(0)
        model = build_model(name, device=dev)
        kw = dict(optimizer=a.optimizer, learning_rate=a.learning_rate, filter_freq=2 if a.ev_filter else 0,
                  steps_to_live=4000 if a.ev_elimination == "gstep" else 0, device=dev, rank=rank, world_size=world, comm=comm,
                  micro_batch_num=a.micro_batch)
        if name == "din":
            L = 20
            eng = din_engine(model, a.batch_size, L, table_rows=(100000, 200000, 1000), **kw)

            def batch(s):
                b = taobao_batch(a.batch_size, L, 100000, 200000, 1000, seed=s * world + rank)
                return din_ids(b), b["labels"], None
        else:
            cards = [1000] * 26
            eng = criteo_engine(model, a.batch_size, table_rows=cards, **kw)

            def batch(s):
                d, ids, y = criteo_batch(a.batch_size, 13, cards, seed=s * world + rank)
                return ids, y, {"dense": d}
        t0 = time.time()
        for s in range(a.steps):
            ids, y, dense = batch(s)
            eng.load_batch(ids.to(dev), y.to(dev), {k: v.to(dev) for k, v in dense.items()} if dense else None)
            if s == 0:
                eng.capture()                  # one eager step on the loaded batch, then the step is a CUDA graph
            else:
                eng.train_step()
            if a.log_every and s % a.log_every == 0 and rank == 0:
                print(f"global_step {s} loss {eng.loss_value():.5f}")
            elif a.log_every and s % a.log_every == 0:
                eng.loss_value()               # the all-reduce of the loss is collective
            if a.checkpoint and a.save_steps and s and s % a.save_steps == 0:
                eng.save(a.checkpoint, incremental=bool(a.incremental_ckpt) and s // a.save_steps > 1)
        torch.cuda.synchronize()
        if rank == 0:
            print(f"{a.steps * a.batch_size * world / (time.time() - t0):.0f} samples/s")
        if world > 1:
            dist.barrier(); dist.destroy_process_group()
        return 0
    if a.protocol != "local":
        print(f"--protocol {a.protocol}: parameter-server roles are started with `python -m deeprec_b200.parallel.ps_train`; training locally here")
    cards = [1000] * 26
    from deeprec_b200.models import zoo
    zoo.table_variant("multihash" if a.multihash else "adaptive" if a.adaptive_emb else "ev")
    try:
        model = build_model(name, ev_option_from_args(a), dev, a.group_embedding or a.emb_fusion, cardinalities=cards)
    finally:
        zoo.table_variant("ev")
    if a.op_fusion:                       # auto graph fusion (do_op_fusion)
        from deeprec_b200 import graph_optimizer
        rep = graph_optimizer.optimize(model)
        print(f"op_fusion: {rep.count()} rewrites")
    opt = make_optimizer(a.optimizer, model, lr=a.learning_rate)
    taobao = name in TAOBAO_MODELS

    def parquet_batches(files):
        from deeprec_b200.data import ParquetDataset
        for rec in ParquetDataset(files, batch_size=a.batch_size, drop_remainder=True):
            d = torch.stack([rec[f"I{i}"].float() for i in range(1, 14)], 1)
            ids = torch.stack([rec[f"C{i}"].long() for i in range(1, 27)], 0)
            yield d.to(dev), ids.to(dev), rec["label"].float().to(dev)

    def gen():
        s = 0
        if a.parquet_dataset and not taobao:
            import glob
            files = sorted(glob.glob(a.parquet_dataset))
            if not files:
                raise FileNotFoundError(a.parquet_dataset)
            if a.workqueue:               # files are work items: any number of workers can share the queue, progress is resumable
                from deeprec_b200.data import WorkQueue
                wq = WorkQueue(files, num_epochs=1 << 30, shuffle=True)
                yield from wq.input_dataset(lambda f: parquet_batches([f]))
            else:
                while True:
                    yield from parquet_batches(files)
            return
        wq = None
        if a.workqueue:                   # synthetic shards as work items
            from deeprec_b200.data import WorkQueue
            wq = WorkQueue([str(i) for i in range(1 << 16)], num_epochs=1 << 20, shuffle=True)
        while True:
            if wq is not None:
                s = int(wq.take())
            if taobao:
                b = taobao_batch(a.batch_size, 20, 100000, 200000, 1000, seed=s)
                yield {k: v.to(dev) for k, v in b.items()}
            else:
                d, ids, y = criteo_batch(a.batch_size, 13, cards, seed=s)
                yield d.to(dev), ids.to(dev), y.to(dev)
            s += 1

    def loss_fn(m, b):
        ctx = torch.autocast(dev.type, dtype=torch.bfloat16) if a.bf16 else torch.autocast(dev.type, enabled=False)
        with ctx:
            return m.loss(b) if taobao else m.loss(*b)

    src = smart_stage(gen(), device=None) if a.smartstaged else gen()
    tr = Trainer(model, opt, loss_fn, a.checkpoint, save_checkpoint_steps=a.save_steps, save_incremental_checkpoint_secs=a.incremental_ckpt,
                 log_every_n_steps=a.log_every, timeline_steps=a.timeline, micro_batch_num=a.micro_batch, watchdog_timeout_s=a.watchdog,
                 hooks=[__import__("deeprec_b200.utils.summary", fromlist=["SummaryHook"]).SummaryHook(a.output_dir, max(1, a.log_every or 100))] if a.output_dir else None)
    t0 = time.time()
    tr.fit(src, a.steps)
    print(f"{a.steps * a.batch_size / (time.time() - t0):.0f} samples/s")
    if not a.no_eval and a.eval_steps > 0:                  # modelzoo train.py: ACC / AUC after training unless --no_eval
        def held_out():
            for s in range(a.eval_steps):
                if taobao:
                    yield {k: v.to(dev) for k, v in taobao_batch(a.batch_size, 20, 100000, 200000, 1000, seed=10_000_000 + s).items()}
                else:
                    d, ids, y = criteo_batch(a.batch_size, 13, cards, seed=10_000_000 + s)
                    yield d.to(dev), ids.to(dev), y.to(dev)

        def predict(m, b):
            out = m(b) if taobao else m(b[0], b[1])
            if isinstance(out, dict):
                out = out["ctr"]
            return torch.sigmoid(out.float()), (b["labels"] if taobao else b[2])
        res = tr.evaluate(held_out(), predict, max_steps=a.eval_steps)
        print(f"Evaluation complete: ACC {res['acc']:.4f}  AUC {res['auc']:.4f}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
