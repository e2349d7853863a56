#!/usr/bin/env python
"""Headline benchmark: DLRM training samples/sec on N H100 GPUs of one node (BASELINE.json).

  python bench.py --gpus 1 --steps 20 --warmup 5
  python bench.py --gpus 1 --steps 20 --warmup 5 --dump-outputs /tmp/out     # + what the last timed step computed, as .npy files
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29500 \
         bench.py --gpus 8 --steps 20 --warmup 5

Model/config: modelzoo DLRM (bottom 512-256-64-16 +BN, 26 EmbeddingVariable tables dim 16, dot interaction,
top 512-256, logits) on synthetic Criteo-Terabyte-shaped data, bf16 MLP compute / fp32 master weights and
embeddings, Adagrad for dense + sparse, weak scaling (fixed per-GPU batch), 26 tables model-parallel.

Data stream (--stream):
  fresh (default)  every prefill / warm-up / timed step consumes a batch NEVER SEEN BEFORE, so key inserts, admission
                   bookkeeping, row allocation and default-row initialisation all run inside the timed region
                   (reported as new_keys_per_step).  The batches are pre-generated into pinned host memory: the C++
                   generator needs ~0.13 s per 65536x26 batch, 100x the GPU step, so it cannot run inside the loop.
  warm             round-1 behaviour (8 rotating batches, tables fully populated before timing) -- labelled secondary.

Arms:  --impl ours (default)  fused unique-first P2P pipeline, one CUDA graph per step
       | nccl_comm            the SAME engine and dense kernels with the reference (SOK) dataflow over NCCL collectives
                              (parallel/nccl_baseline.NcclComm: all-to-all ids / vectors / gradients, all-reduce), eager launches
       | nccl_baseline        NCCL + cuBLAS (torch.nn autocast) + autograd re-creation of the reference step
       | reference            the unmodified DeepRec tree: cannot be installed offline -> prints "unavailable".
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

BASELINE_SAMPLES_PER_SEC = None   # BASELINE.json "published": {} -- the reference publishes no samples/s for this config


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=65536, help="per-GPU batch (weak scaling)")
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "nccl_comm", "nccl_baseline"])
    ap.add_argument("--stream", default="fresh", choices=["fresh", "warm"])
    ap.add_argument("--prefill", type=int, default=8, help="untimed training steps before warm-up (history of the tables)")
    ap.add_argument("--pool", type=int, default=0, help="distinct batches of the timed region (0 = one per step; warm stream: 8)")
    ap.add_argument("--alpha", type=float, default=1.05, help="power-law exponent of the synthetic id distribution (0 = uniform)")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--optimizer", default="adagrad")
    ap.add_argument("--filter-freq", type=int, default=0, help="CounterFilter admission threshold (0 = admit at first sight)")
    ap.add_argument("--sparse-blocks", type=int, default=4, help="resident blocks/SM of the side-stream sparse kernels")
    ap.add_argument("--no-overlap", action="store_true")
    ap.add_argument("--gemm-v1", action="store_true")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last timed step's results (probabilities, loss, updated dense parameters, "
                         "a seeded sample of the updated embedding rows) "
                         "as float32 DIR/<name>.npy; the inputs depend only on the arguments, so two builds can be compared")
    return ap.parse_args()


class ClockSampler:
    """SM clock / power / throttle reasons DURING the timed regions.  In-process NVML from a sampling thread (a 20-step region lasts tens
    of ms: `nvidia-smi -lms` does not even start within it); nvidia-smi is the fallback."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
    REASONS = ((0x8, "hw_slowdown"), (0x40, "hw_thermal_slowdown"), (0x20, "sw_thermal_slowdown"), (0x4, "sw_power_cap"), (0x80, "hw_power_brake"))

    def __init__(self, gpu_index: int):
        self.gpu, self.proc, self.lines = gpu_index, None, []
        self.nvml, self.h, self.stop_flag = None, None, threading.Event()
        self.sm, self.mx, self.pw, self.mask = [], [], [], 0
        try:
            import pynvml
            pynvml.nvmlInit()
            h = None
            try:
                uuid = str(torch.cuda.get_device_properties(gpu_index).uuid)
                h = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid) if not uuid.startswith("GPU-") else uuid)
            except Exception:
                h = pynvml.nvmlDeviceGetHandleByIndex(gpu_index)
            pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
            self.nvml, self.h = pynvml, h
        except Exception:
            self.nvml = None

    def _sample(self):
        n, h = self.nvml, self.h
        try:
            self.sm.append(float(n.nvmlDeviceGetClockInfo(h, n.NVML_CLOCK_SM)))
            self.mx.append(float(n.nvmlDeviceGetMaxClockInfo(h, n.NVML_CLOCK_SM)))
            self.pw.append(n.nvmlDeviceGetPowerUsage(h) / 1e3)
            try:
                self.mask |= int(n.nvmlDeviceGetCurrentClocksEventReasons(h))
            except Exception:
                self.mask |= int(n.nvmlDeviceGetCurrentClocksThrottleReasons(h))
        except Exception:
            pass

    def _loop(self):
        while not self.stop_flag.is_set():
            self._sample()
            time.sleep(0.004)

    def start(self):
        if self.nvml is not None:
            self.t = threading.Thread(target=self._loop, daemon=True); self.t.start()
            return
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100",
                                          "-i", str(self.gpu)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True); self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.nvml is not None:
            self.stop_flag.set(); self.t.join(timeout=2)
            reasons = sorted(name for bit, name in self.REASONS if self.mask & bit)
            return {"sm_mhz": statistics.median(self.sm) if self.sm else None, "sm_max_mhz": max(self.mx) if self.mx else None,
                    "power_w_max": max(self.pw) if self.pw else None, "reasons": reasons, "samples": len(self.sm), "source": "nvml"}
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, pw, reasons = [], [], [], set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2])); pw.append(float(f[3]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "power_w_max": max(pw) if pw else None, "reasons": sorted(reasons), "samples": len(sm), "source": "nvidia-smi"}


def reference_arm(args):
    """The reference is a TensorFlow-1.15 fork built with Bazel 3.7.2 (no setup.py/pyproject at its root); the
    offline `pip install /root/reference` cannot build it (recorded in DESIGN.md)."""
    ref = os.path.join(os.path.dirname(os.path.abspath(__file__)), "baseline", "_ref")
    why = "DeepRec is a TF-1.15/Bazel tree with no pip-installable root (pip install --no-index /root/reference: 'neither setup.py nor pyproject.toml found'); needs Bazel 3.7.2 + network"
    if os.path.isdir(ref) and any(os.scandir(ref)):
        try:
            sys.path.insert(0, ref)
            import tensorflow  # noqa: F401
            why = "baseline/_ref imports but no GPU DLRM runner is wired"   # never reached offline
        except Exception as e:  # pragma: no cover
            why = f"baseline/_ref present but unusable: {type(e).__name__}"
    if int(os.environ.get("RANK", "0")) == 0:
        print(json.dumps({"impl": "reference", "unavailable": why}))
    return 0


def make_host_batches(cfg, n: int, seed: int, alpha: float, rank: int):
    """n distinct synthetic Criteo-Terabyte-shaped batches in PINNED host memory (C++ generator, csrc/host/io_runtime.cc)."""
    from deeprec_b200.data.synthetic import criteo_batch
    out = []
    for i in range(n):
        d, ids, y = criteo_batch(cfg.batch_size, cfg.num_dense, cfg.cardinalities, seed=seed + 100003 * rank + i, alpha=alpha)
        out.append((d.pin_memory(), ids.pin_memory(), y.pin_memory()))
    return out


def unique_ratio(ids: torch.Tensor) -> float:
    """distinct (table, id) pairs / ids of one batch (host-side, diagnostics only)."""
    u = sum(int(torch.unique(ids[t]).numel()) for t in range(ids.shape[0]))
    return u / float(ids.numel())


def dump_outputs(eng, out_dir: str, last_ids: torch.Tensor, rows_per_table: int = 256) -> None:
    """What the timed path hands back after its last step: per-sample click probabilities, the loss, the updated dense parameters
    (MLP weights / biases, BatchNorm statistics) and the embedding rows of a fixed, seeded sample of the last step's ids (what the sparse
    update wrote), each as <out_dir>/<name>.npy -- float32, the sampled ids float64 (exact below 2^53); a few MB in all."""
    import numpy as np
    core = eng.eng if hasattr(eng, "eng") else eng
    arrays = {"prob": core.prob, "loss": core.loss}
    if hasattr(core, "state_dict"):
        arrays.update(core.state_dict())
    tables = getattr(core, "tables", None)
    if tables:
        g = torch.Generator().manual_seed(0)
        pos = torch.randperm(last_ids.shape[1], generator=g)[:rows_per_table].to(last_ids.device)
        for t, tb in sorted(tables.items()):
            keys = last_ids[t, pos].contiguous()
            arrays[f"emb_rows_t{t:02d}"] = tb.lookup(keys)
            arrays[f"emb_ids_t{t:02d}"] = keys.double()
    os.makedirs(out_dir, exist_ok=True)
    for name, t in arrays.items():
        t = t.detach()
        np.save(os.path.join(out_dir, name.replace("/", "__") + ".npy"), (t if t.dtype == torch.float64 else t.float()).cpu().numpy())


def main():
    args = parse_args()
    if args.impl == "reference":
        return reference_arm(args)
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != args.gpus and not (args.gpus == 1 and world == 1):
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torch.distributed.run --nproc-per-node {args.gpus}")
    # host threads next to the GPU (pinned staging buffers, producer thread, OpenMP pool): GPUs 4-7 of an HGX box hang off the second socket
    from deeprec_b200.utils.affinity import bind_to_gpu_numa
    bound = bind_to_gpu_numa(local_rank)
    if bound:
        torch.set_num_threads(max(1, min(torch.get_num_threads(), len(bound))))      # libgomp sized its team before the mask shrank
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    import torch.distributed as dist
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)

    from deeprec_b200.models.dlrm_engine import DLRMConfig, DLRMEngine
    cfg = DLRMConfig(batch_size=args.batch, optimizer=args.optimizer, sparse_blocks_per_sm=args.sparse_blocks,
                     overlap_embedding=not args.no_overlap, gemm_v1=args.gemm_v1, filter_freq=args.filter_freq)
    comm = None
    graph = not args.no_graph
    if args.impl in ("nccl_comm", "nccl_baseline"):
        from deeprec_b200.parallel.nccl_baseline import BaselineDLRM, NcclComm
        comm = NcclComm(rank, world, dev)
        graph = False                       # NCCL collectives are launched eagerly between our kernels
        eng = BaselineDLRM(cfg, dev, rank, world, comm) if args.impl == "nccl_baseline" else DLRMEngine(cfg, dev, rank, world, comm)
    else:
        if world > 1:
            from deeprec_b200.parallel.p2p import P2PComm
            comm = P2PComm(rank, world, dev)
        eng = DLRMEngine(cfg, dev, rank, world, comm)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    def total_keys() -> int:
        tables = eng.eng.tables if hasattr(eng, "eng") else eng.tables
        t = torch.tensor([float(sum(tb.size() for tb in tables.values()))], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t)
        return int(t.item())

    # ---- data: every phase draws from ONE sequence of distinct batches (fresh) or from 8 rotating ones (warm) ---------
    fresh = args.stream == "fresh"
    n_timed = args.steps if (fresh and args.pool <= 0) else (min(args.steps, args.pool) if fresh else (args.pool or 8))
    n_e2e = 0 if args.skip_e2e else n_timed + args.warmup
    if fresh:
        host = make_host_batches(cfg, args.prefill + args.warmup + n_timed + n_e2e, 99, args.alpha, rank)
        pre, warm = host[: args.prefill], host[args.prefill: args.prefill + args.warmup]
        timed = host[args.prefill + args.warmup: args.prefill + args.warmup + n_timed]
        e2e_src = host[args.prefill + args.warmup + n_timed:]
    else:
        host = make_host_batches(cfg, n_timed, 99, args.alpha, rank)
        pre = [host[s % len(host)] for s in range(args.prefill)]
        warm = [host[s % len(host)] for s in range(args.warmup)]
        timed, e2e_src = host, host
    uniq = unique_ratio(timed[0][1])
    dev_timed = [(d.to(dev), i.to(dev), y.to(dev)) for d, i, y in timed]       # device-timed region: inputs resident, > L2 in total
    in_bytes = sum(t.numel() * t.element_size() for t in timed[0])

    # ---- prefill + graph capture + warm-up (all untimed) -------------------------------------------------
    first = pre[0] if pre else warm[0] if warm else timed[0]
    eng.load_batch(*[t.to(dev) for t in first])
    if graph and hasattr(eng, "capture"):
        eng.capture()                      # one eager step on `first`, then the whole step becomes one CUDA graph
        pre = pre[1:] if pre else pre
    for b in pre + warm:
        eng.load_batch(*[t.to(dev, non_blocking=True) for t in b]); eng.train_step()
    barrier()

    # ---- device-timed region: K steps, CUDA events on the launching stream, max over ranks ------------------
    keys0 = total_keys()
    sampler = ClockSampler(local_rank)
    sampler.start()
    l0 = eng.launches
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(args.steps):
        eng.load_batch(*dev_timed[s % len(dev_timed)])
        eng.train_step()
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    launches = eng.launches - l0
    keys1 = total_keys()
    final_loss = eng.loss_value()           # mean over the GLOBAL batch of the last timed step (all-reduced)
    if args.dump_outputs and rank == 0:
        dump_outputs(eng, args.dump_outputs, dev_timed[(args.steps - 1) % len(dev_timed)][1])

    # ---- end-to-end region through the public API: smart_stage (producer thread -> packed pinned H2D on a copy stream, two
    #      batches ahead) -> load_batch -> train_step -> D2H of the loss, every step ------------------------------
    e2e_ms = None
    if not args.skip_e2e:
        from deeprec_b200.data.staged import SmartStageOptions, smart_stage
        seq = [e2e_src[s % len(e2e_src)] for s in range(args.warmup + args.steps)]
        stage = smart_stage(iter(seq), dev, SmartStageOptions(capacity=2, num_threads=1))
        loss_host = torch.zeros(args.steps, dtype=torch.float32).pin_memory()
        for s in range(args.warmup):                               # untimed: producer thread, pinned pool and device ring spin up
            eng.load_batch(*next(stage)); eng.train_step()
        barrier()
        f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        f0.record()
        for s in range(args.steps):
            d, ids, y = next(stage)                                # H2D of THIS step's inputs (17 MB from pinned memory)
            eng.load_batch(d, ids, y)
            eng.train_step()
            loss_host[s].copy_(eng.loss[0], non_blocking=True)     # D2H of the step result
        f1.record()
        barrier()
        e2e_ms = f0.elapsed_time(f1)
        stage.close()

    clocks = sampler.stop()                 # sampled across the device-timed AND the end-to-end region (both under load)

    # max over ranks (device-timed)
    t = torch.tensor([ms, e2e_ms if e2e_ms is not None else 0.0], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, e2e_max = float(t[0]), float(t[1])
    gb = cfg.batch_size * world
    value = gb * args.steps / (ms / 1e3)
    if rank == 0:
        sharding = {"ours": f"mp{world}(emb: every table row-sharded hash(key)%{world}, requester-side dedup)+dp{world}(dense)",
                    "nccl_comm": f"mp{world}(emb: table t on rank t%{world}, SOK all-to-all dataflow over NCCL)+dp{world}(dense, ncclAllReduce)",
                    "nccl_baseline": f"mp{world}(emb: table t on rank t%{world}, NCCL)+dp{world}(dense, cuBLAS + autograd + NCCL)"}[args.impl]
        out = {
            "metric": "DLRM samples/sec (whole box, device-timed, max over ranks)", "value": value, "unit": "samples/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps,
            "higher_is_better": True, "scaling": "weak",
            "vs_baseline": (value / BASELINE_SAMPLES_PER_SEC) if BASELINE_SAMPLES_PER_SEC else None,
            "dtype": "bf16", "data": "synthetic (Criteo-Terabyte-shaped power-law ids, random-init weights)",
            "impl": args.impl,
            "config": {"model": "DLRM modelzoo (bot 512-256-64-16+BN, 26 EV tables dim16, dot, top 512-256)",
                       "global_batch": gb, "seq_len": 1, "parallelism": sharding,
                       "optimizer": args.optimizer, "per_gpu_batch": cfg.batch_size,
                       "stream": ("fresh: every prefill/warm-up/timed step is a never-seen batch (inserts + row init inside the timed region)"
                                  if fresh else "warm: 8 rotating batches, tables populated before timing (no inserts in the timed region)"),
                       "prefill_steps": args.prefill, "distinct_timed_batches": len(dev_timed),
                       "new_keys_per_step": (keys1 - keys0) / float(args.steps), "unique_ratio": uniq, "alpha": args.alpha,
                       "filter_freq": args.filter_freq,
                       "l2": f"{len(dev_timed)} distinct resident batches ({len(dev_timed) * in_bytes / 1e6:.0f} MB) + multi-GB embedding tables > 50 MB L2; no flush",
                       "cuda_graph": bool(graph and hasattr(eng, "capture")), "final_loss": final_loss,
                       "host_cpus": f"{len(bound)} CPUs local to the GPU (NVML ideal set)" if bound else "unpinned"},
            "clocks": clocks,
            "gpu_launches": launches,
        }
        if e2e_ms is not None:
            out["e2e"] = {"value": gb * args.steps / (e2e_max / 1e3), "unit": "samples/s", "h2d_bytes_per_step": in_bytes, "d2h_bytes_per_step": 4,
                          "ms_per_step": e2e_max / args.steps, "api": "data.staged.smart_stage -> DLRMEngine.load_batch -> train_step"}
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
