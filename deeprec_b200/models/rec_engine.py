"""FusedRecEngine -- one CUDA-graph training step for ANY dense network over the unique-first sparse pipeline.

:class:`models.dlrm_engine.DLRMEngine` hand-schedules DLRM's dense net; this engine generalises the same execution design to the
rest of the model zoo (DeepFM: BASELINE config #3, DIN: config #4, and any ``nn.Module`` that maps ``(dense inputs, embeddings
[B, C, D])`` to logits):

  * embeddings: every table row-sharded over the ranks (hash(key) % world), id columns deduplicated on the requester, distinct keys
    probed / inserted / admitted by their owners, rows pushed over NVLink, gradients pre-reduced per key and pulled by the owners,
    row-wise optimizer on the device table (``parallel/sparse_pipeline.py``) -- sequence features are just more id columns of the
    same table (``col_table``), padding ids (-1) produce zero rows and no statistics;
  * dense net: the module's own autograd graph (``nn.FusedMLP`` -> wgmma GEMMs), parameters and gradients re-pointed into ONE flat
    fp32 buffer each, so the optimizer is one fused kernel -- with ``world > 1`` the in-kernel-synchronised one-shot all-reduce +
    optimizer of ``parallel/p2p.py`` over the symmetric gradient buffer;
  * the whole step (forward, backward, both optimizers, flag protocol) is captured into ONE CUDA graph after three eager warm-up
    steps -- per-module Python / launch overhead, the reason the framework-API path ran DeepFM at 0.70 M samples/s, disappears.

Reference: modelzoo/deepfm/train.py:143-191, modelzoo/din/train.py:143-375 (models); group_embedding_lookup_sparse + SOK
(python/ops/embedding_ops.py:1594-1930) for the lookup they sit on.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Callable, Dict, List, Optional, Sequence

import torch
from torch import nn

from .. import _native
from .._native import EvConfig, OptHyper, ptr
from ..ops.device_table import DeviceTable, _chk, _next_pow2, get_context
from ..optim.optimizers import OPT_ADAGRAD, OPT_ADAGRAD_DECAY, OPT_ADAM, OPT_ADAM_ASYNC, OPT_ADAMW, OPT_FTRL, OPT_SGD
from ..parallel.sparse_pipeline import SparsePipeline

_OPT_KIND = {"sgd": OPT_SGD, "gradientdescent": OPT_SGD, "adagrad": OPT_ADAGRAD, "adagraddecay": OPT_ADAGRAD_DECAY,
             "adam": OPT_ADAM, "adamasync": OPT_ADAM_ASYNC, "adamw": OPT_ADAMW, "ftrl": OPT_FTRL}
_OPT_SLOTS = {OPT_SGD: 0, OPT_ADAGRAD: 1, OPT_ADAGRAD_DECAY: 1, OPT_ADAM: 2, OPT_ADAM_ASYNC: 2, OPT_ADAMW: 2, OPT_FTRL: 2}


class FusedRecEngine:
    def __init__(self, net: nn.Module, forward_fn: Callable[..., torch.Tensor], col_table: Sequence[int], table_rows: Sequence[int], batch_size: int,
                 embedding_dim: int = 16, dense_inputs: Optional[Dict[str, tuple]] = None, optimizer: str = "adagrad", learning_rate: float = 0.01,
                 initial_accumulator_value: float = 0.1, filter_freq: int = 0, steps_to_live: int = 0, pad_key: int = -1, seed: int = 1234,
                 max_rows_per_table: int = 1 << 25, device=None, rank: int = 0, world_size: int = 1, comm=None, loss_fn: Optional[Callable] = None,
                 tiered: Optional[Dict[int, dict]] = None, micro_batch_num: int = 1):
        """net: dense module (its parameters are trained); forward_fn(net, dense: dict of static tensors, emb [B, C, D] bf16, ids [C, B]) -> logits [B].
        col_table[c]: table of id column c; table_rows[t]: expected distinct keys of table t (pre-sizing hint, tables grow).
        tiered: {table: {"cache_rows": R, "strategy": 0 (LFU) | 1 (LRU)}} -- those tables keep at most ~R rows PER RANK in HBM over a host DRAM tier
        (ops/tier_manager.py): call ``prefetch(next_ids)`` one batch ahead with this rank's next id columns.  With world_size > 1 every rank holds
        both tiers of the keys it owns and the owners find their keys in every rank's next batch over peer memory (tier_kernels.cu:
        k_tier_publish / k_tier_wait / k_tier_miss_list_mp) -- ``prefetch`` is then a collective, like ``train_step``.
        micro_batch_num: auto micro-batch (graph_execution_state.cc:635-729, ConfigProto.micro_batch_num): the DENSE net's forward + backward run
        over M slices of the batch inside the same step (same CUDA graph), parameter gradients accumulate, one optimizer step -- peak activation
        memory / M.  The sparse pipeline still runs ONCE per step on the whole batch: dedup gets better with batch size, and its buffers are static."""
        self.net, self.forward_fn = net, forward_fn
        self.rank, self.world, self.comm = rank, world_size, comm
        self.emu = _native.emu_active()              # CPU CI: the same step on the CUDA-on-CPU emulation of the kernels (eager, no CUDA graph)
        self.dev = torch.device("cpu") if self.emu else (torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device()))
        self.lib = _native.cuda()
        if not self.emu:
            _native.set_device(self.dev.index)
        self.B, self.D, self.C, self.T = batch_size, embedding_dim, len(col_table), len(table_rows)
        self.kind = _OPT_KIND[optimizer.lower()]
        self.lr, self.init_acc = learning_rate, initial_accumulator_value
        self.loss_fn = loss_fn or (lambda logits, labels: nn.functional.binary_cross_entropy_with_logits(logits.float(), labels))
        self.launches, self._graph = 0, None
        self.micro = max(1, int(micro_batch_num))
        if batch_size % self.micro:
            raise ValueError(f"micro_batch_num {self.micro} must divide the batch size {batch_size}")
        dev = self.dev
        # ---- tables: this rank's hash(key) % world shard of every table
        self.ctx = get_context(dev, self.D, owner=id(self) & 0x7FFFFFFF)
        ns = _OPT_SLOTS[self.kind]
        slot_init = [initial_accumulator_value if self.kind in (OPT_ADAGRAD, OPT_ADAGRAD_DECAY, OPT_FTRL) else 0.0, 0.0, 0.0, 0.0]
        self.tables: Dict[int, DeviceTable] = {}
        g = torch.Generator()
        for t, card in enumerate(table_rows):
            card = int(card)
            if world_size > 1:
                card = card // world_size + card // (8 * world_size) + 1024
            c = EvConfig()
            c.dim, c.num_slots, c.has_scalars = self.D, ns, int(self.kind == OPT_ADAGRAD_DECAY)
            c.init_capacity = card
            c.filter_type, c.filter_freq = (1, filter_freq) if filter_freq > 0 else (0, 0)
            c.bloom_counter_bits = 32
            c.steps_to_live, c.l2_weight_threshold = steps_to_live, -1.0
            c.default_value_dim, c.default_value_no_permission = 4096, 0.0
            c.record_freq = c.record_version = 1
            c.storage_type = 1
            for i in range(4):
                c.slot_init[i] = slot_init[i]
            g.manual_seed(seed + 17 + 1000 * t)
            dm = torch.empty(4096, self.D).normal_(0.0, 1.0 / math.sqrt(self.D), generator=g)
            rows = max(1024, min(card, max_rows_per_table))
            if tiered and t in tiered:            # HBM tier = cache: R rows + head-room for the keys two steps can create before an eviction lands
                ncols_t = sum(1 for ct in col_table if ct == t)
                # (world > 1: a rank owns ~1/W of the W batches' keys -- the same expectation, plus slack for the imbalance of hash(key) % W)
                rows = int(tiered[t]["cache_rows"]) + (2 if world_size == 1 else 3) * ncols_t * batch_size + 4096
                card = rows
            cap = _next_pow2(max(2048, 2 * min(card, rows)))
            self.tables[t] = DeviceTable(c, dm, dev, capacity=cap, row_capacity=rows, owner=id(self) & 0x7FFFFFFF)
        self.tmap = torch.tensor([self.tables[t].gid for t in range(self.T)], dtype=torch.int32, device=dev)
        self.tiers = {}
        if tiered:
            if world_size > 1 and (comm is None or not hasattr(comm, "symmetric")):
                raise ValueError("tiered tables with world_size > 1 need a peer-memory communicator (parallel.p2p.P2PComm)")
            from ..ops.tier_manager import DeviceTierManager
            for t, o in sorted(tiered.items()):            # sorted: the symmetric allocations inside are collective calls
                cols = torch.tensor([c for c, ct in enumerate(col_table) if ct == t], dtype=torch.int64, device=dev)
                n_ids = int(cols.numel()) * batch_size
                mgr = DeviceTierManager(self.tables[t], int(o["cache_rows"]), strategy=int(o.get("strategy", 0)), pad_key=pad_key,
                                        max_batch_keys=max(1 << 16, (2 if world_size == 1 else 4) * n_ids),
                                        comm=comm if world_size > 1 else None, ids_per_prefetch=n_ids)
                self.tiers[t] = (mgr, cols)
        self._host_step = 0
        # ---- sparse pipeline + static buffers
        self.sp = SparsePipeline(dev, rank, world_size, list(col_table), self.T, batch_size, self.D, comm=comm, pad_key=pad_key)
        self.ids = torch.full((self.C, batch_size), pad_key, dtype=torch.int64, device=dev)
        self.labels = torch.zeros(batch_size, dtype=torch.float32, device=dev)
        self.dense: Dict[str, torch.Tensor] = {k: torch.zeros(*shape, dtype=dt, device=dev) for k, (shape, dt) in (dense_inputs or {}).items()}
        self.emb_out = torch.zeros(batch_size, self.C, self.D, dtype=torch.bfloat16, device=dev)
        self.demb = torch.zeros(self.C, batch_size, self.D, dtype=torch.bfloat16, device=dev)
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.max_unique = max(1, self.sp.Btot * min(world_size, 2))
        self.ctx.ensure(self.max_unique)
        self.ctx.claimed_upper = 0
        # ---- dense parameters / gradients -> one flat buffer each
        self.net.to(dev)
        plist = [p for p in self.net.parameters() if p.requires_grad]
        al = lambda n: (n + 63) // 64 * 64           # every parameter starts 256 B aligned (vectorised loads in the GEMM / pack kernels, cuBLAS)
        self.P = sum(al(p.numel()) for p in plist)
        self.params = torch.zeros(self.P, dtype=torch.float32, device=dev)
        self.grads = torch.zeros(self.P, dtype=torch.float32, device=dev) if comm is None else comm.alloc_grads(self.P)
        o, views = 0, []
        for p in plist:
            n = p.numel()
            self.params[o:o + n].copy_(p.detach().float().flatten())
            p.data = self.params[o:o + n].view_as(p)
            views.append(self.grads[o:o + n].view_as(p))
            o += al(n)
        # gradients: autograd allocates .grad itself (from the CUDA graph's private pool once captured -- pre-set .grad views created on
        # another stream make AccumulateGrad insert cross-stream waits that cannot be captured); ONE multi-tensor copy per step packs
        # them into the flat (symmetric, with world > 1) buffer the fused optimizer / all-reduce kernel reads
        self._plist, self._gviews = plist, views
        if world_size > 1:      # identical replicas: rank 0's initial values everywhere
            if hasattr(comm, "host_broadcast"):              # emulation: ranks are threads of this process (parallel/emu_comm.py)
                comm.host_broadcast([self.params] + list(self.net.buffers()))
            else:
                import torch.distributed as dist
                dist.broadcast(self.params, 0)
                for b in self.net.buffers():
                    dist.broadcast(b, 0)
        self.s0 = torch.full((self.P,), initial_accumulator_value if self.kind in (OPT_ADAGRAD, OPT_ADAGRAD_DECAY, OPT_FTRL) else 0.0,
                             dtype=torch.float32, device=dev) if ns > 0 else None
        self.s1 = torch.zeros(self.P, dtype=torch.float32, device=dev) if ns > 1 else None
        hp = OptHyper()
        hp.kind, hp.lr = self.kind, learning_rate
        hp.beta1, hp.beta2, hp.epsilon = 0.9, 0.999, 1e-8
        hp.beta1_power, hp.beta2_power = 0.9, 0.999
        hp.weight_decay, hp.l1, hp.l2, hp.l2_shrinkage, hp.lr_power = 0.0, 0.0, 0.0, 0.0, -0.5
        hp.decay_rate, hp.decay_baseline, hp.init_accum = 0.9, initial_accumulator_value, initial_accumulator_value
        hp.decay_step, hp.global_step = 100000, 0
        self.ctx.set_hyper(hp)
        self.hp_dev = self.ctx.hp_dev
        _native.device_sync(dev)

    # ------------------------------------------------------------------------------------------------------------------
    def _s(self):
        return None if self.emu else C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def _sparse_forward(self, train: bool) -> None:
        self.sp.dedup(self.ids)
        self.sp.lookup(self.ctx, self.tmap, train)
        self.sp.gather(self.emb_out)                  # waits for every owner's ROWS flag in-kernel
        self.launches += 3

    def _sparse_backward(self) -> None:
        self.sp.segsum(self.demb)
        self.sp.reset()
        self.sp.grad(self.ctx, self.tmap)
        _chk(self.lib.dr_cuda_sparse_apply(ptr(self.ctx.structs()), ptr(self.ctx.ulist), ptr(self.ctx.nuniq), self.ctx.ulist.numel(), ptr(self.ctx.gsum),
                                           self.D, ptr(self.hp_dev), self.max_unique, 1, self._s()), "sparse_apply")
        self.launches += 5

    def _step_body(self) -> None:
        for p in self._plist:
            p.grad = None
        # sparse forward outside autograd; the gathered [B, C, D] activation enters the dense net's graph as a leaf whose .grad is what
        # the sparse backward consumes (no custom autograd.Function inside the captured backward)
        self._sparse_forward(True)
        if self.micro == 1:
            emb = self.emb_out.detach().requires_grad_(True)
            logits = self.forward_fn(self.net, self.dense, emb, self.ids)
            loss = self.loss_fn(logits, self.labels) / self.world
            self.loss.copy_(loss.detach().reshape(1))
            loss.backward()
            self.demb.copy_(emb.grad.permute(1, 0, 2))      # [B, C, D] -> feature-major bf16 [C, B, D] (what k_sp_segsum reads coalesced)
        else:                                               # auto micro-batch: slices of the gathered activation, gradients accumulate in .grad
            mb = self.B // self.micro
            self.loss.zero_()
            for m in range(self.micro):
                lo, hi = m * mb, (m + 1) * mb
                emb = self.emb_out[lo:hi].detach().requires_grad_(True)
                logits = self.forward_fn(self.net, {k: v[lo:hi] for k, v in self.dense.items()}, emb, self.ids[:, lo:hi])
                loss = self.loss_fn(logits, self.labels[lo:hi]) / (self.world * self.micro)       # mean over the whole batch = mean of the slice means
                self.loss.add_(loss.detach().reshape(1))
                loss.backward()
                self.demb[:, lo:hi].copy_(emb.grad.permute(1, 0, 2))
        self._sparse_backward()
        # (the gather kernel of this step waited for every owner's ROWS flag, so every peer has finished last step's all-reduce reads
        #  of the flat gradient buffer: it may be overwritten now)
        torch._foreach_copy_(self._gviews, [p.grad if p.grad is not None else torch.zeros_like(p) for p in self._plist])
        if self.comm is not None:
            self.comm.dense_allreduce_update(self)
        else:
            _chk(self.lib.dr_cuda_dense_apply(ptr(self.params), ptr(self.grads), ptr(self.s0) if self.s0 is not None else None,
                                              ptr(self.s1) if self.s1 is not None else None, self.P, ptr(self.hp_dev), 1.0, 0, None, self._s()), "dense_apply")
            self.launches += 1
        _chk(self.lib.dr_cuda_advance_hyper(ptr(self.hp_dev), self._s()), "advance_hyper")
        self.sp.step_end()
        self.launches += 2

    # ------------------------------------------------------------------------------------------------------------------
    def load_batch(self, ids: torch.Tensor, labels: torch.Tensor, dense: Optional[Dict[str, torch.Tensor]] = None, non_blocking: bool = True) -> None:
        """ids: int64 [C, B] id columns (sequence features: one column per position, ``pad_key`` = padding)."""
        self.ids.copy_(ids, non_blocking=non_blocking)
        self.labels.copy_(labels, non_blocking=non_blocking)
        for k, v in (dense or {}).items():
            self.dense[k].copy_(v, non_blocking=non_blocking)

    def train_step_eager(self) -> None:
        self._step_body()

    def capture(self, warmup: int = 3) -> None:
        """Three eager steps on a side stream (autograd / allocator warm-up; they DO train on the loaded batch), then the whole step
        is captured into one CUDA graph."""
        if self.emu:                                  # kernels run synchronously on the host: the eager step IS the step
            for _ in range(warmup):
                self._step_body()
            self.launches_per_step = 0
            return
        cur = torch.cuda.current_stream(self.dev)
        side = torch.cuda.Stream(device=self.dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._step_body()
        cur.wait_stream(side)
        torch.cuda.synchronize(self.dev)
        n0 = self.launches
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._step_body()
        self.launches_per_step = self.launches - n0
        self._graph = g

    def prefetch(self, next_ids: torch.Tensor) -> None:
        """Multi-tier tables: hand the id columns of the NEXT batch (device [C, B]) to the tier managers while this step runs."""
        for mgr, cols in self.tiers.values():
            mgr.prefetch(next_ids.index_select(0, cols).contiguous())

    def train_step(self) -> None:
        for mgr, _ in self.tiers.values():
            mgr.commit(self._host_step)          # promoted rows resident / cold rows demoted before the step's kernels are launched
        self._host_step += 1
        if self._graph is not None:
            self._graph.replay()
        else:
            self.train_step_eager()

    @torch.no_grad()
    def predict(self) -> torch.Tensor:
        """Forward only (tables read-only; BatchNorm in eval mode)."""
        was = self.net.training
        self.net.eval()
        self._sparse_forward(False)
        out = torch.sigmoid(self.forward_fn(self.net, self.dense, self.emb_out, self.ids).float())
        self.sp.reset()
        if self.world > 1:
            self.sp.signal(3)
            self.comm.wait_dense(self.sp)
        self.sp.step_end()
        self.net.train(was)
        return out

    # ---- training-state checkpoints (checkpoint/engine_ckpt.py): full / incremental save, restore under any world size ----------
    def save(self, save_path: str, incremental: bool = False, max_to_keep: int = 5) -> str:
        from ..checkpoint.engine_ckpt import save_engine
        return save_engine(self, save_path, incremental=incremental, max_to_keep=max_to_keep)

    def restore(self, save_path: str, step=None, replay_incremental: bool = True) -> int:
        from ..checkpoint.engine_ckpt import restore_engine
        return restore_engine(self, save_path, step=step, replay_incremental=replay_incremental)

    def loss_value(self, global_mean: bool = True) -> float:
        v = self.loss.clone()
        if global_mean and self.world > 1:
            if hasattr(self.comm, "host_all_reduce"):
                self.comm.host_all_reduce(v)
            else:
                import torch.distributed as dist
                dist.all_reduce(v)
        return float(v.item())


# ---- adapters for the model zoo ------------------------------------------------------------------------------------------------
def criteo_engine(model, batch_size: int, table_rows: Optional[Sequence[int]] = None, **kw) -> FusedRecEngine:
    """Any :class:`models.zoo.CriteoModel` (DeepFM, WDL, DCN, DCNv2, MaskNet, DLRM-DCN): 13 dense + 26 id columns, one table each."""
    T = model.num_sparse
    rows = list(table_rows) if table_rows is not None else [1_000_000] * T
    dense_net = _StripTables(model)

    def fwd(net, dense, emb, ids):
        # bf16 activations end to end (wgmma FusedMLP in / out, BatchNorm, FM kernel); fp32 master weights; the loss is taken in fp32
        with torch.autocast(emb.device.type, dtype=torch.bfloat16):
            return net.inner.logits(dense["dense"].to(torch.bfloat16), emb)
    return FusedRecEngine(dense_net, fwd, list(range(T)), rows, batch_size, embedding_dim=model.emb_dim,
                          dense_inputs={"dense": ((batch_size, model.num_dense), torch.float32)}, **kw)


def din_engine(model, batch_size: int, max_len: int = 50, table_rows: Sequence[int] = (10_000_000, 100_000_000, 10_000), **kw) -> FusedRecEngine:
    """:class:`models.zoo.DIN`: id columns = [user | item | cat | hist_item x L | hist_cat x L] over the three tables (user, item, cat);
    the history positions are columns of the item / category tables, padding (-1) gives zero rows and the attention mask."""
    L = max_len
    col_table = [0, 1, 2] + [1] * L + [2] * L
    dense_net = _StripTables(model)

    def fwd(net, dense, emb, ids):
        u = emb[:, 0]
        q = torch.cat([emb[:, 1], emb[:, 2]], -1)
        k = torch.cat([emb[:, 3:3 + L], emb[:, 3 + L:3 + 2 * L]], -1)             # [B, L, 2D] bf16 (padding rows are already zero)
        mask = (ids[3:3 + L] >= 0).t()
        with torch.autocast(emb.device.type, dtype=torch.bfloat16):
            return net.inner.head(u, q, k, mask)
    return FusedRecEngine(dense_net, fwd, col_table, list(table_rows), batch_size, embedding_dim=model.emb_dim, **kw)


def din_ids(batch: Dict[str, torch.Tensor]) -> torch.Tensor:
    """Taobao-shaped batch dict -> the [3 + 2 L, B] id-column block :func:`din_engine` expects (run it in the input pipeline)."""
    return torch.cat([batch["user"][None], batch["item"][None], batch["cat"][None], batch["hist_item"].t(), batch["hist_cat"].t()], 0).contiguous()


class _StripTables(nn.Module):
    """Wraps a zoo model so that only its DENSE parameters are registered (the EmbeddingVariables are replaced by the engine's tables)."""

    def __init__(self, model: nn.Module):
        super().__init__()
        if hasattr(model, "wide"):
            raise ValueError("models with a second (wide) embedding group are not supported by FusedRecEngine yet")
        for name in ("emb", "user", "item", "cat"):
            if hasattr(model, name) and isinstance(getattr(model, name), nn.Module):
                try:
                    delattr(model, name)
                except AttributeError:
                    pass
        self.inner = model
