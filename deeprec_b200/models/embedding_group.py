"""EmbeddingGroup -- the sparse half of the fused engines (models/dlrm_engine.py, models/rec_engine.py): a set of tables trained by one
optimizer, i.e. this rank's shard of every table, their step context, device-resident hyper-parameters and (unique-first placement) the
:class:`parallel.sparse_pipeline.SparsePipeline`.  A linear group (``is_linear``, Wide & Deep's wide part) takes one fp32 gradient per sample
(``linear_bwd``) in place of per-sample rows (``segsum``).  Every method counts the kernels it launches; so does the pipeline.
Also here: the helpers both engines share."""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional, Sequence

import torch

from .. import _native
from .._native import EvConfig, check, ptr, stream_ptr
from ..ops.device_table import DeviceTable, _next_pow2, get_context
from ..optim.optimizers import OPT_ADAGRAD_DECAY, OPT_SLOTS, engine_hyper, slot0_init
from ..parallel.sparse_pipeline import CH_DENSE, Bags, SparsePipeline


_no_tick = lambda name: None          # noqa: E731  (phase markers: DLRMEngine._tick)


class EmbeddingGroup:
    def __init__(self, dev: torch.device, dim: int, kind: int, learning_rate: float, initial_accumulator_value: float, owner: int, seed: int,
                 tables: Sequence[int], table_rows: Sequence[int], batch_size: int, col_table: Optional[Sequence[int]] = None, rank: int = 0,
                 world: int = 1, comm=None, pad_key: int = -1, filter_freq: int = 0, steps_to_live: int = 0, max_rows_per_table: int = 1 << 25,
                 tiered: Optional[Dict[int, dict]] = None, is_linear: bool = False, bags: Optional[Sequence[tuple]] = None):
        """tables: the tables this rank holds; table_rows[t]: expected distinct keys of table t (pre-sizing hint, tables grow).  col_table[c]:
        table of id column c -- unique-first: a pipeline over the id columns, the hash(key) % world shard of every table; None: table-wise
        placement, whole tables, no pipeline.  owner: key of the step context (one per group).  tiered: as FusedRecEngine's.
        bags: ``(n_cols, combiner)`` multi-hot bags over the id columns (``parallel.sparse_pipeline.Bags``): the group's activation is pooled
        per bag (``pool``) and its backward takes the pooled gradient [F, B, dim] (``pool_segsum``)."""
        self.dev, self.dim, self.is_linear, self.world, self.comm = dev, dim, is_linear, world, comm
        self.lib = _native.cuda()
        self._launches = 0
        self.ctx = get_context(dev, dim, owner=owner)
        self.tables = self._build_tables(kind, initial_accumulator_value, owner, seed, tables, table_rows, batch_size, col_table, tiered,
                                         filter_freq, steps_to_live, max_rows_per_table)
        self.tmap = torch.tensor([self.tables[t].gid for t in tables], dtype=torch.int32, device=dev)
        self.tiers = {}
        if tiered:
            if world > 1 and (comm is None or not hasattr(comm, "symmetric")):
                raise ValueError("tiered tables with world_size > 1 need a peer-memory communicator (parallel.p2p.P2PComm)")
            from ..ops.tier_manager import DeviceTierManager
            for t, o in sorted(tiered.items()):            # sorted: the symmetric allocations inside are collective calls
                cols = torch.tensor([c for c, ct in enumerate(col_table) if ct == t], dtype=torch.int64, device=dev)
                n_ids = int(cols.numel()) * batch_size
                mgr = DeviceTierManager(self.tables[t], int(o["cache_rows"]), strategy=int(o.get("strategy", 0)), pad_key=pad_key,
                                        max_batch_keys=max(1 << 16, (2 if world == 1 else 4) * n_ids),
                                        comm=comm if world > 1 else None, ids_per_prefetch=n_ids)
                self.tiers[t] = (mgr, cols)
        if col_table is not None:
            self.sp = SparsePipeline(dev, rank, world, list(col_table), len(table_rows), batch_size, dim, comm=comm, pad_key=pad_key)
            self.max_unique = max(1, self.sp.Btot * min(world, 2))      # distinct keys a step can bring to this rank (overflow is flagged, not UB)
        else:
            self.sp = None
            self.max_unique = max(1, len(tables) * world * batch_size)
        self.bags = self.pool_w = None
        if bags is not None:
            if is_linear or self.sp is None:
                raise ValueError("bags need a deep group over a unique-first pipeline")
            self.bags = Bags(dev, bags, self.sp.C)
            self.pool_w = torch.zeros(self.bags.F, batch_size, dtype=torch.float32, device=dev)    # per-(bag, sample) factor of the pooling
        self.ctx.ensure(self.max_unique)
        self.ctx.claimed_upper = 0
        self.ctx.set_hyper(engine_hyper(kind, learning_rate, initial_accumulator_value))
        self.hp_dev = self.ctx.hp_dev

    def _build_tables(self, kind, init_acc, owner, seed, tables, table_rows, batch_size, col_table, tiered, filter_freq, steps_to_live,
                      max_rows_per_table) -> Dict[int, DeviceTable]:
        """Default rows normal(0, 1/sqrt(dim)) seeded per table: a key's initial value never depends on the sharding."""
        dim, W = self.dim, self.world
        ns = OPT_SLOTS[kind]
        slot_init = [slot0_init(kind, init_acc), 0.0, 0.0, 0.0]
        out: Dict[int, DeviceTable] = {}
        g = torch.Generator()
        for t in tables:
            card = int(table_rows[t])
            if col_table is not None and W > 1:
                card = card // W + card // (8 * W) + 1024           # this rank's hash(key) % world shard (+ hash imbalance slack)
            c = EvConfig()
            c.dim, c.num_slots, c.has_scalars = dim, ns, int(kind == OPT_ADAGRAD_DECAY)
            c.init_capacity = card
            c.filter_type, c.filter_freq = (1, filter_freq) if filter_freq > 0 else (0, 0)
            c.bloom_counter_bits = 32
            c.steps_to_live, c.l2_weight_threshold = steps_to_live, -1.0
            c.default_value_dim, c.default_value_no_permission = 4096, 0.0
            c.record_freq = c.record_version = 1
            c.storage_type = 1
            for i in range(4):
                c.slot_init[i] = slot_init[i]
            g.manual_seed(seed + 1000 * t)
            dm = torch.empty(4096, dim).normal_(0.0, 1.0 / math.sqrt(dim), generator=g)
            rows = max(1024, min(card, max_rows_per_table))
            if tiered and t in tiered:            # HBM tier = cache: R rows + head-room for the keys two steps can create before an eviction lands
                ncols_t = sum(1 for ct in col_table if ct == t)
                # (world > 1: a rank owns ~1/W of the W batches' keys -- the same expectation, plus slack for the imbalance of hash(key) % W)
                rows = int(tiered[t]["cache_rows"]) + (2 if W == 1 else 3) * ncols_t * batch_size + 4096
                card = rows
            cap = _next_pow2(max(2048, 2 * min(card, rows)))
            out[t] = DeviceTable(c, dm, self.dev, capacity=cap, row_capacity=rows, owner=owner)
        return out

    @property
    def launches(self) -> int:
        return self._launches + (self.sp.launches if self.sp is not None else 0)

    # ---- one step ------------------------------------------------------------------------------------------------------------------
    def forward(self, ids: torch.Tensor, train: bool, tick: Callable[[str], None] = _no_tick) -> None:
        """Requester: dedup + bucket the id columns.  Owner: probe (+admit/claim) the distinct keys of every source and push their rows."""
        self.sp.dedup(ids)
        tick("e_dedup")
        self.sp.lookup(self.ctx, self.tmap, train)

    def backward(self, grad: torch.Tensor, tick: Callable[[str], None] = _no_tick) -> None:
        """grad: the per-sample gradient rows (bf16 [C, B, dim]; with bags the pooled rows [F, B, dim]), or for a linear group the gradient of
        every sample's linear logit (fp32 [B]).  Requester: pre-reduce it per distinct key.  Owner: pull the sources' per-key gradients, then the
        row-wise optimizer."""
        if self.is_linear:
            self.sp.linear_bwd(grad)
        elif self.bags is not None:
            self.sp.pool_segsum(grad, self.pool_w, self.bags)
        else:
            self.sp.segsum(grad)
        tick("g_segsum")
        self.sp.reset()                  # every owner has read my bucket lists / counts (ROWS flags seen by the gather)
        tick("g_reset")
        self.sp.grad(self.ctx, self.tmap)
        tick("g_grad")
        self.apply()

    def apply(self) -> None:
        """Row-wise optimizer over this step's distinct keys (k_apply), then the distinct-key counter restarts (k_reset_counter)."""
        c = self.ctx
        check(self.lib.dr_cuda_sparse_apply(ptr(c.structs()), ptr(c.ulist), ptr(c.nuniq), c.ulist.numel(), ptr(c.gsum), self.dim, ptr(self.hp_dev),
                                            self.max_unique, 1, stream_ptr(self.dev)), "sparse_apply")
        self._launches += 2

    def end_step(self) -> None:
        """Global step / beta powers / decay of the hyper-parameters in device memory, then the pipeline's step boundary."""
        check(self.lib.dr_cuda_advance_hyper(ptr(self.hp_dev), stream_ptr(self.dev)), "advance_hyper")
        self._launches += 1
        if self.sp is not None:
            self.sp.step_end()

    def rendezvous(self) -> None:
        """world > 1: raise this pipeline's DENSE flags and wait for every rank's -- no rank starts its next dedup (which zeroes the ugrad rows
        the owners pull) before every owner has finished this step's pull."""
        if self.world > 1:
            self.sp.signal(CH_DENSE)
            self.comm.wait_dense(self.sp)

    def forward_only_tail(self) -> None:
        """Close a forward-only pass (tables read-only): the bucket lists are free again once every rank has passed the rendezvous."""
        self.sp.reset()
        self.rendezvous()
        self.sp.step_end()


# ---- shared by the engines -------------------------------------------------------------------------------------------------------------
def engine_launches(eng) -> int:
    """Kernel launches of an engine so far: its own dense kernels (and replayed graphs), its groups' and its communicator's."""
    return eng._launches + sum(g.launches for g in eng.groups) + getattr(eng.comm, "launches", 0)


def loss_value(eng, global_mean: bool = True) -> float:
    """Loss of the last step: the mean over the GLOBAL batch (each rank holds its partial sum / (B * world))."""
    v = eng.loss.clone()
    if global_mean and eng.world > 1:
        if hasattr(eng.comm, "host_all_reduce"):          # emulation: ranks are threads (parallel/emu_comm.py)
            eng.comm.host_all_reduce(v)
        else:
            import torch.distributed as dist
            dist.all_reduce(v)
    return float(v.item())
