"""FusedRecEngine -- one CUDA-graph training step for ANY dense network over the unique-first sparse pipeline.

:class:`models.dlrm_engine.DLRMEngine` hand-schedules DLRM's dense net; this engine generalises the same execution design to the
rest of the model zoo (DeepFM: BASELINE config #3, DIN: config #4, WDL, and any ``nn.Module`` that maps ``(dense inputs, embeddings
[B, C, D])`` to logits):

  * embeddings: every table row-sharded over the ranks (hash(key) % world), id columns deduplicated on the requester, distinct keys
    probed / inserted / admitted by their owners, rows pushed over NVLink, gradients pre-reduced per key and pulled by the owners,
    row-wise optimizer on the device table (``parallel/sparse_pipeline.py``) -- sequence features are just more id columns of the
    same table (``col_table``), padding ids (-1) produce zero rows and no statistics;
  * dense net: the module's own autograd graph (``nn.FusedMLP`` -> wgmma GEMMs), parameters and gradients re-pointed into ONE flat
    fp32 buffer each, so the optimizer is one fused kernel -- with ``world > 1`` the in-kernel-synchronised one-shot all-reduce +
    optimizer of ``parallel/p2p.py`` over the symmetric gradient buffer;
  * optional linear group (``linear=True``, Wide & Deep's wide part, reference modelzoo/wide_and_deep/train.py:271-288): dim-4 tables over the
    same id columns on a second pipeline with its own optimizer; the per-sample sum of element 0 of the rows is read in place from the unique
    rows (``k_sp_linear_fwd``) and handed to the dense net as ``linear=`` (fp32 [B]); its gradient goes straight back into the per-key
    fixed-point sums (``k_sp_linear_bwd``) -- no [B, C, 4] activation, no bf16 rounding of the per-sample gradient;
  * the whole step (forward, backward, both optimizers, flag protocol) is captured into ONE CUDA graph after three eager warm-up
    steps -- per-module Python / launch overhead, the reason the framework-API path ran DeepFM at 0.70 M samples/s, disappears.

Reference: modelzoo/deepfm/train.py:143-191, modelzoo/din/train.py:143-375 (models); group_embedding_lookup_sparse + SOK
(python/ops/embedding_ops.py:1594-1930) for the lookup they sit on.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Sequence

import torch
from torch import nn

from .. import _native
from .._native import check, ptr, stream_ptr
from ..checkpoint.engine_ckpt import restore_engine, save_engine
from ..optim.optimizers import OPT_KIND, OPT_SLOTS, slot0_init
from . import embedding_group as _eg
from .embedding_group import EmbeddingGroup


class FusedRecEngine:
    def __init__(self, net: nn.Module, forward_fn: Callable[..., torch.Tensor], col_table: Sequence[int], table_rows: Sequence[int], batch_size: int,
                 embedding_dim: int = 16, dense_inputs: Optional[Dict[str, tuple]] = None, optimizer: str = "adagrad", learning_rate: float = 0.01,
                 initial_accumulator_value: float = 0.1, filter_freq: int = 0, steps_to_live: int = 0, pad_key: int = -1, seed: int = 1234,
                 max_rows_per_table: int = 1 << 25, device=None, rank: int = 0, world_size: int = 1, comm=None, loss_fn: Optional[Callable] = None,
                 tiered: Optional[Dict[int, dict]] = None, micro_batch_num: int = 1, linear: bool = False, linear_optimizer: Optional[str] = None,
                 linear_learning_rate: Optional[float] = None, bags: Optional[Sequence[tuple]] = None, label_dim: int = 1):
        """net: dense module (its parameters are trained); forward_fn(net, dense: dict of static tensors, emb [B, C, D] bf16, ids [C, B]) -> logits [B].
        col_table[c]: table of id column c; table_rows[t]: expected distinct keys of table t (pre-sizing hint, tables grow).
        tiered: {table: {"cache_rows": R, "strategy": 0 (LFU) | 1 (LRU)}} -- those tables keep at most ~R rows PER RANK in HBM over a host DRAM tier
        (ops/tier_manager.py): call ``prefetch(next_ids)`` one batch ahead with this rank's next id columns.  With world_size > 1 every rank holds
        both tiers of the keys it owns and the owners find their keys in every rank's next batch over peer memory (tier_kernels.cu:
        k_tier_publish / k_tier_wait / k_tier_miss_list_mp) -- ``prefetch`` is then a collective, like ``train_step``.
        micro_batch_num: auto micro-batch (graph_execution_state.cc:635-729, ConfigProto.micro_batch_num): the DENSE net's forward + backward run
        over M slices of the batch inside the same step (same CUDA graph), parameter gradients accumulate, one optimizer step -- peak activation
        memory / M.  The sparse pipeline still runs ONCE per step on the whole batch: dedup gets better with batch size, and its buffers are static.
        linear: a second, linear embedding group (the wide part of Wide & Deep): one dim-4 table per table of ``col_table`` over the same id columns,
        of which element 0 is the weight of an id.  Every step computes the per-sample sum of those weights in fp32 (``linear_fwd``, read in place from
        the unique rows) and hands it to ``forward_fn`` as the keyword ``linear=`` (fp32 [B], a leaf whose gradient trains the group); without the
        group forward_fn is called without it.  The group has its own optimizer: ``linear_optimizer`` / ``linear_learning_rate`` (None: the same as
        the deep tables), e.g. FTRL at 0.2 as the reference trains Wide & Deep's linear part.  Linear tables are single-tier.
        bags: multi-hot id bags, a list of ``(n_cols, combiner)`` over the id columns in order (the counts sum to C; combiner ``sum | mean |
        sqrtn``, padding neither adds nor counts).  Bag f pools its columns into slot f of the activation, which is then [B, F, D]: forward_fn
        receives that, and its gradient goes back to every column of the bag (``k_sp_pool`` / ``k_sp_pool_segsum``, in place of gather / segsum).
        Not combined with ``linear``.
        label_dim: labels are [B] (1) or [B, label_dim]; forward_fn may return a dict of logits, which ``loss_fn`` then receives and of which
        ``predict()`` returns the sigmoids."""
        if linear and bags is not None:
            raise ValueError("FusedRecEngine: bags with linear=True (a wide part over pooled bags) is not supported")
        self.net, self.forward_fn = net, forward_fn
        self.rank, self.world, self.comm = rank, world_size, comm
        self.emu = _native.emu_active()              # CPU CI: the same step on the CUDA-on-CPU emulation of the kernels (eager, no CUDA graph)
        self.dev = torch.device("cpu") if self.emu else (torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device()))
        self.lib = _native.cuda()
        if not self.emu:
            _native.set_device(self.dev.index)
        self.B, self.D, self.C, self.T = batch_size, embedding_dim, len(col_table), len(table_rows)
        self.kind = OPT_KIND[optimizer.lower()]
        self.loss_fn = loss_fn or (lambda logits, labels: nn.functional.binary_cross_entropy_with_logits(logits.float(), labels))
        self._launches, self._graph = 0, None
        self.micro = max(1, int(micro_batch_num))
        if batch_size % self.micro:
            raise ValueError(f"micro_batch_num {self.micro} must divide the batch size {batch_size}")
        dev = self.dev
        # ---- embedding groups: this rank's hash(key) % world shard of every table, each group with its own step context (owner key),
        #      optimizer and pipeline
        owner = id(self) & 0x7FFFFFFF
        group = lambda dim, kind, lr, owner, seed, tiered, is_linear, bags=None: EmbeddingGroup(
            dev, dim, kind, lr, initial_accumulator_value, owner, seed, range(self.T), table_rows, batch_size, col_table=col_table, rank=rank,
            world=world_size, comm=comm, pad_key=pad_key, filter_freq=filter_freq, steps_to_live=steps_to_live,
            max_rows_per_table=max_rows_per_table, tiered=tiered, is_linear=is_linear, bags=bags)
        self.deep = group(self.D, self.kind, learning_rate, owner, seed + 17, tiered, False, bags)
        self.tables, self.tiers, self.sp, self.hp_dev = self.deep.tables, self.deep.tiers, self.deep.sp, self.deep.hp_dev
        self._host_step = 0
        # ---- static buffers
        self.ids = torch.full((self.C, batch_size), pad_key, dtype=torch.int64, device=dev)
        self.labels = torch.zeros((batch_size,) if label_dim == 1 else (batch_size, label_dim), dtype=torch.float32, device=dev)
        self.dense: Dict[str, torch.Tensor] = {k: torch.zeros(*shape, dtype=dt, device=dev) for k, (shape, dt) in (dense_inputs or {}).items()}
        slots = self.C if self.deep.bags is None else self.deep.bags.F      # activation rows per sample: id columns, or pooled bags
        self.emb_out = torch.zeros(batch_size, slots, self.D, dtype=torch.bfloat16, device=dev)
        self.demb = torch.zeros(slots, batch_size, self.D, dtype=torch.bfloat16, device=dev)
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
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
        ns = OPT_SLOTS[self.kind]
        self.s0 = torch.full((self.P,), slot0_init(self.kind, initial_accumulator_value), dtype=torch.float32, device=dev) if ns > 0 else None
        self.s1 = torch.zeros(self.P, dtype=torch.float32, device=dev) if ns > 1 else None
        # ---- linear group: dim-4 tables over the same id columns, owner key distinct from the deep group's (whatever its dim)
        self.linear = None
        if linear:
            self.linear = group(4, OPT_KIND[(linear_optimizer or optimizer).lower()], learning_rate if linear_learning_rate is None else linear_learning_rate,
                                -1 - owner, seed + 29, None, True)
            self.lin_tables, self.lin_hp_dev = self.linear.tables, self.linear.hp_dev
            self.lin_out = torch.zeros(batch_size, dtype=torch.float32, device=dev)
            self.lin_dlogit = torch.zeros(batch_size, dtype=torch.float32, device=dev)
        self.groups = [self.deep] + ([self.linear] if linear else [])
        _native.device_sync(dev)

    launches = property(_eg.engine_launches)
    loss_value = _eg.loss_value
    save, restore = save_engine, restore_engine      # training-state checkpoints: full / incremental save, restore under any world size

    # ------------------------------------------------------------------------------------------------------------------
    def _sparse_forward(self, train: bool) -> None:
        self.deep.forward(self.ids, train)
        if self.deep.bags is not None:                # both wait for every owner's ROWS flag in-kernel
            self.sp.pool(self.emb_out, self.deep.pool_w, self.deep.bags)
        else:
            self.sp.gather(self.emb_out)
        if self.linear:
            self.linear.forward(self.ids, train)
            self.linear.sp.linear_fwd(self.lin_out)   # waits for every owner's ROWS flag in-kernel

    def _sparse_backward(self) -> None:
        self.deep.backward(self.demb)
        if self.linear:
            self.linear.backward(self.lin_dlogit)
            self.linear.rendezvous()                  # the deep pipeline's DENSE flags are raised with the dense all-reduce

    def _linear_leaf(self, lo: int, hi: int):
        """The linear logits of samples [lo, hi) as a leaf of the dense net's graph, and the keyword that hands it to forward_fn."""
        if not self.linear:
            return None, {}
        lin = self.lin_out[lo:hi].detach().requires_grad_(True)
        return lin, {"linear": lin}

    def _linear_grad(self, lin, lo: int, hi: int) -> None:
        if lin is None:
            return
        if lin.grad is None:                                # forward_fn did not use the linear logits
            self.lin_dlogit[lo:hi].zero_()
        else:
            self.lin_dlogit[lo:hi].copy_(lin.grad)

    def _step_body(self) -> None:
        for p in self._plist:
            p.grad = None
        # sparse forward outside autograd; the gathered [B, C, D] activation enters the dense net's graph as a leaf whose .grad is what
        # the sparse backward consumes (no custom autograd.Function inside the captured backward)
        self._sparse_forward(True)
        if self.micro == 1:
            emb = self.emb_out.detach().requires_grad_(True)
            lin, kw = self._linear_leaf(0, self.B)
            logits = self.forward_fn(self.net, self.dense, emb, self.ids, **kw)
            loss = self.loss_fn(logits, self.labels) / self.world
            self.loss.copy_(loss.detach().reshape(1))
            loss.backward()
            self.demb.copy_(emb.grad.permute(1, 0, 2))      # [B, C, D] -> feature-major bf16 [C, B, D] (what k_sp_segsum reads coalesced)
            self._linear_grad(lin, 0, self.B)
        else:                                               # auto micro-batch: slices of the gathered activation, gradients accumulate in .grad
            mb = self.B // self.micro
            self.loss.zero_()
            for m in range(self.micro):
                lo, hi = m * mb, (m + 1) * mb
                emb = self.emb_out[lo:hi].detach().requires_grad_(True)
                lin, kw = self._linear_leaf(lo, hi)
                logits = self.forward_fn(self.net, {k: v[lo:hi] for k, v in self.dense.items()}, emb, self.ids[:, lo:hi], **kw)
                loss = self.loss_fn(logits, self.labels[lo:hi]) / (self.world * self.micro)       # mean over the whole batch = mean of the slice means
                self.loss.add_(loss.detach().reshape(1))
                loss.backward()
                self.demb[:, lo:hi].copy_(emb.grad.permute(1, 0, 2))
                self._linear_grad(lin, lo, hi)
        self._sparse_backward()
        # (the gather kernel of this step waited for every owner's ROWS flag, so every peer has finished last step's all-reduce reads
        #  of the flat gradient buffer: it may be overwritten now)
        torch._foreach_copy_(self._gviews, [p.grad if p.grad is not None else torch.zeros_like(p) for p in self._plist])
        if self.comm is not None:
            self.comm.dense_allreduce_update(self)
        else:
            check(self.lib.dr_cuda_dense_apply(ptr(self.params), ptr(self.grads), ptr(self.s0) if self.s0 is not None else None,
                                               ptr(self.s1) if self.s1 is not None else None, self.P, ptr(self.hp_dev), 1.0, None, stream_ptr(self.dev)),
                  "dense_apply")
            self._launches += 1
        for g in self.groups:
            g.end_step()

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
                n0 = self.launches
                self._step_body()
            self.launches_per_step = self.launches - n0
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
    def predict(self):
        """Forward only (tables read-only; BatchNorm in eval mode): the sigmoid of the logits, a dict of them for a multi-output forward_fn."""
        was = self.net.training
        self.net.eval()
        self._sparse_forward(False)
        kw = {"linear": self.lin_out} if self.linear else {}
        logits = self.forward_fn(self.net, self.dense, self.emb_out, self.ids, **kw)
        out = {k: torch.sigmoid(v.float()) for k, v in logits.items()} if isinstance(logits, dict) else torch.sigmoid(logits.float())
        for g in self.groups:
            g.forward_only_tail()
        self.net.train(was)
        return out


# ---- adapters for the model zoo ------------------------------------------------------------------------------------------------
def criteo_engine(model, batch_size: int, table_rows: Optional[Sequence[int]] = None, **kw) -> FusedRecEngine:
    """Any :class:`models.zoo.CriteoModel` (DeepFM, WDL, DCN, DCNv2, MaskNet, DLRM-DCN): 13 dense + 26 id columns, one table each.  WDL's wide
    tables become the engine's linear group (``linear_optimizer`` / ``linear_learning_rate`` in ``kw`` train it with its own optimizer)."""
    T = model.num_sparse
    rows = list(table_rows) if table_rows is not None else [1_000_000] * T
    wide = hasattr(model, "wide")
    dense_net = _StripTables(model)

    def fwd(net, dense, emb, ids, linear=None):
        # bf16 activations end to end (wgmma FusedMLP in / out, BatchNorm, FM kernel); fp32 master weights; the loss is taken in fp32
        with torch.autocast(emb.device.type, dtype=torch.bfloat16):
            if linear is not None:                     # WDL: the wide logit is the engine's fp32 linear sum
                return net.inner.wide_deep_logits(dense["dense"].to(torch.bfloat16), emb, linear[:, None])
            return net.inner.logits(dense["dense"].to(torch.bfloat16), emb)
    return FusedRecEngine(dense_net, fwd, list(range(T)), rows, batch_size, embedding_dim=model.emb_dim,
                          dense_inputs={"dense": ((batch_size, model.num_dense), torch.float32)}, linear=wide, **kw)


def din_engine(model, batch_size: int, max_len: int = 50, table_rows: Sequence[int] = (10_000_000, 100_000_000, 10_000), **kw) -> FusedRecEngine:
    """:class:`models.zoo.DIN`, :class:`models.zoo.DIEN` and :class:`models.zoo.BST`: id columns = [user | item | cat | hist_item x L |
    hist_cat x L] over the three tables (user, item, cat); the history positions are columns of the item / category tables, padding (-1) gives
    zero rows and the attention mask.  DIEN's two GRUs run on :func:`nn.fused_gru`, which stops each sample after ``mask.sum(1)`` steps: its
    padding must be a tail (every id after the first -1 of a history is -1 too), as :func:`din_ids` of the project's Taobao-shaped batches
    gives.  BST's encoder block runs on :func:`nn.fused_encoder_layer` with the key mask [history mask | True]; its padding may sit anywhere.
    DIN's and DIEN's attention units run on :func:`nn.fused_din_attention`."""
    from ..nn import fused_din_attention, fused_encoder_layer, fused_gru
    from .zoo import BST, DIEN, DIN
    L = max_len
    col_table = [0, 1, 2] + [1] * L + [2] * L
    dense_net = _StripTables(model)
    kw_head = ({"gru": fused_gru, "attention": fused_din_attention} if isinstance(model, DIEN) else {"encoder": fused_encoder_layer}
               if isinstance(model, BST) else {"attention": fused_din_attention} if isinstance(model, DIN) else {})

    def fwd(net, dense, emb, ids):
        u = emb[:, 0]
        q = torch.cat([emb[:, 1], emb[:, 2]], -1)
        k = torch.cat([emb[:, 3:3 + L], emb[:, 3 + L:3 + 2 * L]], -1)             # [B, L, 2D] bf16 (padding rows are already zero)
        mask = (ids[3:3 + L] >= 0).t()
        with torch.autocast(emb.device.type, dtype=torch.bfloat16):
            return net.inner.head(u, q, k, mask, **kw_head)
    return FusedRecEngine(dense_net, fwd, col_table, list(table_rows), batch_size, embedding_dim=model.emb_dim, **kw)


def din_ids(batch: Dict[str, torch.Tensor]) -> torch.Tensor:
    """Taobao-shaped batch dict -> the [3 + 2 L, B] id-column block :func:`din_engine` expects (run it in the input pipeline)."""
    return torch.cat([batch["user"][None], batch["item"][None], batch["cat"][None], batch["hist_item"].t(), batch["hist_cat"].t()], 0).contiguous()


POOLED_SEQ_MODELS = ("dssm", "esmm", "mmoe", "dbmtl", "ple", "simple_multitask")


def pooled_seq_engine(model, batch_size: int, max_len: int = 50, combiner: str = "sum",
                      table_rows: Sequence[int] = (10_000_000, 100_000_000, 10_000), **kw) -> FusedRecEngine:
    """:class:`models.zoo.DSSM` and the multi-task models (ESMM, MMoE, DBMTL, PLE, SimpleMultiTask), which only consume the pooled behaviour
    history: the id columns of :func:`din_ids` ([user | item | cat | hist_item x L | hist_cat x L]) pooled into five bags
    [user | item | cat | hist_item | hist_cat] with ``combiner`` (``sum`` is what the framework path's ``_embed_pooled`` computes; the reference
    pools these columns with ``mean``), so the dense net sees a [B, 5, D] activation.  Multi-task models train on labels [B, 2] (click, conversion:
    :func:`taobao_engine_batch`) with the model's own ``multitask_loss``.  MMoE and PLE run their experts, gates and towers through
    :data:`nn.FUSED_MOE` (grouped expert GEMMs and the fused softmax-gate mixture)."""
    from ..nn import FUSED_MOE
    from .zoo import DSSM, MMoE, PLE, _MultiTask
    L = max_len
    col_table = [0, 1, 2] + [1] * L + [2] * L
    bags = [(1, combiner), (1, combiner), (1, combiner), (L, combiner), (L, combiner)]
    multitask = isinstance(model, _MultiTask)
    if not multitask and not isinstance(model, DSSM):
        raise ValueError(f"pooled_seq_engine: {type(model).__name__} is neither DSSM nor a multi-task model")
    dense_net = _StripTables(model)
    kw_tl = {"moe": FUSED_MOE} if isinstance(model, (MMoE, PLE)) else {}

    def fwd(net, dense, emb, ids):
        u = emb[:, 0]
        q = torch.cat([emb[:, 1], emb[:, 2]], -1)
        pooled = torch.cat([emb[:, 3], emb[:, 4]], -1)
        with torch.autocast(emb.device.type, dtype=torch.bfloat16):
            if multitask:
                return net.inner.tower_logits(torch.cat([u, q, pooled], -1), **kw_tl)
            return net.inner.head(u, q, pooled)
    if multitask:
        kw.setdefault("loss_fn", lambda out, y: dense_net.inner.multitask_loss({k: v.float() for k, v in out.items()}, y[:, 0], y[:, 1]))
    return FusedRecEngine(dense_net, fwd, col_table, list(table_rows), batch_size, embedding_dim=model.emb_dim, bags=bags,
                          label_dim=2 if multitask else 1, **kw)


def taobao_engine_batch(batch: Dict[str, torch.Tensor]):
    """Taobao-shaped batch dict -> ``(ids, labels [B, 2], None)`` for a multi-task :func:`pooled_seq_engine`: the click label and the conversion
    label built as :meth:`models.zoo._MultiTask.loss` builds it."""
    y = batch["labels"].float()
    return din_ids(batch), torch.stack([y, y * (batch["item"] % 2 == 0).to(y.dtype)], 1), None


class _StripTables(nn.Module):
    """Wraps a zoo model so that only its DENSE parameters are registered (the EmbeddingVariables are replaced by the engine's tables)."""

    def __init__(self, model: nn.Module):
        super().__init__()
        for name in ("emb", "wide", "user", "item", "cat"):       # WDL's wide tables: the engine's linear group
            if hasattr(model, name) and isinstance(getattr(model, name), nn.Module):
                try:
                    delattr(model, name)
                except AttributeError:
                    pass
        self.inner = model
