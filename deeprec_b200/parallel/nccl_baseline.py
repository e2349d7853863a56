"""In-repo NCCL re-creation of the reference's synchronous multi-GPU dataflow -- the measured BASELINE.

The reference's sync path (Horovod + SOK, SURVEY §3.4) cannot be built offline, so this module reproduces its
dataflow with ``torch.distributed`` NCCL collectives and unfused kernels, on the same model/config:

  NCCL all-to-all(ids) -> hash probe + gather (separate kernels) -> NCCL all-to-all(vectors) -> dense MLP ->
  NCCL all-reduce(dense grads) -> separate optimizer kernel -> NCCL all-to-all(sparse grads) ->
  dedup/segment-sum -> sparse Adagrad.

``NcclComm`` plugs into :class:`DLRMEngine` through the same three hooks as :class:`parallel.p2p.P2PComm`, so the
two arms differ ONLY in how the three communication-bound paths are executed.  ``BaselineDLRM`` additionally
swaps the dense net for cuBLAS (torch.nn + autocast bf16) to give the full "NCCL + cuBLAS" arm.
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

import torch
import torch.distributed as dist

from .. import _native
from .._native import OptHyper, check, ptr, stream_ptr


class NcclComm:
    unique_first = False         # reference (SOK) dataflow: table-wise placement, every id / vector / gradient row crosses the wire

    def _a2a(self, out, inp, recv_counts, send_counts):
        if self.world == 1:
            out.copy_(inp)
        else:
            dist.all_to_all_single(out, inp, recv_counts, send_counts, group=self.group)
        self.launches += 1

    def __init__(self, rank: int, world: int, dev: torch.device, group=None):
        self.rank, self.world, self.dev, self.group = rank, world, dev, group
        self.lib = _native.cuda()
        _native.set_device(dev.index)
        self.launches = 0            # kernels and collectives this communicator launches (the engine's embedding group counts its apply)

    def alloc_grads(self, P: int) -> torch.Tensor:
        return torch.zeros(P, dtype=torch.float32, device=self.dev)

    def alloc_exchange(self, T: int, B: int, D: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        z = lambda *s, dt: torch.zeros(*s, dtype=dt, device=self.dev)
        return z(T, B, dt=torch.int64), z(T, B, D, dt=torch.bfloat16), z(T, B, D, dt=torch.bfloat16)

    def _setup(self, eng) -> None:
        if hasattr(eng, "_nb"):
            return
        W, B, D = self.world, eng.B, eng.D
        owned = [[t for t in range(eng.T) if eng.owner_of[t] == r] for r in range(W)]
        nl = len(owned[self.rank])

        class NB:
            pass
        nb = NB()
        nb.owned = owned
        nb.idx = [torch.tensor(o, dtype=torch.int64, device=self.dev) for o in owned]
        nb.send_counts_ids = [len(o) * B for o in owned]                 # what I send to each owner
        nb.recv_counts_ids = [nl * B] * W                                # what I receive from each requester
        nb.keys_send = torch.empty(eng.T * B, dtype=torch.int64, device=self.dev)
        nb.keys_recv = torch.empty(max(1, W * nl * B), dtype=torch.int64, device=self.dev)     # [W][nl][B]
        nb.rows_send = torch.empty(max(1, W * nl * B), D, dtype=torch.bfloat16, device=self.dev)
        nb.rows_recv = torch.empty(eng.T * B, D, dtype=torch.bfloat16, device=self.dev)
        nb.grad_send = torch.empty(eng.T * B, D, dtype=torch.bfloat16, device=self.dev)
        nb.grad_recv = torch.empty(max(1, W * nl * B), D, dtype=torch.bfloat16, device=self.dev)
        nb.perm = torch.cat(nb.idx) if eng.T else torch.empty(0, dtype=torch.int64, device=self.dev)   # table order grouped by owner
        # offsets for table-index search inside the kernels: segment = (src rank, local table) of size B
        g = eng.group
        nb.tmap = g.tmap.repeat(W).contiguous() if nl else g.tmap                                     # [W * nl]
        nb.step_ptr = C.c_void_p(g.hp_dev.data_ptr() + OptHyper.global_step.offset)
        eng._nb = nb

    def lookup_forward(self, eng, train: bool) -> None:
        self._setup(eng)
        nb, W, B, D, lib = eng._nb, self.world, eng.B, eng.D, self.lib
        nl = len(nb.owned[self.rank])
        s = stream_ptr(self.dev)
        # 1. pack ids by owner, NCCL all-to-all (C2)
        nb.keys_send.copy_(eng.ids.index_select(0, nb.perm).view(-1))
        self.launches += 1
        self._a2a(nb.keys_recv[: W * nl * B], nb.keys_send, nb.recv_counts_ids, nb.send_counts_ids)
        # 2. probe + gather as separate kernels (K1/K3)
        n = W * nl * B
        if n:
            ctx = eng.group.ctx
            st = ctx.structs()
            check(lib.dr_cuda_table_lookup(ptr(st), ptr(nb.tmap), W * nl, ptr(nb.keys_recv), None, B, n, int(train), nb.step_ptr, ptr(eng.pos),
                                           ptr(ctx.ulist) if train else None, ptr(ctx.nuniq) if train else None,
                                           ctx.ulist.numel() if train else 0, s), "lookup")
            check(lib.dr_cuda_table_gather(ptr(st), ptr(nb.tmap), W * nl, D, ptr(nb.keys_recv), ptr(eng.pos), None, B, n, ptr(nb.rows_send), 1, 0, 0, 1, s), "gather")
            self.launches += 2
        # 3. NCCL all-to-all of the vectors (C3) + un-permute into feature-major order (S2 reorderKernel)
        self._a2a(nb.rows_recv, nb.rows_send[: W * nl * B], [c for c in nb.send_counts_ids], [c for c in nb.recv_counts_ids])
        eng.emb.index_copy_(0, nb.perm, nb.rows_recv.view(eng.T, B, D))
        self.launches += 1

    def sparse_backward(self, eng) -> None:
        nb, W, B, D, lib = eng._nb, self.world, eng.B, eng.D, self.lib
        nl = len(nb.owned[self.rank])
        s = stream_ptr(self.dev)
        nb.grad_send.copy_(eng.demb.index_select(0, nb.perm).view(-1, D))
        self.launches += 1
        self._a2a(nb.grad_recv[: W * nl * B], nb.grad_send, nb.recv_counts_ids, nb.send_counts_ids)     # C4
        n = W * nl * B
        if n:
            ctx = eng.group.ctx
            check(lib.dr_cuda_sparse_accumulate(ptr(ctx.structs()), ptr(nb.tmap), W * nl, D, ptr(eng.pos), None, B, n, ptr(nb.grad_recv), 1, 0, 0, 1,
                                                None, None, ptr(ctx.gsum), s), "accumulate")
            self.launches += 1
        eng.group.apply()

    def dense_allreduce_update(self, eng) -> None:
        if self.world > 1:
            dist.all_reduce(eng.grads, group=self.group)                                                                              # C1
            self.launches += 1
        s = stream_ptr(self.dev)
        check(self.lib.dr_cuda_dense_apply(ptr(eng.params), ptr(eng.grads), ptr(eng.s0) if eng.s0 is not None else None,
                                           ptr(eng.s1) if eng.s1 is not None else None, eng.P, ptr(eng.hp_dev), 1.0, None, s), "dense_apply")
        self.launches += 1


class BaselineDLRM:
    """"NCCL + cuBLAS" arm: reference dataflow with library GEMMs (torch.nn, autocast bf16) for the dense net,
    torch autograd for the interaction, NCCL for all three collectives, unfused table kernels."""

    def __init__(self, cfg, dev, rank, world, comm):
        from ..models.dlrm import DLRM
        from ..models.dlrm_engine import DLRMEngine
        self.cfg, self.dev, self.rank, self.world = cfg, dev, rank, world
        # reuse the engine for table construction / exchange buffers; its dense kernels are NOT used
        comm = comm if comm is not None else NcclComm(rank, world, dev)
        self.eng = DLRMEngine(cfg, dev, rank, world, comm)
        self.comm = comm
        self.net = DLRM(cfg.num_dense, [1] * len(cfg.cardinalities), cfg.embedding_dim, cfg.mlp_bot, cfg.mlp_top, use_ev=False, device=dev,
                        bn_eps=cfg.bn_eps, bn_momentum=cfg.bn_momentum)
        self.net.tables = torch.nn.ModuleList()          # embeddings come from the model-parallel tables
        self.opt = torch.optim.Adagrad(self.net.parameters(), lr=cfg.learning_rate, initial_accumulator_value=cfg.initial_accumulator_value, eps=0.0)
        self.loss = torch.zeros(1, device=dev)
        self.launches = 0
        self.B, self.T, self.D = cfg.batch_size, len(cfg.cardinalities), cfg.embedding_dim

    def load_batch(self, dense, ids, labels, non_blocking=True):
        self.eng.load_batch(dense, ids, labels, non_blocking)

    def train_step(self):
        from ..models.dlrm import dot_interaction
        eng, net = self.eng, self.net
        self.comm.lookup_forward(eng, True)
        emb = eng.emb.permute(1, 0, 2).float().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            x = net.bot(eng.dense_in)
            z = dot_interaction(x.float(), emb)
            logit = net.logits(net.top(z)).squeeze(-1)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logit.float(), eng.labels) / self.world
        self.opt.zero_grad(set_to_none=True)
        loss.backward()
        eng.demb.copy_(emb.grad.permute(1, 0, 2))
        self.comm.sparse_backward(eng)
        if self.world > 1:
            flat = torch.cat([p.grad.view(-1) for p in net.parameters()])
            dist.all_reduce(flat)
            o = 0
            for p in net.parameters():
                p.grad.copy_(flat[o:o + p.numel()].view_as(p)); o += p.numel()
        self.opt.step()
        check(eng.lib.dr_cuda_advance_hyper(ptr(eng.hp_dev), stream_ptr(self.dev)), "advance")
        self.loss.copy_(loss.detach() * self.world)
        self.launches += 120      # ~60 ATen/cuBLAS kernels fwd+bwd+optimizer; only our table kernels are "ours"

    def loss_value(self):
        return float(self.loss.item())
