"""Communicator for the CUDA-on-CPU emulation (``_native.cuda_emulation()``): the ranks of a job are THREADS of one process, a symmetric buffer
is one host allocation per rank whose address every other rank simply knows -- the same ``symmetric()`` / ``host_barrier()`` surface as
:class:`parallel.p2p.P2PComm`, so :class:`parallel.sparse_pipeline.SparsePipeline` and the flag protocol of ``csrc/cuda/sp_sync.cuh`` run unchanged,
rank against rank, under ThreadSanitizer (tests/test_cuda_emu_sparse_pipeline.py).  CPU CI only."""
from __future__ import annotations

import ctypes as C
import threading
from typing import Dict, List

import torch

from .. import _native
from .._cuda_sigs import Peers
from .._native import check, ptr


class EmuWorld:
    """Shared by the rank threads: rendezvous barrier + the table of published buffer addresses."""

    def __init__(self, world: int):
        self.world = world
        self.barrier = threading.Barrier(world)
        self.lock = threading.Lock()
        self.published: Dict[int, List[int]] = {}


class _EmuSymmetricBuffer:
    def __init__(self, comm: "EmuComm", nbytes: int, index: int):
        nbytes = max(256, int(nbytes))
        self.nbytes = nbytes
        self._raw = torch.zeros(nbytes, dtype=torch.uint8)
        self.local = self._raw.data_ptr()
        w = comm.shared
        with w.lock:
            w.published.setdefault(index, [0] * w.world)[comm.rank] = self.local
        w.barrier.wait()
        self.peers = Peers()
        for r in range(w.world):
            self.peers.ptr[r] = w.published[index][r]
        w.barrier.wait()

    def tensor(self, dtype: torch.dtype, shape) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= s
        nb = n * torch.empty((), dtype=dtype).element_size()
        assert nb <= self.nbytes
        return self._raw[:nb].view(dtype).view(*shape)

    def peers_ref(self):
        return C.byref(self.peers)


class EmuComm:
    unique_first = True

    def __init__(self, shared: EmuWorld, rank: int):
        self.shared, self.rank, self.world = shared, rank, shared.world
        self.dev = torch.device("cpu")
        self._n = 0
        self._buffers = []
        self.launches = 0            # kernels of the step's all-reduce / rendezvous calls (the pipeline counts its own DENSE signal)

    def symmetric(self, nbytes: int) -> _EmuSymmetricBuffer:
        """Collective: every rank thread calls it in the same order."""
        b = _EmuSymmetricBuffer(self, nbytes, self._n)
        self._n += 1
        self._buffers.append(b)
        return b

    def host_barrier(self) -> None:
        self.shared.barrier.wait()

    # ---- what the engines ask of a communicator beyond symmetric buffers (parallel.p2p.P2PComm's surface) ---------------------------------------
    def alloc_grads(self, P: int) -> torch.Tensor:
        self.grads_buf = self.symmetric(P * 4)
        return self.grads_buf.tensor(torch.float32, (P,))

    def dense_allreduce_update(self, eng) -> None:
        """DENSE flag + the one-shot peer-pull all-reduce fused with the optimizer (comm_kernels.cu: k_allreduce_apply polls the flags itself)."""
        sp = eng.sp
        sp.signal(3)
        check(_native.cuda().dr_comm_allreduce_apply_sync(self.grads_buf.peers_ref(), self.world, ptr(eng.params), ptr(eng.s0) if eng.s0 is not None else None,
                                                          ptr(eng.s1) if eng.s1 is not None else None, eng.P, ptr(eng.hp_dev), None, sp.sync_ref(), None),
              "allreduce_apply")
        self.launches += 1

    def wait_dense(self, sp) -> None:
        check(_native.cuda().dr_comm_allreduce_apply_sync(self.grads_buf.peers_ref(), self.world, None, None, None, 0, None, None, sp.sync_ref(), None),
              "wait_dense")
        self.launches += 1

    def host_broadcast(self, tensors, src: int = 0) -> None:
        """Rank ``src``'s values into every rank's tensors (engine construction)."""
        w = self.shared
        if self.rank == src:
            with w.lock:
                w.published["bcast"] = [t.detach().clone() for t in tensors]
        w.barrier.wait()
        if self.rank != src:
            with torch.no_grad():
                for t, v in zip(tensors, w.published["bcast"]):
                    t.copy_(v)
        w.barrier.wait()

    def host_all_reduce(self, t: torch.Tensor) -> None:
        """Sum over the ranks, in place (metrics)."""
        w = self.shared
        with w.lock:
            w.published.setdefault("allred", {})[self.rank] = t.detach().clone()
        w.barrier.wait()
        total = sum(w.published["allred"][r] for r in range(self.world))
        w.barrier.wait()
        t.copy_(total)
        w.barrier.wait()
