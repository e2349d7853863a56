"""NVLink peer-memory communicator: CUDA-IPC symmetric buffers + the fused P2P kernels.

torch.distributed (NCCL) is used ONLY as plumbing: to exchange the 64-byte IPC handles at start-up.  On the step's hot path
there is no NCCL call and no barrier kernel: the kernels in csrc/cuda/sparse_pipeline.cu / comm_kernels.cu load and store
peer memory themselves and synchronise with release/acquire flags raised by the LAST block of the producing kernel
(csrc/cuda/sp_sync.cuh).

Per training step (flag channels of :mod:`parallel.sparse_pipeline`):
  DEDUP  requester finished bucketing its unique keys   -> owners' k_sp_lookup waits PER SOURCE (starts on ready sources)
  ROWS   owner finished pushing rows into every urow     -> the requester's interaction kernel waits in-kernel
  GRAD   requester finished pre-reducing its gradients   -> owners' k_sp_grad waits per source, pulls unique fp32 rows
  DENSE  dense gradients complete (k_sp_signal)          -> k_allreduce_apply waits in-kernel, reduces + applies the optimizer
Buffer reuse across steps is ordered by the DENSE wait (a full rendezvous) -- see DESIGN.md §comm.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List

import torch
import torch.distributed as dist

from .. import _native
from .._cuda_sigs import Peers
from .._native import check, ptr, stream_ptr
from .sparse_pipeline import CH_DENSE

vp = C.c_void_p


class _RawCuda:
    def __init__(self, addr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (addr, False), "version": 3}


class SymmetricBuffer:
    """Same-size device allocation on every rank, mapped into every rank's address space."""

    def __init__(self, comm: "P2PComm", nbytes: int):
        lib = comm.lib
        nbytes = max(256, int(nbytes))
        self.comm, self.nbytes = comm, nbytes
        local = vp()
        check(lib.dr_comm_alloc(nbytes, C.byref(local)), "alloc")
        self.local = local.value
        handle = (C.c_char * 64)()
        check(lib.dr_comm_get_handle(vp(self.local), handle), "ipc_get_handle")
        handles: List[bytes] = [None] * comm.world
        dist.all_gather_object(handles, bytes(handle.raw), group=comm.group)
        self.peers = Peers()
        self._opened = []
        for r in range(comm.world):
            if r == comm.rank:
                self.peers.ptr[r] = self.local
            else:
                p = vp()
                buf = C.create_string_buffer(handles[r], 64)
                check(lib.dr_comm_open_handle(buf, C.byref(p)), f"ipc_open_handle(rank {r})")
                self.peers.ptr[r] = p.value
                self._opened.append(p.value)
        self._raw = torch.as_tensor(_RawCuda(self.local, nbytes), device=comm.dev)

    def tensor(self, dtype: torch.dtype, shape) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= s
        nb = n * torch.empty((), dtype=dtype).element_size()
        assert nb <= self.nbytes
        return self._raw[:nb].view(dtype).view(*shape)

    def peers_ref(self):
        return C.byref(self.peers)


class P2PComm:
    unique_first = True          # engines build a parallel.sparse_pipeline.SparsePipeline on top of this communicator
    NVLS_2PHASE_BYTES = int(os.environ.get("DEEPREC_NVLS_2PHASE_BYTES", 8 << 20))  # dense gradients at least this large take the two-phase NVLS all-reduce (one-shot below: fewer launches)

    def __init__(self, rank: int, world: int, dev: torch.device, group=None):
        self.rank, self.world, self.dev, self.group = rank, world, dev, group
        self.lib = _native.cuda()
        check(self.lib.dr_cuda_set_device(dev.index), "set_device")
        for r in range(world):
            if r != rank and not self.lib.dr_comm_can_access_peer(dev.index, r):
                raise RuntimeError(f"GPU {dev.index} cannot access peer {r}: NVLink P2P is required")
        self.signals = SymmetricBuffer(self, 16 * 16 * 4)
        self.epochs = torch.zeros(16, dtype=torch.int32, device=dev)
        self._buffers: List[SymmetricBuffer] = [self.signals]
        self.launches = 0            # kernels of the step's all-reduce / rendezvous calls (the pipeline counts its own DENSE signal)
        dist.barrier(group=group)

    def symmetric(self, nbytes: int) -> SymmetricBuffer:
        b = SymmetricBuffer(self, nbytes)
        self._buffers.append(b)
        return b

    def host_barrier(self) -> None:
        torch.cuda.synchronize(self.dev)
        dist.barrier(group=self.group)

    def alloc_grads(self, P: int) -> torch.Tensor:
        """Symmetric dense-gradient buffer.  With NVLS (multicast objects supported on every rank, DEEPREC_NVLS != 0) it is a VMM
        allocation bound to a multicast object: the backward writes the local unicast mapping, the fused all-reduce + optimizer reads the
        multicast mapping with multimem.ld_reduce (csrc/cuda/nvls.cu); otherwise a CUDA-IPC buffer read with the one-shot peer pull."""
        self.nvls = self._try_nvls(P * 4)
        if self.nvls is not None:
            return self.nvls["tensor"][:P]
        self.grads_buf = self.symmetric(P * 4)
        return self.grads_buf.tensor(torch.float32, (P,))

    def _all_ok(self, ok: bool) -> bool:
        t = torch.tensor([1 if ok else 0], dtype=torch.int32, device=self.dev)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.group)
        return bool(t.item())

    def _try_nvls(self, nbytes: int):
        import os
        import socket
        lib = self.lib
        if not self._all_ok(os.environ.get("DEEPREC_NVLS", "1") != "0" and lib.dr_nvls_supported(self.dev.index) == 1):
            return None
        size = int(lib.dr_nvls_size(max(nbytes, 1 << 16), self.world))
        if not self._all_ok(size > 0):
            return None
        state, fd = vp(), C.c_int(-1)
        P2PComm._nvls_seq = getattr(P2PComm, "_nvls_seq", 0) + 1
        addr = f"\0deeprec_nvls_{os.environ.get('MASTER_PORT', '0')}_{P2PComm._nvls_seq}"
        ok = True
        if self.rank == 0:
            ok = lib.dr_nvls_create(size, self.world, self.dev.index, C.byref(state), C.byref(fd)) == 0
            srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
            try:
                srv.bind(addr); srv.listen(self.world); srv.settimeout(60)
            except OSError:
                ok = False
            okall = self._all_ok(ok)
            if okall:
                try:
                    for _ in range(self.world - 1):                      # the multicast handle travels as a POSIX fd (SCM_RIGHTS)
                        c, _a = srv.accept()
                        socket.send_fds(c, [b"h"], [fd.value]); c.close()
                except OSError:
                    ok = False
            srv.close()
            if not okall:
                return None
        else:
            if not self._all_ok(True):
                return None
            try:
                c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM); c.settimeout(60)
                for _ in range(200):
                    try:
                        c.connect(addr); break
                    except OSError:
                        import time
                        time.sleep(0.05)
                _m, fds, _f, _a = socket.recv_fds(c, 16, 1); c.close()
                ok = len(fds) == 1 and lib.dr_nvls_import(fds[0], size, self.world, self.dev.index, C.byref(state)) == 0
            except OSError:
                ok = False
        if not self._all_ok(ok):
            return None
        if not self._all_ok(lib.dr_nvls_add_device(state) == 0):           # every device joins the team BEFORE any memory is bound
            return None
        local, mc = vp(), vp()
        if not self._all_ok(lib.dr_nvls_bind(state, C.byref(local), C.byref(mc)) == 0):
            return None
        raw = torch.as_tensor(_RawCuda(local.value, size), device=self.dev)
        return {"state": state, "mc": mc.value, "local": local.value, "size": size, "tensor": raw.view(torch.float32)}

    def barrier(self, channel: int) -> None:
        """Stand-alone device-side rank barrier (tests / utilities; the training step does not use it)."""
        check(self.lib.dr_comm_barrier(self.signals.peers_ref(), ptr(self.epochs), channel, self.rank, self.world, stream_ptr(self.dev)), "barrier")

    def dense_allreduce_update(self, eng) -> None:
        """DENSE flag + one-shot all-reduce fused with the optimizer (the kernel polls the flags itself)."""
        sp = eng.sp
        sp.signal(CH_DENSE)
        if getattr(self, "nvls", None) is not None and eng.P * 4 >= self.NVLS_2PHASE_BYTES:
            # large dense nets: reduce-scatter (multimem.ld_reduce) + in-switch broadcast (multimem.st), then the optimizer from local memory
            check(self.lib.dr_nvls_allreduce_2phase(vp(self.nvls["mc"]), vp(self.nvls["local"]), self.rank, self.world, ptr(eng.params),
                                                    ptr(eng.s0) if eng.s0 is not None else None, ptr(eng.s1) if eng.s1 is not None else None, eng.P,
                                                    ptr(eng.hp_dev), sp.sync_ref(), stream_ptr(self.dev)), "nvls_allreduce_2phase")
            self.launches += 2
            return
        if getattr(self, "nvls", None) is not None:     # in-switch reduction: one multimem.ld_reduce per 16 B instead of W peer loads
            check(self.lib.dr_nvls_allreduce_apply(vp(self.nvls["mc"]), ptr(eng.params), ptr(eng.s0) if eng.s0 is not None else None,
                                                   ptr(eng.s1) if eng.s1 is not None else None, eng.P, ptr(eng.hp_dev), None, sp.sync_ref(), stream_ptr(self.dev)),
                  "nvls_allreduce_apply")
            self.launches += 1
            return
        check(self.lib.dr_comm_allreduce_apply_sync(self.grads_buf.peers_ref(), self.world, ptr(eng.params), ptr(eng.s0) if eng.s0 is not None else None,
                                                    ptr(eng.s1) if eng.s1 is not None else None, eng.P, ptr(eng.hp_dev), None, sp.sync_ref(), stream_ptr(self.dev)),
              "allreduce_apply")
        self.launches += 1

    def wait_dense(self, sp) -> None:
        """In-kernel rendezvous on the DENSE flags without any reduction (forward-only passes)."""
        if getattr(self, "nvls", None) is not None:
            check(self.lib.dr_nvls_allreduce_apply(vp(self.nvls["mc"]), None, None, None, 0, None, None, sp.sync_ref(), stream_ptr(self.dev)), "wait_dense")
        else:
            check(self.lib.dr_comm_allreduce_apply_sync(self.grads_buf.peers_ref(), self.world, None, None, None, 0, None, None, sp.sync_ref(), stream_ptr(self.dev)),
                  "wait_dense")
        self.launches += 1

    def allreduce(self, out: torch.Tensor, two_phase: bool = False) -> None:
        """All-reduce of the symmetric grads buffer into ``out`` (tests / metrics).  ``two_phase`` (NVLS only) reduces IN PLACE: the
        gradient buffer itself holds the sum afterwards."""
        self.barrier(3)
        if getattr(self, "nvls", None) is not None and two_phase:
            check(self.lib.dr_nvls_allreduce_2phase(vp(self.nvls["mc"]), vp(self.nvls["local"]), self.rank, self.world, None, None, None, out.numel(), None,
                                                    None, stream_ptr(self.dev)), "nvls_allreduce_2phase")
            self.barrier(5)                         # every slice owner has broadcast its slice: my local buffer now holds the full sum
            out.copy_(self.nvls["tensor"][: out.numel()])
        elif getattr(self, "nvls", None) is not None:
            check(self.lib.dr_nvls_allreduce_apply(vp(self.nvls["mc"]), None, None, None, out.numel(), None, ptr(out), None, stream_ptr(self.dev)), "nvls_allreduce")
        else:
            check(self.lib.dr_comm_allreduce_apply(self.grads_buf.peers_ref(), self.world, None, None, None, out.numel(), None, ptr(out), stream_ptr(self.dev)), "allreduce")
        self.barrier(4)        # nobody overwrites its contribution before every rank has read it
