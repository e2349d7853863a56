"""Asynchronous parameter-server training (the reference's primary distributed mode: SURVEY §2.5 / §2.16 "DP, async (parameter
server)", tensorflow/core/distributed_runtime/ + contrib/star_server pull/push semantics).

Roles (one process each, ``torch.distributed.rpc`` / TensorPipe as the transport — no graph partitioning, no Send/Recv ops):

  * ``ps{i}``      owns shard *i* of every EmbeddingVariable (``key % 1000 % num_ps``, the fixed_size_partitioner rule also used by the
                   checkpoint re-sharding) and a slice of the dense parameters, together with the optimizer state.  Updates are
                   applied the moment a worker pushes them: no barrier, no aggregation across workers (async SGD).
  * ``worker{j}``  runs the model; embedding lookups are *pulls*, sparse and dense gradients are *pushes*.

Transport optimisations kept from the reference:
  * FuseRecv (``tensor_fuse``, base_rendezvous_mgr.h:178-185): all tables' lookups of a step travel in ONE RPC per PS
    (``pull_many``), likewise all sparse gradients (``push_many``);
  * SliceSend/SliceRecv (kernels/slice_sendrecv_ops.cc): dense tensors larger than ``slice_bytes`` are transferred in slices so a
    huge parameter never needs one giant message (``pull_dense`` / ``push_dense``).

Elastic scaling (contrib/elastic_grpc_server: ``ElasticTrainingService{IsReadyScaling, ReadyToUpdate, UpdateServerDef,
FetchParamsMeta}``, elastic_training.proto:71-76): the job starts ``num_ps`` PS processes of which the first ``active_ps`` own
shards.  ``PSClient.scale(n)`` quiesces the servers, moves every row whose owner changes under ``key % 1000 % n`` directly
PS -> PS (rows + optimizer slots + freq / version: ``ExportAndRemove`` / ``RestoreFromKeysAndValues``), then publishes the new
server definition; other workers notice the bumped definition version on their next pull / push (the PS rejects requests made
under a stale definition) and re-route transparently.

The synchronous NVLink path (parallel/p2p.py) is the fast path on an H100 box; this module is the functional equivalent of the
PS mode for CPU clusters / heterogeneous setups and for the reference's async-training semantics (stale reads, lock-free rows).
"""
from __future__ import annotations

import os
import threading
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed.rpc as rpc
from torch import nn

from ..config import EmbeddingVariableOption
from ..embedding_variable import EmbeddingVariable, get_embedding_variable

_SERVER: Optional["ParameterServer"] = None
STALE_DEF = "StaleServerDef"


class _StaleServerDef(Exception):
    pass


# ---- native data plane (csrc/host/ps_server.cc): pulls / pushes over TCP served by C++ threads on the HostEV engine -----------------------
_NATIVE_BOUND = False


def _nlib():
    global _NATIVE_BOUND
    import ctypes as C
    from .. import _native
    lib = _native.host()
    if not _NATIVE_BOUND:
        P, INT, i64p = C.c_void_p, C.c_int, C.POINTER(C.c_int64)
        lib.dr_ps_server_start.restype, lib.dr_ps_server_start.argtypes = P, [C.c_char_p, INT, C.POINTER(INT)]
        lib.dr_ps_server_add_table.restype, lib.dr_ps_server_add_table.argtypes = INT, [P, P, INT, P]
        lib.dr_ps_server_set_def.restype, lib.dr_ps_server_set_def.argtypes = None, [P, INT, INT]
        lib.dr_ps_server_inflight.restype, lib.dr_ps_server_inflight.argtypes = INT, [P]
        lib.dr_ps_server_stats.restype, lib.dr_ps_server_stats.argtypes = None, [P, C.POINTER(C.c_uint64)]
        lib.dr_ps_server_stop.restype, lib.dr_ps_server_stop.argtypes = None, [P]
        lib.dr_ps_client_connect.restype, lib.dr_ps_client_connect.argtypes = P, [C.c_char_p, INT]
        lib.dr_ps_client_close.restype, lib.dr_ps_client_close.argtypes = None, [P]
        lib.dr_ps_client_send.restype = INT
        lib.dr_ps_client_send.argtypes = [P, INT, INT, INT, C.POINTER(INT), i64p, C.POINTER(P), C.POINTER(P), C.POINTER(INT)]
        lib.dr_ps_partition.restype, lib.dr_ps_partition.argtypes = None, [P, C.c_int64, INT, P, P]
        lib.dr_ps_client_recv.restype = INT
        lib.dr_ps_client_recv.argtypes = [P, INT, i64p, C.POINTER(INT), C.POINTER(P), C.POINTER(C.c_uint64)]
        _NATIVE_BOUND = True
    return lib


def ps_partition(flat: torch.Tensor, num_ps: int):
    """(order, counts): positions of ``flat`` grouped by owning server (stable), keys per server -- one native pass instead of ``num_ps``
    boolean masks (``ps_owner`` stays the definition: ``key % 1000 % num_ps``)."""
    from .._native import ptr
    k = flat.to(torch.int64).contiguous()
    order = torch.empty(k.numel(), dtype=torch.int64)
    counts = torch.zeros(num_ps, dtype=torch.int64)
    if k.numel():
        _nlib().dr_ps_partition(ptr(k), k.numel(), int(num_ps), ptr(order), ptr(counts))
    return order, counts.tolist()


def ps_owner(keys: torch.Tensor, num_ps: int) -> torch.Tensor:
    return torch.remainder(torch.remainder(keys.to(torch.int64), 1000), num_ps)


class ParameterServer:
    """State of one PS process.  All methods are invoked through RPC (module-level trampolines below)."""

    def __init__(self, index: int, num_ps: int, active_ps: Optional[int] = None):
        self.index, self.num_ps = index, num_ps
        self.active = num_ps if active_ps is None else active_ps      # the first ``active`` PS own shards
        self.def_version = 0                                          # bumped by UpdateServerDef
        self.frozen = False                                           # rows are moving: every pull / push is turned away
        self.ev_specs: Dict[str, tuple] = {}
        self.evs: Dict[str, EmbeddingVariable] = {}
        self.opts: Dict[str, object] = {}
        self.dense: Dict[str, torch.Tensor] = {}
        self.dense_state: Dict[str, torch.Tensor] = {}
        self.dense_lr = 0.01
        self.lock = threading.Lock()            # guards creation / the dense block; rows rely on the engine's own lock-free paths
        self._gate = threading.Condition()      # admission gate of pulls / pushes (elastic scaling fence)
        self._inflight = 0
        self.pushes = 0
        # native data plane: a TCP listener served by C++ threads; tables register as they are created (plain host tables only)
        self.native, self.native_port, self.native_ids = None, 0, {}
        if os.environ.get("DEEPREC_PS_NATIVE", "1") != "0":
            import ctypes as C
            port = C.c_int(0)
            h = _nlib().dr_ps_server_start(os.environ.get("DEEPREC_PS_BIND", "").encode(), 0, C.byref(port))
            if h:
                self.native, self.native_port = h, int(port.value)

    def _native_def(self) -> None:
        if self.native:
            _nlib().dr_ps_server_set_def(self.native, int(self.def_version), int(self.frozen))

    def _native_quiesce(self, timeout: float = 60.0) -> bool:
        """Native requests admitted before the freeze have finished (the C++ side counts them)."""
        import time
        if not self.native:
            return True
        t0 = time.time()
        while _nlib().dr_ps_server_inflight(self.native) > 0:
            if time.time() - t0 > timeout:
                return False
            time.sleep(0.001)
        return True

    def native_endpoint(self):
        """(host, port, {variable: (table id, dim)}) of the native data plane; port 0 when it is off."""
        return _advertise_host(), self.native_port, dict(self.native_ids)

    # ---- variables ----------------------------------------------------------------------------------------------------
    def create_ev(self, name: str, dim: int, optimizer: str, opt_kw: dict, option: Optional[EmbeddingVariableOption], seed: int) -> bool:
        from ..optim.optimizers import GlobalStep, make_optimizer
        with self.lock:
            if name not in self.evs:
                ev = get_embedding_variable(f"{name}/part_{self.index}", dim, ev_option=option, seed=seed)
                self.evs[name] = ev
                self.opts[name] = make_optimizer(optimizer, [], [ev], global_step=GlobalStep(), **opt_kw)
                self.ev_specs[name] = (dim, optimizer, dict(opt_kw), option, seed)
                tbl = ev.table
                if self.native and hasattr(tbl, "h") and type(tbl).__name__ == "HostTable":     # multi-tier tables stay on the RPC path
                    import ctypes as C
                    opt = self.opts[name]
                    hp = opt._hyper(opt.param_groups[0])
                    self.native_ids[name] = (int(_nlib().dr_ps_server_add_table(self.native, C.c_void_p(tbl.h), dim, C.byref(hp))), dim)
        return True

    def create_dense(self, name: str, value: torch.Tensor, lr: float) -> bool:
        with self.lock:
            if name not in self.dense:
                self.dense[name] = value.clone()
                self.dense_state[name] = torch.full_like(value, 0.1)      # Adagrad accumulator
            self.dense_lr = lr
        return True

    # ---- pull / push ------------------------------------------------------------------------------------------------------
    def _stale(self, def_version: Optional[int]) -> bool:
        """Requests made while rows are moving, or under an outdated server definition, are turned away (the reply is the
        ``STALE_DEF`` marker, not an exception: it is an expected event during scaling)."""
        return self.frozen or (def_version is not None and def_version != self.def_version)

    def _admit(self, def_version: Optional[int]) -> bool:
        """Admission of one pull / push: the staleness check and the in-flight count change under ONE lock, so a request is either
        turned away or counted before ``is_ready_scaling`` can observe a drained server."""
        with self._gate:
            if self._stale(def_version):
                return False
            self._inflight += 1
            return True

    def _done(self) -> None:
        with self._gate:
            self._inflight -= 1
            if self._inflight == 0:
                self._gate.notify_all()

    def pull_many(self, reqs: Sequence[Tuple[str, torch.Tensor]], def_version: Optional[int] = None):
        if not self._admit(def_version):
            return STALE_DEF
        try:
            return [self.evs[n].table.lookup(ids) for n, ids in reqs]
        finally:
            self._done()

    def push_many(self, grads: Sequence[Tuple[str, torch.Tensor, torch.Tensor]], def_version: Optional[int] = None):
        if not self._admit(def_version):
            return STALE_DEF
        try:
            with self.lock:              # one applier at a time per PS keeps the optimizer's step counter / beta powers coherent; the
                for name, ids, g in grads:   # whole request is one critical section, so a freeze never lands between two of its tables
                    opt, ev = self.opts[name], self.evs[name]
                    ev._record_grad(ids, g)
                    opt.step()
                    self.pushes += 1
            return self.pushes
        finally:
            self._done()

    def pull_dense(self, name: str, lo: int, hi: int) -> torch.Tensor:
        return self.dense[name].view(-1)[lo:hi].clone()

    def push_dense(self, name: str, lo: int, grad: torch.Tensor) -> bool:
        with self.lock:
            w, a = self.dense[name].view(-1), self.dense_state[name].view(-1)
            hi = lo + grad.numel()
            a[lo:hi] += grad * grad
            w[lo:hi] -= self.dense_lr * grad / a[lo:hi].sqrt()
        return True

    def stats(self) -> Dict[str, int]:
        npush = 0
        if self.native:
            import ctypes as C
            out = (C.c_uint64 * 6)()
            _nlib().dr_ps_server_stats(self.native, out)
            npush = int(out[1])
        return {n: int(e.total_count()) for n, e in self.evs.items()} | {"pushes": self.pushes + npush}

    # ---- FileSliceSend / FileSliceRecv (kernels/file_slice_sendrecv_ops.cc): files travel in slices, never as one message ----------
    def file_write_slice(self, path: str, offset: int, data: bytes, truncate: bool) -> int:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "wb" if truncate else "r+b") as f:
            f.seek(offset)
            f.write(data)
        return len(data)

    def file_read_slice(self, path: str, offset: int, nbytes: int) -> bytes:
        with open(path, "rb") as f:
            f.seek(offset)
            return f.read(nbytes)

    def file_size(self, path: str) -> int:
        return os.path.getsize(path) if os.path.exists(path) else -1

    # ---- elastic scaling (ElasticTrainingService) ----------------------------------------------------------------------------------
    def server_def(self) -> Tuple[int, int]:
        return self.active, self.def_version

    def is_ready_scaling(self, timeout: float = 60.0) -> bool:
        """IsReadyScaling: stop admitting pulls / pushes, then WAIT until every request admitted before the freeze has finished
        (in-flight count drained) -- only then may rows move.  A push that was admitted earlier completes against the old
        placement; one that arrives later gets STALE_DEF and is re-routed by the client under the new server definition."""
        with self._gate:
            self.frozen = True
            self._native_def()
            ok = self._gate.wait_for(lambda: self._inflight == 0, timeout=timeout)
        return bool(ok) and self._native_quiesce(timeout)

    def fetch_params_meta(self) -> Dict[str, Tuple[int, int]]:
        """FetchParamsMeta: {variable: (dim, rows held by this PS)}."""
        return {n: (e.embedding_dim, int(e.total_count())) for n, e in self.evs.items()}

    def scale_export(self, new_active: int) -> int:
        """ReadyToUpdate on an old owner: ship every row whose owner changes straight to its new PS; returns #rows moved."""
        from .elastic import export_and_remove
        moved = 0
        with self.lock:
            keep = self.index if self.index < new_active else -1
            for name, ev in self.evs.items():
                parts = export_and_remove(ev, keep, new_active, ps_owner)
                for dst, part in enumerate(parts):
                    if dst != keep and part["keys"].numel():
                        moved += rpc.rpc_sync(f"ps{dst}", _rpc_scale_import, args=(name, self.ev_specs[name], part))
        return moved

    def scale_import(self, name: str, spec: tuple, part: Dict[str, torch.Tensor]) -> int:
        from .elastic import restore_from_keys_and_values
        if name not in self.evs:                  # a PS that joins the active set learns the variable from the sender
            self.create_ev(name, *spec)
        return restore_from_keys_and_values(self.evs[name], part)      # full-stride rows: embedding + optimizer slots

    def update_server_def(self, new_active: int, def_version: int) -> bool:
        """UpdateServerDef: from now on requests must be made under ``def_version``."""
        with self.lock:
            self.active, self.def_version, self.frozen = new_active, def_version, False
            self._native_def()
        return True

    def frequency(self, name: str, ids: torch.Tensor) -> torch.Tensor:
        return self.evs[name].get_frequency(ids)

    def save(self, prefix: str, step: int) -> str:
        from ..checkpoint.saver import Saver
        with self.lock:                  # pushes are applied under the same lock: the checkpoint is a consistent cut between two of them
            was = self.frozen
            if self.native and not was:      # native pushes do not take self.lock: fence them for the duration of the snapshot (clients retry)
                self.frozen = True; self._native_def(); self._native_quiesce()
            try:
                return Saver(embedding_variables=list(self.evs.values())).save(f"{prefix}.ps{self.index}", step)
            finally:
                if self.native and not was:
                    self.frozen = False; self._native_def()


def _srv() -> ParameterServer:
    if _SERVER is None:
        raise RuntimeError("this process is not a parameter server (call run_ps first)")
    return _SERVER


# RPC trampolines (TensorPipe pickles functions by reference: they must be importable top-level names)
def _rpc_create_ev(*a): return _srv().create_ev(*a)
def _rpc_create_dense(*a): return _srv().create_dense(*a)
def _rpc_pull_many(*a): return _srv().pull_many(*a)
def _rpc_push_many(*a): return _srv().push_many(*a)
def _rpc_file_write_slice(*a): return _srv().file_write_slice(*a)
def _rpc_file_read_slice(*a): return _srv().file_read_slice(*a)
def _rpc_file_size(*a): return _srv().file_size(*a)
def _rpc_server_def(): return _srv().server_def()
def _rpc_is_ready_scaling(): return _srv().is_ready_scaling()
def _rpc_fetch_params_meta(): return _srv().fetch_params_meta()
def _rpc_scale_export(*a): return _srv().scale_export(*a)
def _rpc_scale_import(*a): return _srv().scale_import(*a)
def _rpc_update_server_def(*a): return _srv().update_server_def(*a)
def _rpc_pull_dense(*a): return _srv().pull_dense(*a)
def _rpc_push_dense(*a): return _srv().push_dense(*a)
def _rpc_stats(): return _srv().stats()
def _rpc_frequency(*a): return _srv().frequency(*a)
def _rpc_save(*a): return _srv().save(*a)
def _rpc_native_endpoint(): return _srv().native_endpoint()


def init_rpc(name: str, rank: int, world_size: int, master_port: int, master_addr: str = "127.0.0.1", threads: int = 8) -> None:
    os.environ.setdefault("MASTER_ADDR", master_addr)
    os.environ.setdefault("MASTER_PORT", str(master_port))
    opts = rpc.TensorPipeRpcBackendOptions(num_worker_threads=threads, init_method=f"tcp://{master_addr}:{master_port}")
    rpc.init_rpc(name, rank=rank, world_size=world_size, rpc_backend_options=opts)


def run_ps(index: int, num_ps: int, num_workers: int, master_port: int, stats_path: Optional[str] = None,
           active_ps: Optional[int] = None) -> None:
    """Body of a PS process: serve until every worker has shut down (optionally dump final statistics as JSON).
    ``active_ps`` < ``num_ps`` starts with spare servers that ``PSClient.scale`` can bring in later."""
    global _SERVER
    _SERVER = ParameterServer(index, num_ps, active_ps)
    init_rpc(f"ps{index}", index, num_ps + num_workers, master_port)
    rpc.shutdown()          # blocks until all workers called shutdown
    if stats_path:
        import json
        with open(stats_path, "w") as f:
            json.dump(_SERVER.stats(), f)


class _NativePush:
    """Future of one asynchronous native push (set by the connection's sender thread)."""

    def __init__(self):
        self.result, self._ev = None, threading.Event()

    def _set(self, r) -> None:
        self.result = r
        self._ev.set()

    def wait(self):
        self._ev.wait()
        if isinstance(self.result, Exception):
            raise self.result
        return self.result


class _NativeConn:
    """A worker's link to the native data plane of one PS (csrc/host/ps_server.cc): TWO TCP connections -- pulls are synchronous on the first;
    pushes go through a sender thread on the second (send + acknowledgement per push, in order), so a push being applied on the server never
    delays the next pull, and the training loop never blocks on a multi-megabyte send.  ctypes releases the GIL around the socket calls."""

    def __init__(self, host: str, port: int, ids: Dict[str, Tuple[int, int]]):
        import queue
        self.lib = _nlib()
        self.h = self.lib.dr_ps_client_connect(host.encode(), int(port))
        self.hp = self.lib.dr_ps_client_connect(host.encode(), int(port)) if self.h else None
        if not self.h or not self.hp:
            self.close()
            raise ConnectionError(f"native PS data plane {host}:{port} unreachable")
        self.ids = ids                                          # variable -> (table id, dim)
        self.q: "queue.Queue" = queue.Queue()
        self.sender = threading.Thread(target=self._send_loop, daemon=True)
        self.sender.start()

    def close(self) -> None:
        if getattr(self, "sender", None) is not None and self.sender.is_alive():
            self.q.put(None)
            self.sender.join(timeout=30)
        for a in ("h", "hp"):
            if getattr(self, a, None):
                self.lib.dr_ps_client_close(getattr(self, a)); setattr(self, a, None)

    def _arrays(self, items, with_grads: bool):
        import ctypes as C
        nt = len(items)
        tids, ns, dims = (C.c_int * nt)(), (C.c_int64 * nt)(), (C.c_int * nt)()
        kp, gp, keep = (C.c_void_p * nt)(), (C.c_void_p * nt)(), []
        for i, it in enumerate(items):
            tid, dim = self.ids[it[0]]
            k = it[1].to(torch.int64).contiguous()
            keep.append(k)
            tids[i], ns[i], dims[i], kp[i] = tid, k.numel(), dim, k.data_ptr() if k.numel() else None
            if with_grads:
                g = it[2].to(torch.float32).contiguous()
                keep.append(g)
                gp[i] = g.data_ptr() if g.numel() else None
        return nt, tids, ns, dims, kp, gp, keep

    def _send_loop(self) -> None:
        import ctypes as C
        while True:
            job = self.q.get()
            if job is None:
                return
            fut, (nt, tids, ns, dims, kp, gp, _keep), dv = job
            try:
                if self.lib.dr_ps_client_send(self.hp, 2, int(dv), nt, tids, ns, kp, gp, dims) != 0:
                    raise ConnectionError("native PS connection lost")
                aux = C.c_uint64(0)
                rc = self.lib.dr_ps_client_recv(self.hp, 0, None, None, None, C.byref(aux))
                if rc < 0:
                    raise ConnectionError("native PS connection lost")
                if rc == 2:
                    raise RuntimeError("native PS rejected a malformed push")
                fut._set(STALE_DEF if rc == 1 else int(aux.value))
            except Exception as e:  # noqa: BLE001 -- delivered to the waiter
                fut._set(e)

    def drain_until(self, fut=None) -> None:
        """Block until every push handed to the sender thread so far has been acknowledged."""
        done = _NativePush()
        self.q.put((done, self._arrays([], True), -1))          # an empty push is answered in order after everything before it
        done.wait()

    def push(self, items, def_version: int) -> _NativePush:
        f = _NativePush()
        self.q.put((f, self._arrays(items, True), def_version))
        return f

    def pull_send(self, items, def_version: int):
        nt, tids, ns, dims, kp, _gp, _keep = self._arrays(items, False)
        if self.lib.dr_ps_client_send(self.h, 1, int(def_version), nt, tids, ns, kp, None, dims) != 0:
            raise ConnectionError("native PS connection lost")
        return nt, ns, dims

    def pull_recv(self, ticket):
        import ctypes as C
        nt, ns, dims = ticket
        rows = [torch.empty(int(ns[i]), int(dims[i]), dtype=torch.float32) for i in range(nt)]
        rp = (C.c_void_p * nt)(*[r.data_ptr() if r.numel() else None for r in rows])
        rc = self.lib.dr_ps_client_recv(self.h, nt, ns, dims, rp, None)
        if rc < 0:
            raise ConnectionError("native PS connection lost")
        if rc == 2:
            raise RuntimeError("native PS rejected a malformed pull")
        return STALE_DEF if rc == 1 else rows


def _advertise_host() -> str:
    """Address workers reach this PS at: DEEPREC_PS_ADVERTISE, loopback for single-host jobs, else the interface that routes to the master."""
    import socket
    h = os.environ.get("DEEPREC_PS_ADVERTISE")
    if h:
        return h
    master = os.environ.get("MASTER_ADDR", "127.0.0.1")
    if master in ("127.0.0.1", "localhost"):
        return "127.0.0.1"
    try:
        with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s_:
            s_.connect((master, 9))
            return s_.getsockname()[0]
    except OSError:
        return "127.0.0.1"


class PSClient:
    """Worker-side handle.  ``num_ps`` PS processes occupy RPC ranks [0, num_ps); this worker is rank num_ps + worker_index.
    ``transport``: "native" (default; DEEPREC_PS_TRANSPORT) sends sparse pulls / pushes over the C++ data plane of each PS and falls back to
    RPC per request for variables a PS did not register there (multi-tier tables); "rpc" keeps everything on torch.distributed.rpc."""

    def __init__(self, worker_index: int, num_ps: int, num_workers: int, master_port: int, slice_bytes: int = 4 << 20,
                 active_ps: Optional[int] = None, transport: Optional[str] = None):
        self.total_ps = num_ps                                  # processes in the job (dense parameters hash over all of them)
        self.num_ps = num_ps if active_ps is None else active_ps  # servers that currently own embedding shards
        self.def_version = 0
        self.worker_index, self.slice_elems = worker_index, max(1, slice_bytes // 4)
        init_rpc(f"worker{worker_index}", num_ps + worker_index, num_ps + num_workers, master_port)
        self._pending: List = []
        self.transport = (transport or os.environ.get("DEEPREC_PS_TRANSPORT", "native")).lower()
        self._conns: Dict[int, Optional[_NativeConn]] = {}

    def _conn(self, p: int, names) -> Optional[_NativeConn]:
        """Native connection to PS ``p`` if every variable in ``names`` is registered on its data plane, else None (-> RPC)."""
        if self.transport != "native":
            return None
        c = self._conns.get(p, False)
        if c is False or (c is not None and any(n not in c.ids for n in names)):
            host, port, ids = rpc.rpc_sync(f"ps{p}", _rpc_native_endpoint)
            if c not in (False, None):
                c.ids = ids                                     # variables created after the connection was opened
            else:
                try:
                    c = _NativeConn(host, port, ids) if port else None
                except ConnectionError:
                    c = None
                self._conns[p] = c
        return c if c is not None and all(n in c.ids for n in names) else None

    # ---- elastic scaling ---------------------------------------------------------------------------------------------------------
    def refresh_server_def(self) -> None:
        self.num_ps, self.def_version = rpc.rpc_sync("ps0", _rpc_server_def)

    def fetch_params_meta(self) -> List[Dict[str, Tuple[int, int]]]:
        return [rpc.rpc_sync(f"ps{p}", _rpc_fetch_params_meta) for p in range(self.total_ps)]

    def scale(self, new_active_ps: int) -> int:
        """Change the number of PS that own embedding shards (1 <= n <= total).  Returns the number of rows that moved."""
        if not 1 <= new_active_ps <= self.total_ps:
            raise ValueError(f"new_active_ps must be in [1, {self.total_ps}]")
        self.wait()
        self.refresh_server_def()
        old = self.num_ps
        if new_active_ps == old:
            return 0
        for p in range(self.total_ps):                                               # IsReadyScaling: fence every server
            assert rpc.rpc_sync(f"ps{p}", _rpc_is_ready_scaling)
        moved = sum(rpc.rpc_sync(f"ps{p}", _rpc_scale_export, args=(new_active_ps,)) for p in range(old))   # ReadyToUpdate
        for p in range(self.total_ps):                                               # UpdateServerDef (lifts the fence)
            rpc.rpc_sync(f"ps{p}", _rpc_update_server_def, args=(new_active_ps, self.def_version + 1))
        self.num_ps, self.def_version = new_active_ps, self.def_version + 1
        return moved

    def _with_current_def(self, fn):
        """Run ``fn`` (which issues RPCs under self.def_version); on a stale-definition rejection re-read the definition and retry."""
        import time
        for _ in range(1200):
            try:
                return fn()
            except _StaleServerDef:
                time.sleep(0.05)
                self.refresh_server_def()
        raise RuntimeError("server definition did not settle")

    def shutdown(self) -> None:
        self.wait()
        for c in self._conns.values():
            if c:
                c.drain_until(None); c.close()
        self._conns.clear()
        rpc.shutdown()

    def wait(self) -> None:
        pending, self._pending = self._pending, []
        for item in [i for i in pending if not isinstance(i, tuple)]:               # dense slices
            item.wait()
        self._settle_pushes([i for i in pending if isinstance(i, tuple)])

    # ---- variables ------------------------------------------------------------------------------------------------------------
    def create_embedding(self, name: str, dim: int, optimizer: str = "adagrad", option: Optional[EmbeddingVariableOption] = None,
                         seed: int = 0, **opt_kw) -> "PSEmbedding":
        for p in range(self.total_ps):
            rpc.rpc_sync(f"ps{p}", _rpc_create_ev, args=(name, dim, optimizer, opt_kw, option, seed))
        return PSEmbedding(self, name, dim)

    def register_dense(self, module: nn.Module, lr: float = 0.01) -> None:
        """Dense parameters live on PS (hash(name) % num_ps); every worker starts from the PS copy."""
        self._dense = [(n, p) for n, p in module.named_parameters() if p.numel() > 0]
        for n, p in self._dense:
            rpc.rpc_sync(self._dense_owner(n), _rpc_create_dense, args=(n, p.detach().clone(), lr))
        self.pull_dense()

    def _dense_owner(self, name: str) -> str:
        import zlib
        return f"ps{zlib.crc32(name.encode()) % self.total_ps}"

    # ---- FuseRecv-style batched pull / push ----------------------------------------------------------------------------------------
    def pull_many(self, reqs: Sequence[Tuple[str, torch.Tensor]]) -> List[torch.Tensor]:
        """One RPC per PS for ALL tables of the step; rows are stitched back into request order."""
        return self._with_current_def(lambda: self._pull_many(reqs))

    def _pull_many(self, reqs):
        per_ps: List[List[Tuple[str, torch.Tensor]]] = [[] for _ in range(self.num_ps)]
        orders = []
        for name, ids in reqs:
            flat = ids.reshape(-1)
            order, counts = ps_partition(flat, self.num_ps)
            orders.append(order)
            for p, part in enumerate(torch.split(flat[order], counts)):
                per_ps[p].append((name, part))
        names = [n for n, _ in reqs]
        conns = [self._conn(p, names) for p in range(self.num_ps)]
        # every request is on the wire before the first answer is read: the servers work in parallel on either transport
        tickets = [conns[p].pull_send(per_ps[p], self.def_version) if conns[p] is not None
                   else rpc.rpc_async(f"ps{p}", _rpc_pull_many, args=(per_ps[p], self.def_version)) for p in range(self.num_ps)]
        res = [conns[p].pull_recv(tickets[p]) if conns[p] is not None else tickets[p].wait() for p in range(self.num_ps)]
        if any(isinstance(r, str) for r in res):
            raise _StaleServerDef()
        out = []
        for i, (name, ids) in enumerate(reqs):
            dim = res[0][i].shape[1]
            rows = torch.empty(ids.numel(), dim)
            rows[orders[i]] = torch.cat([res[p][i] for p in range(self.num_ps)])       # un-permute: one scatter per table
            out.append(rows.view(*ids.shape, dim))
        return out

    def push_many(self, grads: Sequence[Tuple[str, torch.Tensor, torch.Tensor]], asynchronous: bool = True) -> None:
        """Sparse gradients, one fused RPC per PS.  Asynchronous pushes that a PS rejects because the server definition changed
        in flight are re-sent under the new definition by ``wait()``."""
        sent = self._send_pushes(grads)
        if asynchronous:
            self._pending.extend(sent)
        else:
            self._settle_pushes(sent)

    def _send_pushes(self, grads) -> List[Tuple[object, list]]:
        """Partition by owner under the current definition and fire one RPC per PS; returns (future, payload) pairs."""
        per_ps: List[List] = [[] for _ in range(self.num_ps)]
        for name, ids, g in grads:
            flat, g2 = ids.reshape(-1), g.reshape(-1, g.shape[-1])
            order, counts = ps_partition(flat, self.num_ps)
            fs, gs = torch.split(flat[order], counts), torch.split(g2[order], counts)
            for p in range(self.num_ps):
                if counts[p]:
                    per_ps[p].append((name, fs[p], gs[p]))
        out = []
        for p in range(self.num_ps):
            if not per_ps[p]:
                continue
            c = self._conn(p, [n for n, _i, _g in per_ps[p]])
            fut = c.push(per_ps[p], self.def_version) if c is not None else rpc.rpc_async(f"ps{p}", _rpc_push_many, args=(per_ps[p], self.def_version))
            out.append((fut, per_ps[p]))
        return out

    def _settle_pushes(self, sent: List[Tuple[object, list]]) -> None:
        """Wait for pushes; ONLY the payloads a PS turned away are re-partitioned and re-sent (nothing is applied twice)."""
        import time
        for _ in range(1200):
            rejected = [g for f, payload in sent if isinstance(f.wait(), str) for g in payload]
            if not rejected:
                return
            time.sleep(0.05)
            self.refresh_server_def()
            sent = self._send_pushes(rejected)
        raise RuntimeError("server definition did not settle")

    # ---- SliceSend/Recv-style dense transfer --------------------------------------------------------------------------------------
    def pull_dense(self) -> None:
        for n, p in self._dense:
            flat, owner = p.data.view(-1), self._dense_owner(n)
            futs = [(lo, rpc.rpc_async(owner, _rpc_pull_dense, args=(n, lo, min(lo + self.slice_elems, flat.numel()))))
                    for lo in range(0, flat.numel(), self.slice_elems)]
            for lo, f in futs:
                v = f.wait()
                flat[lo: lo + v.numel()] = v

    def push_dense(self) -> None:
        for n, p in self._dense:
            if p.grad is None:
                continue
            g, owner = p.grad.detach().view(-1), self._dense_owner(n)
            for lo in range(0, g.numel(), self.slice_elems):
                self._pending.append(rpc.rpc_async(owner, _rpc_push_dense, args=(n, lo, g[lo: lo + self.slice_elems].clone())))

    # ---- FileSliceSend / FileSliceRecv: ship a file (checkpoint shard, SSD .emb file, warm-up data) to / from a server in slices --------
    def send_file(self, ps_index: int, local_path: str, remote_path: str, slice_bytes: int = 4 << 20) -> int:
        sent, futs = 0, []
        with open(local_path, "rb") as f:
            while True:
                chunk = f.read(slice_bytes)
                if not chunk and sent > 0:
                    break
                futs.append(rpc.rpc_async(f"ps{ps_index}", _rpc_file_write_slice, args=(remote_path, sent, chunk, sent == 0)))
                if sent == 0:
                    futs[-1].wait()           # the first slice creates / truncates the file before the others land
                sent += len(chunk)
                if not chunk:
                    break
        for f_ in futs:
            f_.wait()
        return sent

    def recv_file(self, ps_index: int, remote_path: str, local_path: str, slice_bytes: int = 4 << 20) -> int:
        size = rpc.rpc_sync(f"ps{ps_index}", _rpc_file_size, args=(remote_path,))
        if size < 0:
            raise FileNotFoundError(f"ps{ps_index}:{remote_path}")
        futs = [(o, rpc.rpc_async(f"ps{ps_index}", _rpc_file_read_slice, args=(remote_path, o, min(slice_bytes, size - o)))) for o in range(0, size, slice_bytes)]
        os.makedirs(os.path.dirname(os.path.abspath(local_path)), exist_ok=True)
        with open(local_path, "wb") as f:
            for o, fut in futs:
                f.seek(o)
                f.write(fut.wait())
        return size

    def stats(self) -> List[Dict[str, int]]:
        return [rpc.rpc_sync(f"ps{p}", _rpc_stats) for p in range(self.num_ps)]

    def frequency(self, name: str, ids: torch.Tensor) -> torch.Tensor:
        flat = ids.reshape(-1)
        own = ps_owner(flat, self.num_ps)
        out = torch.zeros(flat.numel(), dtype=torch.int64)
        for p in range(self.num_ps):
            m = own == p
            if m.any():
                out[m] = rpc.rpc_sync(f"ps{p}", _rpc_frequency, args=(name, flat[m]))
        return out

    def save(self, prefix: str, step: int) -> List[str]:
        return [rpc.rpc_sync(f"ps{p}", _rpc_save, args=(prefix, step)) for p in range(self.num_ps)]


class _PSLookup(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, emb: "PSEmbedding", ids: torch.Tensor, rows: torch.Tensor):
        ctx.emb, ctx.ids = emb, ids
        return rows

    @staticmethod
    def backward(ctx, g):
        ctx.emb._grads.append((ctx.ids, g.detach()))
        return None, None, None, None


class PSEmbedding(nn.Module):
    """An EmbeddingVariable whose rows live on the parameter servers."""

    def __init__(self, client: PSClient, name: str, dim: int):
        super().__init__()
        self.client, self.name, self.embedding_dim = client, name, dim
        self._anchor = nn.Parameter(torch.zeros(0))
        self._grads: List[Tuple[torch.Tensor, torch.Tensor]] = []

    def forward(self, ids: torch.Tensor) -> torch.Tensor:
        return group_pull(self.client, [self], [ids])[0]

    def pop_grads(self) -> List[Tuple[str, torch.Tensor, torch.Tensor]]:
        out = [(self.name, i, g) for i, g in self._grads]
        self._grads = []
        return out


def group_pull(client: PSClient, embs: Sequence[PSEmbedding], ids: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    """Fused pull of several tables (one RPC per PS) returning autograd-tracked rows."""
    rows = client.pull_many([(e.name, i) for e, i in zip(embs, ids)])
    if torch.is_grad_enabled():
        return [_PSLookup.apply(e._anchor, e, i, r) for e, i, r in zip(embs, ids, rows)]
    return rows


def push_gradients(client: PSClient, embs: Sequence[PSEmbedding], asynchronous: bool = True) -> None:
    """Push every recorded sparse gradient (one fused RPC per PS) and the dense gradients; asynchronous by default."""
    grads = [g for e in embs for g in e.pop_grads()]
    if grads:
        client.push_many(grads, asynchronous)
    if getattr(client, "_dense", None):
        client.push_dense()
