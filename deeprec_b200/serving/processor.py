"""Python side of the native Processor (C ABI in csrc/cuda/serving_runtime.cu) + the client SDK wire format.

``Processor`` loads the in-tree library with ctypes and calls ``initialize / process / batch_process /
get_serving_model_info`` exactly as an RPC front-end would (serving/processor/serving/processor.h in the reference;
the Go/Java/Python SDK demos of serving/sdk map onto ``encode_request`` / ``decode_response``)."""
from __future__ import annotations

import ctypes as C
import json
import os
import struct
from typing import List, Sequence, Tuple

import numpy as np

from .. import build as _build

REQ_MAGIC, RESP_MAGIC = 0x51525244, 0x53525244


def encode_request(dense: np.ndarray, ids: np.ndarray) -> bytes:
    """dense [B, num_dense] float32, ids [num_sparse, B] int64 (feature-major) -> PredictRequest bytes."""
    dense = np.ascontiguousarray(dense, dtype=np.float32)
    ids = np.ascontiguousarray(ids, dtype=np.int64)
    B, nd = dense.shape
    ns = ids.shape[0]
    assert ids.shape[1] == B
    return struct.pack("<6I", REQ_MAGIC, 1, B, nd, ns, 0) + dense.tobytes() + ids.tobytes()


def decode_response(buf: bytes) -> Tuple[np.ndarray, int, int]:
    magic, batch, status, _r, version = struct.unpack_from("<4Iq", buf, 0)
    if magic != RESP_MAGIC:
        raise ValueError("bad PredictResponse")
    n_out = _r if _r > 1 else 1                          # multi-task models: `reserved` = probabilities per row -> [batch, n_out]
    probs = np.frombuffer(buf, dtype=np.float32, count=batch * n_out, offset=24).copy()
    return (probs.reshape(batch, n_out) if n_out > 1 else probs), status, version


class _Abi:
    """The four entry points (+ release / free) of one runtime, bound with ctypes."""

    def __init__(self, lib, prefix: str):
        def fn(name, restype, argtypes):
            f = getattr(lib, prefix + name)
            f.restype, f.argtypes = restype, argtypes
            return f
        self.initialize = fn("initialize", C.c_void_p, [C.c_char_p, C.c_char_p, C.POINTER(C.c_int)])
        self.process = fn("process", C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int)])
        self.batch_process = fn("batch_process", C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_void_p), C.POINTER(C.c_int)])
        self.get_serving_model_info = fn("get_serving_model_info", C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int)])
        rel = "dr_cpu_serving_" if prefix else "dr_serving_"
        self.dr_serving_release, self.dr_serving_free = getattr(lib, rel + "release"), getattr(lib, rel + "free")
        self.dr_serving_release.argtypes, self.dr_serving_free.argtypes = [C.c_void_p], [C.c_void_p]
        self.dr_serving_release.restype = self.dr_serving_free.restype = None


class Processor:
    """``device="cuda"``: the GPU runtime (csrc/cuda/serving_runtime.cu: device tables, bf16 / fp8 wgmma MLP; DLRM exports and op-program
    exports of the other Criteo-style models);
    ``device="cpu"``: the CPU runtime (csrc/host/cpu_serving.cc: host tables, fp32 MLP on the OpenMP pool).  Same saved-model directory,
    request encodings, ModelConfig keys and hot-swap protocol.  Default: cuda when a GPU is visible, else cpu."""

    def __init__(self, savedmodel_dir: str, config: dict | None = None, device: str | None = None):
        program = False
        try:
            with open(os.path.join(savedmodel_dir, "saved_model.json")) as f:
                program = json.load(f).get("arch") == "program"
        except (OSError, ValueError):
            pass
        if device is None:
            import torch
            # both runtimes interpret op-program exports (DeepFM, DCN, WDL, ... -- export_saved_model_program): the GPU one runs the LINEAR ops
            # on the wgmma GEMM and the glue ops on csrc/cuda/program_kernels.cu, the CPU one is csrc/host/cpu_serving.cc::RunProgram
            device = "cuda" if torch.cuda.is_available() else "cpu"
        self.device, self.program = device, program
        if device == "cpu":
            from .. import _native
            self.lib = _Abi(_native.host(), "dr_cpu_")
        elif device == "cuda_emu":
            # the GPU runtime compiled for the host (csrc/cuda/emu/cuda_emu.h: one host thread per CUDA thread, host-loop GEMM stand-in): CPU CI of
            # the op-program interpreter and its kernels, optionally under ASAN / TSAN (DEEPREC_EMU_SANITIZE)
            self.lib = _Abi(C.CDLL(_build.build_cuda_emu(os.environ.get("DEEPREC_EMU_SANITIZE") or None)), "")
        else:
            path = os.path.join(_build.LIB, "libdeeprec_cuda.so")
            if not os.path.exists(path):
                path = _build.build_cuda()
            self.lib = _Abi(C.CDLL(path), "")
        state = C.c_int(0)
        cfg = dict(config or {})
        self.model = self.lib.initialize(savedmodel_dir.encode(), json.dumps(cfg).encode(), C.byref(state))
        if not self.model or state.value != 0:
            raise RuntimeError(f"Processor.initialize failed for {savedmodel_dir} (state {state.value})")

    def process(self, request: bytes) -> Tuple[int, bytes]:
        out, n = C.c_void_p(), C.c_int(0)
        rc = self.lib.process(self.model, request, len(request), C.byref(out), C.byref(n))
        data = C.string_at(out, n.value) if out else b""
        if out:
            self.lib.dr_serving_free(out)
        return rc, data

    def predict(self, dense: np.ndarray, ids: np.ndarray) -> np.ndarray:
        rc, data = self.process(encode_request(dense, ids))
        if rc != 200:
            raise RuntimeError(f"process returned {rc}")
        return decode_response(data)[0]

    def predict_proto(self, request_pb: bytes) -> bytes:
        """PredictRequest protobuf bytes -> PredictResponse protobuf bytes (the runtime's ``process`` accepts both encodings)."""
        rc, data = self.process(request_pb)
        if rc != 200:
            raise RuntimeError(f"process returned {rc}")
        return data

    def batch_process(self, requests: Sequence[bytes]) -> Tuple[int, List[bytes]]:
        n = len(requests)
        bufs = [C.create_string_buffer(r, len(r)) for r in requests]
        ins = (C.c_void_p * n)(*[C.cast(b, C.c_void_p) for b in bufs])
        sizes = (C.c_int * (n + 1))(n, *[len(r) for r in requests])
        outs = (C.c_void_p * n)()
        osz = (C.c_int * n)()
        rc = self.lib.batch_process(self.model, ins, sizes, outs, osz)
        res = []
        for i in range(n):
            res.append(C.string_at(outs[i], osz[i]) if outs[i] else b"")
            if outs[i]:
                self.lib.dr_serving_free(outs[i])
        return rc, res

    def model_info(self) -> dict:
        out, n = C.c_void_p(), C.c_int(0)
        self.lib.get_serving_model_info(self.model, C.byref(out), C.byref(n))
        s = C.string_at(out, n.value).decode()
        self.lib.dr_serving_free(out)
        return json.loads(s)

    def close(self) -> None:
        if self.model:
            self.lib.dr_serving_release(self.model)
            self.model = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ProcessorGroup:
    """One native Processor per GPU behind a single ``process`` entry (ModelConfig ``gpu_ids_list``; SessionGroup.md: total sessions =
    ``session_num x len(gpu_ids)``).  Every replica polls the same ``checkpoint_dir`` and hot-swaps on its own; requests go to the
    replicas round-robin (``RR``) or by ``hint % n`` / thread id (``MOD``), each replica then picks one of its sessions."""

    def __init__(self, savedmodel_dir: str, config: dict | None = None):
        import itertools
        import threading
        cfg = dict(config or {})
        gpus = list(cfg.pop("gpu_ids_list", None) or [cfg.get("gpu_id", 0)])
        self.policy = str(cfg.get("select_session_policy", "RR")).upper()
        self.replicas: List[Processor] = [Processor(savedmodel_dir, dict(cfg, gpu_id=int(g)), device="cuda") for g in gpus]
        self.gpu_ids = [int(g) for g in gpus]
        self._rr = itertools.count()
        self._ident = threading.get_ident

    def _pick(self, hint: int | None) -> Processor:
        n = len(self.replicas)
        if self.policy == "MOD":
            return self.replicas[(hint if hint is not None else self._ident()) % n]
        return self.replicas[next(self._rr) % n]

    def process(self, request: bytes, hint: int | None = None) -> Tuple[int, bytes]:
        return self._pick(hint).process(request)

    def predict(self, dense: np.ndarray, ids: np.ndarray, hint: int | None = None) -> np.ndarray:
        return self._pick(hint).predict(dense, ids)

    def batch_process(self, requests: Sequence[bytes]) -> Tuple[int, List[bytes]]:
        """Requests are spread over the replicas (request i -> replica i % n), each replica runs its share as one batch_process call."""
        n = len(self.replicas)
        out: List[bytes] = [b""] * len(requests)
        rc_all = 200
        for r, proc in enumerate(self.replicas):
            idx = list(range(r, len(requests), n))
            if not idx:
                continue
            rc, res = proc.batch_process([requests[i] for i in idx])
            rc_all = rc if rc != 200 else rc_all
            for i, b in zip(idx, res):
                out[i] = b
        return rc_all, out

    def model_info(self) -> dict:
        infos = [p.model_info() for p in self.replicas]
        return {"gpu_ids": self.gpu_ids, "sessions": sum(i["sessions"] for i in infos), "requests": sum(i["requests"] for i in infos),
                "failures": sum(i["failures"] for i in infos), "model_version": min(i["model_version"] for i in infos), "replicas": infos}

    def close(self) -> None:
        for p in self.replicas:
            p.close()
