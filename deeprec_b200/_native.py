"""ctypes bindings to the two in-tree native libraries.

``host()``  -> libdeeprec_host.so  (C++17 host engine; always available, built on demand)
``cuda()``  -> libdeeprec_cuda.so  (sm_90a kernels; REQUIRED on a GPU box: no silent
                                    eager/PyTorch fallback -- a missing library raises)
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import torch

from . import build as _build

_LOCK = threading.Lock()
_HOST = None
_CUDA = None

i64 = C.c_int64
i32 = C.c_int32
f32 = C.c_float
f64 = C.c_double
vp = C.c_void_p
cp = C.c_char_p


class EvConfig(C.Structure):
    """Mirror of DrEvConfig (csrc/common/ev_types.h)."""
    _fields_ = [
        ("dim", i64), ("num_slots", i32), ("has_scalars", i32), ("init_capacity", i64),
        ("filter_type", i32), ("bloom_counter_bits", i32), ("filter_freq", i64),
        ("bloom_max_elements", i64), ("bloom_fpp", f64), ("steps_to_live", i64),
        ("l2_weight_threshold", f32), ("default_value_no_permission", f32),
        ("default_value_dim", i64), ("record_freq", i32), ("record_version", i32),
        ("is_inference", i32), ("storage_type", i32), ("hbm_cache_rows", i64),
        ("cache_strategy", i32), ("num_partitions", i32), ("slot_init", f32 * 4),
    ]


class OptHyper(C.Structure):
    """Mirror of DrOptHyper (csrc/common/ev_types.h)."""
    _fields_ = [
        ("kind", i32), ("apply_sparse_rmsprop", i32),
        ("lr", f32), ("beta1", f32), ("beta2", f32), ("epsilon", f32),
        ("beta1_power", f32), ("beta2_power", f32), ("weight_decay", f32),
        ("l1", f32), ("l2", f32), ("l2_shrinkage", f32), ("lr_power", f32),
        ("decay_rate", f32), ("decay_baseline", f32), ("init_accum", f32),
        ("decay_step", i64), ("global_step", i64),
    ]


def _sig(lib, name, restype, argtypes):
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = argtypes
    return fn


def _bind_host(lib):
    P = vp
    _sig(lib, "dr_host_ev_create", vp, [C.POINTER(EvConfig)])
    _sig(lib, "dr_host_ev_destroy", None, [vp])
    _sig(lib, "dr_host_ev_stride", i64, [vp])
    _sig(lib, "dr_host_ev_set_default", None, [vp, P])
    _sig(lib, "dr_host_ev_size", i64, [vp])
    _sig(lib, "dr_host_ev_total_keys", i64, [vp])
    _sig(lib, "dr_host_ev_lookup", None, [vp, P, i64, P])
    _sig(lib, "dr_host_ev_lookup_slot", None, [vp, P, i64, C.c_int, P])
    _sig(lib, "dr_host_ev_get_freq", None, [vp, P, i64, P])
    _sig(lib, "dr_host_ev_get_version", None, [vp, P, i64, P])
    _sig(lib, "dr_host_ev_apply", None, [vp, P, P, P, i64, C.POINTER(OptHyper)])
    _sig(lib, "dr_host_ev_shrink", i64, [vp, i64])
    _sig(lib, "dr_host_ev_remove", i64, [vp, P, i64])
    _sig(lib, "dr_host_ev_snapshot_begin", None, [vp, C.c_int, C.c_int, C.c_int, C.POINTER(i64), C.POINTER(i64)])
    _sig(lib, "dr_host_ev_snapshot_read", None, [vp] + [P] * 9)
    _sig(lib, "dr_host_ev_snapshot_end", None, [vp])
    _sig(lib, "dr_host_ev_clear_dirty", None, [vp])
    _sig(lib, "dr_host_ev_import", i64, [vp, P, P, i64, P, P, i64, C.c_int, C.c_int, C.c_int])
    _sig(lib, "dr_host_ev_export_keys", None, [vp, P, i64, P, P, P, P])
    _sig(lib, "dr_host_bloom_info", i64, [vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)])
    _sig(lib, "dr_host_bloom_read", None, [vp, P])
    _sig(lib, "dr_host_bloom_write", None, [vp, P])
    _sig(lib, "dr_host_unique", i64, [P, i64, P, P, P])
    _sig(lib, "dr_host_segment_sum", None, [P, P, i64, i64, P, i64])
    _sig(lib, "dr_host_num_threads", C.c_int, [])
    _sig(lib, "dr_host_dot_interaction_fwd", None, [P, P, i64, C.c_int, C.c_int, P])
    _sig(lib, "dr_host_dot_interaction_bwd", None, [P, P, P, i64, C.c_int, C.c_int, P, P])
    _sig(lib, "dr_host_ev_apply_raw", None, [vp, P, i64, P, i64, C.POINTER(OptHyper)])
    _sig(lib, "dr_host_ev_apply_multi", None, [vp, C.c_int, P, P, P, P, P, C.POINTER(OptHyper)])
    _sig(lib, "dr_host_ev_lookup_pooled", None, [vp, P, i64, i64, P, i64])
    _sig(lib, "dr_host_group_lookup", None, [P, C.c_int, P, i64, P])
    _sig(lib, "dr_host_group_apply_raw", None, [P, C.c_int, P, i64, P, C.POINTER(OptHyper)])
    # SSD tier (csrc/host/ssd_store.cc)
    _sig(lib, "dr_ssd_create", vp, [cp, i64, i64, C.c_int])
    _sig(lib, "dr_ssd_destroy", None, [vp])
    for nm in ("dr_ssd_size", "dr_ssd_num_files", "dr_ssd_bytes", "dr_ssd_compactions"):
        _sig(lib, nm, i64, [vp])
    _sig(lib, "dr_ssd_put", None, [vp, P, P, P, P, i64])
    _sig(lib, "dr_ssd_get", None, [vp, P, i64, P, P, P, P])
    _sig(lib, "dr_ssd_contains", None, [vp, P, i64, P])
    _sig(lib, "dr_ssd_remove", i64, [vp, P, i64])
    _sig(lib, "dr_ssd_export_keys", i64, [vp, P, i64])
    _sig(lib, "dr_ssd_compact", i64, [vp, C.c_double])
    _sig(lib, "dr_ssd_flush", None, [vp])
    # io runtime
    _sig(lib, "dr_bundle_writer_open", vp, [cp])
    _sig(lib, "dr_bundle_writer_add", C.c_int, [vp, cp, cp, P, C.c_int, P, i64])
    _sig(lib, "dr_bundle_writer_close", C.c_int, [vp])
    _sig(lib, "dr_bundle_reader_open", vp, [cp])
    _sig(lib, "dr_bundle_reader_close", None, [vp])
    _sig(lib, "dr_bundle_reader_count", i64, [vp])
    _sig(lib, "dr_bundle_reader_entry", C.c_int, [vp, i64, C.c_char_p, C.c_int, C.c_char_p, C.c_int, P, C.POINTER(i64)])
    _sig(lib, "dr_bundle_reader_read", C.c_int, [vp, cp, P, i64, C.c_int])
    _sig(lib, "dr_stage_create", vp, [i64])
    _sig(lib, "dr_stage_destroy", None, [vp])
    _sig(lib, "dr_stage_put", C.c_int, [vp, i64, i64])
    _sig(lib, "dr_stage_take", C.c_int, [vp, C.POINTER(i64), i64])
    _sig(lib, "dr_stage_close", None, [vp])
    _sig(lib, "dr_stage_cancel", i64, [vp, P, i64])
    _sig(lib, "dr_stage_resume", None, [vp])
    _sig(lib, "dr_stage_size", i64, [vp])
    _sig(lib, "dr_wq_create", vp, [cp, i64, C.c_int, C.c_uint64])
    _sig(lib, "dr_wq_destroy", None, [vp])
    _sig(lib, "dr_wq_take", C.c_int, [vp, C.c_char_p, C.c_int])
    _sig(lib, "dr_wq_add", None, [vp, cp])
    _sig(lib, "dr_wq_state", None, [vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)])
    _sig(lib, "dr_wq_restore", None, [vp, i64, i64])
    _sig(lib, "dr_wq_remaining", i64, [vp])
    _sig(lib, "dr_gen_criteo", None, [C.c_uint64, i64, C.c_int, C.c_int, P, f64, P, P, P, C.c_int])
    _sig(lib, "dr_gen_taobao", None, [C.c_uint64, i64, C.c_int, i64, i64, i64, f64, P, P, P, P, P, P, P])
    return lib


def host():
    global _HOST
    if _HOST is None:
        with _LOCK:
            if _HOST is None:
                path = _build.build_host()
                _HOST = _bind_host(C.CDLL(path))
    return _HOST


def cuda_available() -> bool:
    return torch.cuda.is_available()


_EMU = None          # libdeeprec_cuda_emu.so (csrc/cuda/emu/cuda_emu.h): the SIMT kernels compiled for the host
_EMU_DEPTH = 0


class cuda_emulation:
    """``with cuda_emulation():`` -- the op wrappers that support it treat CPU tensors as device tensors and call the CUDA-on-CPU emulation
    build of the same kernels (one host thread per CUDA thread; ``sanitize="address"`` / ``"thread"`` builds need the sanitizer runtime
    preloaded).  For CPU CI of kernel logic, never a production path: it is 3-4 orders of magnitude slower than the GPU."""

    def __init__(self, sanitize: str | None = None):
        self.sanitize = sanitize or os.environ.get("DEEPREC_EMU_SANITIZE") or None

    def __enter__(self):
        global _EMU, _EMU_DEPTH
        with _LOCK:
            if _EMU is None or getattr(_EMU, "_sanitize", None) != self.sanitize:
                lib = C.CDLL(_build.build_cuda_emu(self.sanitize))
                lib._sanitize = self.sanitize
                _EMU = lib
            _EMU_DEPTH += 1
        return _EMU

    def __exit__(self, *exc):
        global _EMU_DEPTH
        with _LOCK:
            _EMU_DEPTH -= 1
        return False


def emu_active() -> bool:
    return _EMU_DEPTH > 0


def on_device(t: torch.Tensor) -> bool:
    """Dispatch predicate of the op wrappers: CUDA tensors, or any tensor while the kernel emulation is active."""
    return t.is_cuda or _EMU_DEPTH > 0


def cuda():
    """The sm_90a kernel library.  Raises if it is missing (never falls back silently)."""
    global _CUDA
    if _EMU_DEPTH > 0:
        if not getattr(_EMU, "_sigs_bound", False):
            from . import _cuda_sigs
            _cuda_sigs.bind(_EMU, missing_ok=True)          # entry points of the wgmma / NVLS translation units do not exist in the emulation
            _EMU._sigs_bound = True
        return _EMU
    if _CUDA is None:
        with _LOCK:
            if _CUDA is None:
                path = os.path.join(_build.LIB, "libdeeprec_cuda.so")
                if not os.path.exists(path):
                    path = _build.build_cuda()
                from . import _cuda_sigs
                lib = _cuda_sigs.bind(C.CDLL(path))
                lib.dr_cuda_set_device.argtypes, lib.dr_cuda_set_device.restype = [C.c_int], C.c_int
                lib.dr_cuda_set_sparse_blocks_per_sm.argtypes, lib.dr_cuda_set_sparse_blocks_per_sm.restype = [C.c_int], C.c_int
                if torch.cuda.is_available():
                    lib.dr_cuda_set_device(torch.cuda.current_device())
                _CUDA = lib
    return _CUDA


def stream_sync(device=None) -> None:
    """Wait for the current stream (no-op while the kernel emulation is active: emulated launches are synchronous)."""
    if _EMU_DEPTH > 0:
        return
    torch.cuda.current_stream(device).synchronize()


def device_sync(device=None) -> None:
    """torch.cuda.synchronize(device), or nothing while the kernel emulation is active."""
    if _EMU_DEPTH > 0:
        return
    torch.cuda.synchronize(device)


def set_device(index: int) -> None:
    """The kernel library links its own static cudart: its current device must follow torch's."""
    if _EMU_DEPTH > 0:
        return
    rc = cuda().dr_cuda_set_device(int(index))
    if rc != 0:
        raise RuntimeError(f"dr_cuda_set_device({index}) failed: {rc}")


def ptr(t: torch.Tensor | None):
    """Raw data pointer of a contiguous tensor (or NULL)."""
    if t is None:
        return None
    assert t.is_contiguous(), "native ops need contiguous tensors"
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    if _EMU_DEPTH > 0:
        return None
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
