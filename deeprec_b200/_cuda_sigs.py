"""ctypes signatures of libdeeprec_cuda.so (csrc/cuda/*.cu, extern "C" section of each file)."""
from __future__ import annotations

import ctypes as C

i64, i32, f32, vp = C.c_int64, C.c_int32, C.c_float, C.c_void_p
P = C.c_void_p
INT = C.c_int


class DeviceTableStruct(C.Structure):
    """Mirror of DrDeviceTable (csrc/cuda/table.cuh)."""
    _fields_ = [
        ("slots", vp),
        ("rows", vp), ("free_list", vp), ("counters", vp), ("default_matrix", vp), ("bloom", vp),
        ("capacity", i64), ("row_capacity", i64), ("default_value_dim", i64), ("bloom_m", i64),
        ("dim", i32), ("stride", i32), ("num_slots", i32), ("has_scalars", i32),
        ("filter_type", i32), ("filter_freq", i32), ("bloom_k", i32), ("is_inference", i32),
        ("no_permission", f32), ("slot_init", f32 * 4),
        ("steps_to_live", i32), ("l2_weight_threshold", f32),
    ]


_MISSING_OK = False


def _sig(lib, name, argtypes, restype=INT):
    if _MISSING_OK and not hasattr(lib, name):
        return None
    fn = getattr(lib, name)
    fn.argtypes = argtypes
    fn.restype = restype
    return fn


def bind(lib, missing_ok: bool = False):
    global _MISSING_OK
    _MISSING_OK = missing_ok
    try:
        return _bind(lib)
    finally:
        _MISSING_OK = False


def _bind(lib):
    from ._native import OptHyper
    TP = C.POINTER(DeviceTableStruct)
    HP = C.POINTER(OptHyper)
    S = vp  # cudaStream_t
    _sig(lib, "dr_cuda_sizeof_table", [])
    _sig(lib, "dr_cuda_fill_i64", [P, i64, i64, S])
    _sig(lib, "dr_cuda_table_lookup", [P, P, INT, P, P, i64, i64, INT, P, P, P, P, i64, S])
    _sig(lib, "dr_cuda_table_gather", [P, P, INT, INT, P, P, P, i64, i64, P, INT, i64, i64, INT, S])
    _sig(lib, "dr_cuda_table_init_slots", [P, i64, S])
    _sig(lib, "dr_cuda_table_get_meta", [TP, P, i64, P, P, P, S])
    _sig(lib, "dr_cuda_table_gather_slot", [TP, P, i64, INT, P, S])
    _sig(lib, "dr_cuda_table_rehash", [TP, TP, S])
    _sig(lib, "dr_cuda_table_shrink", [TP, INT, P, S])
    _sig(lib, "dr_cuda_table_remove", [TP, P, i64, P, S])
    _sig(lib, "dr_cuda_table_snapshot", [TP, INT, INT, INT, P, P, P, P, P, P, P, P, S])
    _sig(lib, "dr_cuda_table_export_keys", [TP, P, i64, P, P, P, P, S])
    _sig(lib, "dr_cuda_table_clear_dirty", [TP, S])
    _sig(lib, "dr_cuda_table_import", [TP, P, P, INT, P, P, i64, INT, INT, INT, P, S])
    _sig(lib, "dr_cuda_sparse_accumulate", [P, P, INT, INT, P, P, i64, i64, P, INT, i64, i64, INT, P, P, P, S])
    _sig(lib, "dr_cuda_sparse_apply", [P, P, P, i64, P, INT, P, i64, INT, S])
    _sig(lib, "dr_cuda_advance_hyper", [P, S])
    _sig(lib, "dr_cuda_dense_apply", [P, P, P, P, i64, P, f32, P, S])
    _sig(lib, "dr_cuda_combine_fwd", [P, P, INT, i64, INT, P, P, P, P, P, P, INT, i64, i64, P, P, S])
    _sig(lib, "dr_cuda_unique", [P, i64, P, P, i64, P, P, P, P, P, S])
    _sig(lib, "dr_cuda_segment_sum", [P, P, i64, INT, P, S])
    _sig(lib, "dr_cuda_gemm_tn", [P, i64, P, i64, INT, INT, INT, P, INT, P, i64, P, i64, P, INT, S])
    _sig(lib, "dr_cuda_gemm_tn_ex", [P, i64, P, i64, INT, INT, INT, P, INT, P, i64, INT, P, i64, P, P, P, INT, INT, S])
    _sig(lib, "dr_cuda_gemm_fp8_tn", [P, i64, P, i64, INT, INT, INT, P, P, INT, P, i64, INT, f32, S])
    _sig(lib, "dr_cuda_quantize_e4m3", [P, INT, i64, INT, i64, P, INT, f32, S])
    _sig(lib, "dr_cuda_quantize_weights_e4m3", [P, INT, INT, i64, P, INT, P, S])
    _sig(lib, "dr_cuda_absmax_bf16", [P, i64, P, S])
    _sig(lib, "dr_cuda_quantize_mxfp8", [P, INT, i64, INT, i64, P, INT, P, S])
    _sig(lib, "dr_cuda_gemm_mxfp8_tn", [P, P, P, P, INT, INT, INT, P, INT, P, i64, INT, S])
    _sig(lib, "dr_cuda_bn_fold", [P, P, INT, i64, P, P, f32, f32, P, P, P, P, P, P, INT, P, P, INT, INT, P, P, S])
    _sig(lib, "dr_cuda_dw_fixup", [P, P, P, P, INT, INT, INT, S])
    _sig(lib, "dr_cuda_bn_bwd_apply_v2", [P, P, i64, INT, i64, P, P, P, P, P, P, INT, P, S])
    _sig(lib, "dr_cuda_gemm_dw", [P, i64, P, i64, INT, INT, INT, P, i64, INT, S])
    _sig(lib, "dr_cuda_colstats", [P, P, i64, INT, i64, i64, P, P, S])
    _sig(lib, "dr_cuda_bn_finalize", [P, P, INT, i64, P, P, f32, f32, P, P, P, P, P, P, INT, S])
    _sig(lib, "dr_cuda_bn_apply", [P, i64, INT, i64, P, P, P, i64, S])
    _sig(lib, "dr_cuda_bn_bwd_finalize", [P, P, INT, i64, P, P, P, P, P, P, f32, S])
    _sig(lib, "dr_cuda_bn_bwd_apply", [P, P, i64, INT, i64, P, P, P, P, P, P, INT, S])
    _sig(lib, "dr_cuda_head", [P, i64, i64, INT, P, P, P, f32, P, P, P, P, P, INT, INT, P, S])
    _sig(lib, "dr_cuda_pack_weights", [P, INT, INT, P, P, INT, S])
    _sig(lib, "dr_cuda_cast_pad", [P, i64, INT, P, INT, S])
    _sig(lib, "dr_cuda_l2_flush", [P, i64, f32, S])
    _sig(lib, "dr_cuda_dot_interaction_fwd", [P, i64, P, i64, i64, INT, INT, i64, P, i64, S])
    _sig(lib, "dr_cuda_dot_interaction_bwd", [P, i64, P, i64, P, i64, i64, INT, INT, i64, P, i64, P, i64, i64, S])
    _sig(lib, "dr_cuda_fm_fwd", [P, i64, i64, INT, INT, i64, P, i64, P, S])
    _sig(lib, "dr_cuda_fm_bwd", [P, i64, P, i64, i64, P, INT, INT, i64, P, i64, i64, INT, S])
    _sig(lib, "dr_cuda_gru_fwd", [P, P, P, P, INT, INT, INT, P, S])
    _sig(lib, "dr_cuda_gru_bwd", [P, P, P, P, P, P, INT, INT, INT, P, P, P, P, P, S])
    # comm (optional symbols: present once comm_kernels.cu is built)
    for name, args in _COMM_SIGS.items():
        if hasattr(lib, name):
            _sig(lib, name, args[0], args[1] if len(args) > 1 else INT)
    return lib


_COMM_SIGS: dict = {}


def register_comm_sig(name, argtypes, restype=INT):
    _COMM_SIGS[name] = (argtypes, restype)
