"""ctypes declarations of libdeeprec_cuda.so: every entry point the package calls (the extern "C" section of each csrc/cuda/*.cu) and
the C structs they take.  ``_native`` binds them when it loads the library (tests/test_cuda_sigs.py checks them against the C sources)."""
from __future__ import annotations

import ctypes as C

i64, i32, u32, f32, vp = C.c_int64, C.c_int32, C.c_uint32, C.c_float, C.c_void_p
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


class Peers(C.Structure):
    """Mirror of DrPeers (csrc/cuda/sp_sync.cuh)."""
    _fields_ = [("ptr", vp * 16)]


class SpSync(C.Structure):
    """Mirror of DrSpSync."""
    _fields_ = [("flags", Peers), ("state", vp), ("rank", i32), ("W", i32)]


class SpGeom(C.Structure):
    """Mirror of DrSpGeom."""
    _fields_ = [("col_table", vp), ("hoff", vp), ("boff", vp), ("C", i32), ("T", i32), ("W", i32), ("rank", i32), ("B", i64),
                ("dim", i32), ("ldinv", i32), ("pad_key", i64)]


class SpBags(C.Structure):
    """Mirror of DrSpBags."""
    _fields_ = [("off", vp), ("comb", vp), ("col_bag", vp), ("F", i32)]


class AgGeom(C.Structure):
    """Mirror of DrAgGeom."""
    _fields_ = [("W", i32), ("rank", i32), ("dim", i32), ("table_index", i32), ("B", i64), ("nnz_cap", i64)]


class AgPeers(C.Structure):
    """Mirror of DrAgPeers."""
    _fields_ = [("keys", Peers), ("rows", Peers), ("meta", Peers), ("partial", Peers), ("grad", Peers)]


SIGNATURES: dict = {}          # entry point -> (argtypes, restype)


def _sig(name, argtypes, restype=INT):
    SIGNATURES[name] = (argtypes, restype)


TP = C.POINTER(DeviceTableStruct)
PP, SP, GP, BP = C.POINTER(Peers), C.POINTER(SpSync), C.POINTER(SpGeom), C.POINTER(SpBags)
AGP, APP = C.POINTER(AgGeom), C.POINTER(AgPeers)
S = vp  # cudaStream_t
# tables, optimizers, embedding
_sig("dr_cuda_sizeof_table", [])
_sig("dr_cuda_fill_i64", [P, i64, i64, S])
_sig("dr_cuda_table_lookup", [P, P, INT, P, P, i64, i64, INT, P, P, P, P, i64, S])
_sig("dr_cuda_table_gather", [P, P, INT, INT, P, P, P, i64, i64, P, INT, i64, i64, INT, S])
_sig("dr_cuda_table_init_slots", [P, i64, S])
_sig("dr_cuda_table_get_meta", [TP, P, i64, P, P, P, S])
_sig("dr_cuda_table_gather_slot", [TP, P, i64, INT, P, S])
_sig("dr_cuda_table_rehash", [TP, TP, S])
_sig("dr_cuda_table_shrink", [TP, INT, P, S])
_sig("dr_cuda_table_remove", [TP, P, i64, P, S])
_sig("dr_cuda_table_snapshot", [TP, INT, INT, INT, P, P, P, P, P, P, P, P, S])
_sig("dr_cuda_table_snapshot_since", [TP, i64, P, P, P, P, P, S])
_sig("dr_cuda_table_export_keys", [TP, P, i64, P, P, P, P, S])
_sig("dr_cuda_table_clear_dirty", [TP, S])
_sig("dr_cuda_table_import", [TP, P, P, INT, P, P, i64, INT, INT, INT, P, S])
_sig("dr_cuda_sparse_accumulate", [P, P, INT, INT, P, P, i64, i64, P, INT, i64, i64, INT, P, P, P, S])
_sig("dr_cuda_sparse_apply", [P, P, P, i64, P, INT, P, i64, INT, S])
_sig("dr_cuda_advance_hyper", [P, S])
_sig("dr_cuda_dense_apply", [P, P, P, P, i64, P, f32, P, S])
_sig("dr_cuda_combine_fwd", [P, P, INT, i64, INT, P, P, P, P, P, P, INT, i64, i64, P, P, S])
_sig("dr_cuda_unique", [P, i64, P, P, i64, P, P, P, P, P, S])
_sig("dr_cuda_segment_sum", [P, P, i64, INT, P, S])
# GEMM, quantisation, BatchNorm, head
_sig("dr_cuda_gemm_tn", [P, i64, P, i64, INT, INT, INT, P, INT, P, i64, P, i64, P, INT, S])
_sig("dr_cuda_gemm_tn_ex", [P, i64, P, i64, INT, INT, INT, P, INT, P, i64, INT, P, i64, P, P, P, INT, INT, S])
_sig("dr_cuda_gemm_tn_cross", [P, i64, P, i64, INT, INT, INT, P, INT, P, i64, P, i64, P, i64, P, i64, INT, S])
_sig("dr_cuda_gemm_tn_ln", [P, i64, P, i64, INT, INT, INT, P, P, P, f32, INT, P, i64, P, i64, P, INT, S])
_sig("dr_cuda_gemm_fp8_tn", [P, i64, P, i64, INT, INT, INT, P, P, INT, P, i64, INT, f32, S])
_sig("dr_cuda_quantize_e4m3", [P, INT, i64, INT, i64, P, INT, f32, S])
_sig("dr_cuda_quantize_weights_e4m3", [P, INT, INT, i64, P, INT, P, S])
_sig("dr_cuda_absmax_bf16", [P, i64, P, S])
_sig("dr_cuda_quantize_mxfp8", [P, INT, i64, INT, i64, P, INT, P, S])
_sig("dr_cuda_gemm_mxfp8_tn", [P, P, P, P, INT, INT, INT, P, INT, P, i64, INT, S])
_sig("dr_cuda_bn_fold", [P, P, INT, i64, P, P, f32, f32, P, P, P, P, P, P, INT, P, P, INT, INT, P, P, S])
_sig("dr_cuda_dw_fixup", [P, P, P, P, INT, INT, INT, S])
_sig("dr_cuda_bn_bwd_apply_v2", [P, P, i64, INT, i64, P, P, P, P, P, P, INT, P, S])
_sig("dr_cuda_gemm_dw", [P, i64, P, i64, INT, INT, INT, P, i64, INT, S])
_sig("dr_cuda_gemm_tn_grouped", [INT, P, P, P, P, INT, INT, INT, P, INT, P, P, P, P, P, INT, S])
_sig("dr_cuda_gemm_dw_grouped", [INT, P, P, P, P, INT, INT, INT, P, P, INT, S])
_sig("dr_cuda_moe_mix_fwd", [P, i64, i64, INT, INT, INT, P, P, P, P, P, P, P, P, P, P, S])
_sig("dr_cuda_moe_mix_bwd", [P, i64, i64, INT, INT, INT, P, P, P, P, P, P, P, P, P, P, i64, P, P, P, S])
_sig("dr_cuda_colstats", [P, P, i64, INT, i64, i64, P, P, S])
_sig("dr_cuda_bn_finalize", [P, P, INT, i64, P, P, f32, f32, P, P, P, P, P, P, INT, S])
_sig("dr_cuda_bn_apply", [P, i64, INT, i64, P, P, P, i64, S])
_sig("dr_cuda_bn_bwd_finalize", [P, P, INT, i64, P, P, P, P, P, P, f32, S])
_sig("dr_cuda_bn_bwd_apply", [P, P, i64, INT, i64, P, P, P, P, P, P, INT, S])
_sig("dr_cuda_head", [P, i64, i64, INT, P, P, P, f32, P, P, P, P, P, INT, INT, P, S])
_sig("dr_cuda_det_colsum", [P, INT, i64, INT, P, P, S])
_sig("dr_cuda_pack_weights", [P, INT, INT, P, P, INT, S])
_sig("dr_cuda_cross_bwd", [P, i64, P, i64, P, i64, i64, INT, P, i64, P, i64, INT, P, S])
_sig("dr_cuda_cross_split", [P, i64, P, i64, i64, INT, INT, P, i64, P, S])
_sig("dr_cuda_ln_relu_bwd", [P, i64, P, i64, P, i64, P, P, i64, INT, P, i64, P, P, S])
_sig("dr_cuda_bn_apply_mul", [P, i64, P, P, P, i64, i64, INT, P, i64, S])
_sig("dr_cuda_bn_mul_bwd", [P, i64, P, i64, P, i64, P, P, i64, INT, P, i64, P, i64, P, P, S])
_sig("dr_cuda_cast_pad", [P, i64, INT, P, INT, S])
_sig("dr_cuda_l2_flush", [P, i64, f32, S])
# interactions, GRU, self-attention, DIN attention, fused element-wise ops
_sig("dr_cuda_dot_interaction_fwd", [P, i64, P, i64, i64, INT, INT, i64, P, i64, S])
_sig("dr_cuda_dot_interaction_bwd", [P, i64, P, i64, P, i64, i64, INT, INT, i64, P, i64, P, i64, i64, S])
_sig("dr_cuda_dot_interaction_fwd_u", [P, i64, P, P, INT, INT, INT, i64, P, i64, SP, S])
_sig("dr_cuda_dot_interaction_bwd_u", [P, i64, P, i64, P, P, INT, INT, INT, i64, P, i64, P, i64, i64, S])
_sig("dr_cuda_dlrm_inter_gemm", [P, i64, P, P, INT, INT, INT, i64, P, i64, INT, P, P, i64, P, i64, SP, S])
_sig("dr_cuda_fm_fwd", [P, i64, i64, INT, INT, i64, P, i64, P, S])
_sig("dr_cuda_fm_bwd", [P, i64, P, i64, i64, P, INT, INT, i64, P, i64, i64, INT, S])
_sig("dr_cuda_gru_fwd", [P, P, P, P, INT, INT, INT, P, S])
_sig("dr_cuda_gru_bwd", [P, P, P, P, P, P, INT, INT, INT, P, P, P, P, P, S])
_sig("dr_cuda_mha_fwd", [P, P, INT, INT, INT, INT, P, S])
_sig("dr_cuda_mha_bwd", [P, P, P, P, INT, INT, INT, INT, P, S])
_sig("dr_cuda_din_att_fwd", [P, P, INT, P, INT, INT, INT, P, P, INT, P, P, INT, P, INT, P, S])
_sig("dr_cuda_din_att_bwd", [P, P, INT, P, P, INT, INT, INT, P, P, INT, P, P, INT, P, INT, P, P, P, P, P, P, P, P, P, S])
_sig("dr_cuda_din_attention_fwd", [P, P, P, i64, INT, INT, P, P, INT, P, P, INT, P, f32, P, S])
_sig("dr_cuda_din_attention_bwd", [P, P, P, P, i64, INT, INT, P, P, INT, P, P, INT, P, f32, P, P, P, P, P, P, P, P, S])
_sig("dr_cuda_layer_norm_fwd", [P, i64, INT, P, P, f32, P, P, P, S])
_sig("dr_cuda_layer_norm_bwd", [P, P, i64, INT, P, P, P, P, P, P, S])
_sig("dr_cuda_l2_normalize_fwd", [P, i64, INT, f32, P, P, S])
_sig("dr_cuda_l2_normalize_bwd", [P, P, P, i64, INT, P, S])
_sig("dr_cuda_gelu_fwd", [P, i64, INT, P, S])
_sig("dr_cuda_gelu_bwd", [P, P, i64, INT, P, S])
_sig("dr_cuda_dice_fwd", [P, i64, INT, P, P, P, P, S])
# sparse utilities
_sig("dr_cuda_sparse_utils_workspace", [i64, i64], i64)
_sig("dr_cuda_sparse_prune_fill", [P, P, P, i64, i64, INT, INT, i64, P, P, P, P, P, P, S])
_sig("dr_cuda_sparse_slice", [P, P, INT, i64, INT, P, P, P, P, P, P, S])
_sig("dr_cuda_sparse_reshape", [P, i64, INT, P, INT, P, P, S])
_sig("dr_cuda_sparse_segment_fwd", [P, i64, INT, P, P, i64, i64, INT, P, S])
_sig("dr_cuda_sparse_segment_bwd", [P, i64, INT, P, P, i64, i64, INT, P, S])
# unique-first sparse pipeline (sparse_pipeline.cu)
_sig("dr_sp_init_scratch", [P, i64, S])
_sig("dr_sp_dedup", [P, GP, P, P, P, P, P, P, P, SP, S])
_sig("dr_sp_segsum", [P, P, GP, P, SP, S])
_sig("dr_sp_gather", [P, P, GP, P, SP, S])
_sig("dr_sp_gather_pitched", [P, P, GP, P, i64, SP, S])
_sig("dr_sp_pool", [P, P, GP, BP, P, P, SP, S])
_sig("dr_sp_pool_segsum", [P, P, P, GP, BP, P, SP, S])
_sig("dr_sp_linear_fwd", [P, P, GP, P, SP, S])
_sig("dr_sp_linear_bwd", [P, P, GP, P, SP, S])
_sig("dr_sp_lookup", [P, P, GP, i64, PP, PP, PP, PP, PP, INT, P, P, P, P, P, i64, SP, S])
_sig("dr_sp_grad", [P, P, GP, i64, PP, P, P, P, P, SP, S])
_sig("dr_sp_reset", [GP, i64, P, P, P, P, S])
_sig("dr_sp_signal", [SP, INT, S])
_sig("dr_sp_step_end", [P, S])
_sig("dr_sp_stats", [GP, P, P, S])
# all-gather embedding (ag_embedding.cu)
_sig("dr_ag_lookup", [P, AGP, APP, INT, P, P, P, P, P, i64, SP, S])
_sig("dr_ag_reduce", [AGP, APP, P, P, SP, S])
_sig("dr_ag_grad", [P, AGP, APP, P, P, P, P, i64, SP, S])
_sig("dr_ag_sizeof_geom", [])
# device, peer memory, NVLS (comm_kernels.cu, nvls.cu)
_sig("dr_cuda_set_device", [INT])
_sig("dr_cuda_get_device", [])
_sig("dr_cuda_set_sparse_blocks_per_sm", [INT])
_sig("dr_cuda_set_sparse_sms", [INT])
_sig("dr_cuda_sm_partition", [INT, INT, C.POINTER(INT), C.POINTER(vp)])
_sig("dr_cuda_graph_kernel_contexts", [P, C.POINTER(vp), INT])
_sig("dr_comm_alloc", [i64, C.POINTER(vp)])
_sig("dr_comm_free", [P])
_sig("dr_comm_get_handle", [P, P])
_sig("dr_comm_open_handle", [P, C.POINTER(vp)])
_sig("dr_comm_close_handle", [P])
_sig("dr_comm_can_access_peer", [INT, INT])
_sig("dr_comm_barrier", [PP, P, INT, INT, INT, S])
_sig("dr_comm_allreduce_apply", [PP, INT, P, P, P, i64, P, P, S])
_sig("dr_comm_allreduce_apply_sync", [PP, INT, P, P, P, i64, P, P, SP, S])
_sig("dr_nvls_supported", [INT])
_sig("dr_nvls_size", [i64, INT], i64)
_sig("dr_nvls_create", [i64, INT, INT, C.POINTER(vp), C.POINTER(INT)])
_sig("dr_nvls_import", [INT, i64, INT, INT, C.POINTER(vp)])
_sig("dr_nvls_add_device", [P])
_sig("dr_nvls_bind", [P, C.POINTER(vp), C.POINTER(vp)])
_sig("dr_nvls_allreduce_apply", [P, P, P, P, i64, P, P, P, S])
_sig("dr_nvls_allreduce_2phase", [P, P, INT, INT, P, P, P, i64, P, P, S])
# HBM / DRAM tier manager (tier_kernels.cu)
_sig("dr_tier_create", [vp, vp, vp, INT, i64, i64, INT], vp)
_sig("dr_tier_destroy", [vp], None)
_sig("dr_tier_prefetch", [vp, vp, vp, i64, i64, u32, S])
_sig("dr_tier_prefetch_mp", [vp, vp, vp, i64, i64, u32, vp, vp, INT, INT, S])
_sig("dr_tier_commit", [vp, vp, u32, S], i64)
_sig("dr_tier_evict", [vp, vp, i32, u32, i64, INT, S])
_sig("dr_tier_drain", [vp], None)
_sig("dr_tier_stats", [vp, vp], None)


def bind(lib, skip_missing: bool = False):
    """Declare every entry point on ``lib``.  ``skip_missing``: leave out the names ``lib`` does not export (the CUDA-on-CPU emulation
    build has no wgmma / NVLS / tensor-core GRU translation units); otherwise a missing name raises."""
    for name, (argtypes, restype) in SIGNATURES.items():
        if skip_missing and not hasattr(lib, name):
            continue
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = argtypes, restype
    assert lib.dr_ag_sizeof_geom() == C.sizeof(AgGeom)
    return lib
