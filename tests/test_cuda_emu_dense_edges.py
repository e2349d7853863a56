"""The dense-path kernels of the DLRM step on the CUDA-on-CPU emulation against the float64 oracle (tests/dense_ref.py): column statistics,
BatchNorm forward (finalize / fold, training and eval) and backward, the dW fix-up, the logit head, weight packing and input cast, and one
DLRMEngine step checked stage by stage with its BatchNorm state and predict().  The same cases (tests/dense_cases.py) run on an H100 in
tests/test_gpu_dense_edges.py.  The emulation has num_sms() == 2, so its grids differ from the H100's; every bound holds for any grid."""
import os

import pytest

import dense_cases as K
from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(1500)]
QUICK = os.environ.get("DEEPREC_EMU_QUICK") == "1"

COLSTATS = [(N, B) for N in ([8, 40, 512] if QUICK else K.COLSTATS_N) for B in K.colstats_batches(N, big=N <= 16)]
BN_BWD = [(N, B) for N in ([24, 512] if QUICK else K.COLSTATS_N) for B in K.bn_bwd_batches(N, big=False) if N * B <= 1 << 21]


@pytest.mark.parametrize("N,B", COLSTATS)
def test_colstats(N, B):
    with _native.cuda_emulation():
        K.colstats_case("cpu", N, B)


def test_colstats_and_bn_bwd_apply_v2_reject_bad_widths():
    with _native.cuda_emulation():
        K.colstats_rejects_case("cpu")


@pytest.mark.parametrize("kind,K_,B,Nn,Kp", [("finalize", 16, 1000, 1, None), ("finalize", 1024, 333, 1, None), ("fold", 5, 1000, 1, 8),
                                             ("fold", 16, 4097, 16, 16), ("fold", 260, 999, 1024, 264)])
def test_bn_forward(kind, K_, B, Nn, Kp):
    with _native.cuda_emulation():
        K.bn_forward_case("cpu", kind, K_, B, Nn, Kp)


@pytest.mark.parametrize("N,B", [(8, 1), (24, 7), (512, 4097)])
def test_bn_apply(N, B):
    with _native.cuda_emulation():
        K.bn_apply_case("cpu", N, B)


@pytest.mark.parametrize("N,B,gas", [(16, 1000, 1.0), (1000, 77, 0.5)])
def test_bn_bwd_finalize(N, B, gas):
    with _native.cuda_emulation():
        K.bn_bwd_finalize_case("cpu", N, B, gas)


@pytest.mark.parametrize("N,B", BN_BWD)
@pytest.mark.parametrize("version,relu_mask,dbias", [(1, 1, False), (2, 1, True), (2, 0, True), (2, 1, False)])
def test_bn_bwd_apply(N, B, version, relu_mask, dbias):
    with _native.cuda_emulation():
        K.bn_bwd_apply_case("cpu", N, B, version, relu_mask, dbias)


@pytest.mark.parametrize("N,K_,Kp", [(1, 5, 8), (16, 9, 16), (300, 517, 520)])
def test_dw_fixup(N, K_, Kp):
    with _native.cuda_emulation():
        K.dw_fixup_case("cpu", N, K_, Kp)


@pytest.mark.parametrize("variant", ["train", "scaled", "saturated", "eval"])
@pytest.mark.parametrize("B", K.HEAD_B)
@pytest.mark.parametrize("K_", K.HEAD_K)
def test_head(K_, B, variant):
    with _native.cuda_emulation():
        K.head_case("cpu", K_, B, variant)


def test_head_rejects_width_128():
    with _native.cuda_emulation():
        K.head_rejects_case("cpu")


@pytest.mark.parametrize("N,Kp", K.PACK_SHAPES)
@pytest.mark.parametrize("ldt_pad,with_t", [(0, True), (21, True), (0, False)])
def test_pack_weights_bit_exact(N, Kp, ldt_pad, with_t):
    with _native.cuda_emulation():
        K.pack_weights_case("cpu", N, Kp, ldt_pad, with_t)


@pytest.mark.parametrize("B,C_,Cp", K.CAST_SHAPES)
def test_cast_pad_bit_exact(B, C_, Cp):
    with _native.cuda_emulation():
        K.cast_pad_case("cpu", B, C_, Cp)


@pytest.mark.parametrize("over", [{}, {"gemm_v1": True}], ids=["default", "gemm_v1"])
def test_dlrm_step_stage_by_stage(over):
    with _native.cuda_emulation():
        K.engine_step_case("cpu", 256, **over)


def test_dlrm_step_rejects_unsupported_head_width():
    with _native.cuda_emulation():
        K.engine_bad_head_width_case("cpu")
