"""The dense-path kernels of the DLRM step (csrc/cuda/dense_kernels.cu) on an H100 against the float64 oracle (tests/dense_ref.py): column
statistics, BatchNorm forward (finalize / fold, training and eval) and backward, the dW fix-up, the logit head, weight packing and input
cast, and one DLRMEngine step checked stage by stage with its BatchNorm state and predict().  The same cases (tests/dense_cases.py) run on
the CUDA-on-CPU emulation in tests/test_cuda_emu_dense_edges.py."""
import pytest

import dense_cases as K

pytestmark = pytest.mark.gpu

COLSTATS = [(N, B) for N in K.COLSTATS_N for B in K.colstats_batches(N)]
BN_BWD = [(N, B) for N in K.COLSTATS_N for B in K.bn_bwd_batches(N)]


@pytest.mark.parametrize("N,B", COLSTATS)
def test_colstats(N, B):
    K.colstats_case("cuda", N, B)


def test_colstats_and_bn_bwd_apply_v2_reject_bad_widths():
    K.colstats_rejects_case("cuda")


@pytest.mark.parametrize("kind,K_,B,Nn,Kp", [("finalize", 16, 1000, 1, None), ("finalize", 64, 4097, 1, None), ("finalize", 1024, 333, 1, None),
                                             ("fold", 5, 1000, 1, 8), ("fold", 16, 4097, 16, 16), ("fold", 260, 999, 1024, 264),
                                             ("fold", 512, 65537, 256, 512)])
def test_bn_forward(kind, K_, B, Nn, Kp):
    K.bn_forward_case("cuda", kind, K_, B, Nn, Kp)


@pytest.mark.parametrize("N,B", [(8, 1), (24, 7), (512, 4097), (2048, 1001), (16, 65537)])
def test_bn_apply(N, B):
    K.bn_apply_case("cuda", N, B)


@pytest.mark.parametrize("N,B,gas", [(16, 1000, 1.0), (1000, 77, 0.5), (512, 4096, 0.25)])
def test_bn_bwd_finalize(N, B, gas):
    K.bn_bwd_finalize_case("cuda", N, B, gas)


@pytest.mark.parametrize("N,B", BN_BWD)
@pytest.mark.parametrize("version,relu_mask,dbias", [(1, 1, False), (1, 0, False), (2, 1, True), (2, 0, True), (2, 1, False)])
def test_bn_bwd_apply(N, B, version, relu_mask, dbias):
    K.bn_bwd_apply_case("cuda", N, B, version, relu_mask, dbias)


@pytest.mark.parametrize("N,K_,Kp", [(1, 5, 8), (16, 9, 16), (1024, 517, 520)])
def test_dw_fixup(N, K_, Kp):
    K.dw_fixup_case("cuda", N, K_, Kp)


@pytest.mark.parametrize("variant", ["train", "scaled", "saturated", "eval"])
@pytest.mark.parametrize("B", K.HEAD_B)
@pytest.mark.parametrize("K_", K.HEAD_K)
def test_head(K_, B, variant):
    K.head_case("cuda", K_, B, variant)


def test_head_rejects_width_128():
    K.head_rejects_case("cuda")


@pytest.mark.parametrize("N,Kp", K.PACK_SHAPES)
@pytest.mark.parametrize("ldt_pad,with_t", [(0, True), (21, True), (0, False)])
def test_pack_weights_bit_exact(N, Kp, ldt_pad, with_t):
    K.pack_weights_case("cuda", N, Kp, ldt_pad, with_t)


@pytest.mark.parametrize("B,C_,Cp", K.CAST_SHAPES)
def test_cast_pad_bit_exact(B, C_, Cp):
    K.cast_pad_case("cuda", B, C_, Cp)


@pytest.mark.parametrize("B,over", [(1000, {}), (4096, {}), (1000, {"gemm_v1": True}), (1000, {"mlp_bot": (1024, 64, 16)}),
                                    (1000, {"mlp_top": (1024, 512)}), (1000, {"mlp_top": (512, 1024)})],
                         ids=["default-B1000", "default-B4096", "gemm_v1", "bot-1024-64-16", "top-512", "top-1024"])
def test_dlrm_step_stage_by_stage(B, over):
    K.engine_step_case("cuda", B, **over)


def test_dlrm_step_rejects_unsupported_head_width():
    K.engine_bad_head_width_case("cuda")
