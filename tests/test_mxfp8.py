"""MXFP8 format helpers (ops/mxfp8.py): the torch model of the block-scaled quantiser pins the number format (E4M3 elements, UE8M0 scale per
32 along K, smallest power of two that keeps the block inside +-448) and the scale-word layout."""
import torch

from deeprec_b200.ops import mxfp8


def test_round_trip_error_and_scale_minimality():
    torch.manual_seed(0)
    x = torch.randn(300, 200) * torch.logspace(-6, 4, 300).unsqueeze(1)          # rows of very different magnitude
    x[5] = 0
    x[7, :40] = 0
    q, sf = mxfp8.quantize_mxfp8_reference(x)
    assert q.shape == (300, 256) and q.dtype == torch.uint8 and sf.numel() == mxfp8.sf_words(300, 256) == 3 * 2 * 128
    d = mxfp8.dequantize_mxfp8(q, sf)
    assert torch.equal(d[:, 200:], torch.zeros(300, 56))
    xb = torch.zeros(300, 256); xb[:, :200] = x
    amax = xb.reshape(300, 8, 32).abs().amax(2, keepdim=True)
    err = (d - xb).reshape(300, 8, 32).abs()
    assert (err <= amax * 2 ** -4 + 1e-37).all()                                  # 3 mantissa bits: half an ulp of the block maximum's binade
    e = mxfp8.block_exponents(xb)
    qmax = q.view(torch.float8_e4m3fn).float().abs().reshape(300, 8, 32).amax(2)
    nz = amax.squeeze(2) > 2.0 ** -100
    assert (qmax[nz] <= 448).all() and (qmax[nz] > 208).all()                     # the scale is the smallest admissible power of two
    assert (e[~(amax.squeeze(2) > 0)] == -126).all()


def test_scale_word_layout_is_the_tcgen05_cp_order():
    R, Kp = 256, 384
    idx = mxfp8._sf_index(R, Kp // 128, "cpu")
    assert sorted(idx.reshape(-1).tolist()) == list(range(mxfp8.sf_words(R, Kp)))          # a bijection when R is a multiple of 128
    assert idx[0, 0] == 0 and idx[1, 0] == 4 and idx[32, 0] == 1 and idx[127, 0] == 31 * 4 + 3
    assert idx[0, 1] == 128 and idx[128, 0] == 3 * 128 and idx[129, 2] == (3 + 2) * 128 + 4
    x = torch.zeros(R, Kp)
    x[33, 128 + 64] = 3.0            # row 33, k block 1, sub-block 2
    q, sf = mxfp8.quantize_mxfp8_reference(x)
    w = int(sf[(0 * 3 + 1) * 128 + (33 % 32) * 4 + 33 // 32]) & 0xFFFFFFFF
    assert [(w >> (8 * j)) & 0xFF for j in range(4)] == [1, 1, 127 - 7, 1]                   # 3 / 2^-7 = 384 <= 448 < 768
    assert q.view(torch.float8_e4m3fn).float()[33, 192] == 384.0


def test_mxfp8_linear_host_path_tracks_fp32():
    torch.manual_seed(1)
    lin = torch.nn.Linear(100, 37)
    x = torch.randn(64, 100)
    layer = mxfp8.MXFP8Linear(lin, relu=True)
    assert layer.wq.shape == (40, 128)
    y = layer(x).float()
    ref = lin(x).relu()
    assert y.shape == ref.shape and (y - ref).abs().max() / ref.abs().max() < 4e-2


def test_graph_optimizer_rewrites_eval_mlp_to_mxfp8():
    from deeprec_b200 import graph_optimizer as go
    torch.manual_seed(2)
    net = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 32), torch.nn.ReLU(), torch.nn.Linear(32, 1)).eval()
    x = torch.randn(50, 64)
    ref, ref_h = net(x), net[:4](x)
    rep = go.optimize(net, go.OptimizerOptions(mxfp8_inference=True))
    assert rep.count("LinearToMXFP8") == 2 and type(net[-1]) is torch.nn.Linear           # the 1-wide logit layer stays a plain Linear
    assert [type(m).__name__ for m in net] == ["MXFP8Linear", "MXFP8Linear", "Linear"]
    out = net(x)
    h = net[:2](x)
    assert (h - ref_h).abs().max() / ref_h.abs().max() < 6e-2                              # two fp8 layers
    assert (out - ref).abs().max() / ref.abs().max() < 0.2                                # the logit is a cancelling sum of those activations
    net2 = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU())                 # training mode: untouched by the inference rewrite
    assert go.optimize(net2, go.OptimizerOptions(mxfp8_inference=True)).count("LinearToMXFP8") == 0
