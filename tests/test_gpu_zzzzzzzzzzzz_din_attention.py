"""DIN attention unit on csrc/cuda/din_att_kernels.cu (sm_90a): kernels against the float64 oracle of tests/din_attention_cases.py, exact
values, refusals, bitwise repeatability under graph replay, and the DIN / DIEN engines that train on it."""
import pytest
import torch

import din_attention_cases as A

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
SHAPES = [(D, H1, H2) for D in (16, 32, 64) for (H1, H2) in ((80, 40), (16, 8), (128, 64))]
LENS = (1, 15, 16, 17, 50, 64, 65, 128)


@pytest.mark.parametrize("D,H1,H2", SHAPES)
@pytest.mark.parametrize("mode", (0, 1))
def test_kernels_match_the_float64_oracle(D, H1, H2, mode):
    for i, L in enumerate(LENS):
        A.check_case(3, L, D, H1, H2, mode, seed=i, dev=DEV, k_dtype=torch.float32 if i % 3 == 2 else torch.bfloat16)
    A.check_case(1, 50, D, H1, H2, mode, seed=11, dev=DEV)


@pytest.mark.parametrize("mode", (0, 1))
@pytest.mark.parametrize("L", (50, 128))
def test_kernels_at_a_large_batch(mode, L):
    A.check_case(4099, L, 32, 80, 40, mode, seed=3, dev=DEV)


@pytest.mark.parametrize("mode", (0, 1))
def test_samples_without_a_valid_position_add_nothing(mode):
    A.empty_rows_add_nothing(DEV, mode)


def test_unsupported_shapes_return_minus_2_and_the_op_raises():
    from deeprec_b200.nn import fused_din_attention
    for (B, L, D, H1, H2) in ((2, 10, 24, 80, 40), (2, 10, 80, 80, 40), (2, 10, 32, 72, 40), (2, 10, 32, 144, 40), (2, 10, 32, 80, 36),
                              (2, 10, 32, 80, 72), (2, 129, 32, 80, 40)):
        c = A.make_case(B, L, D, H1, H2, 0, DEV)
        rc, _, _, _ = A.run_kernels(c, 0)
        assert rc == -2, (B, L, D, H1, H2, rc)
        att = torch.nn.Sequential(torch.nn.Linear(4 * D, H1), torch.nn.Sigmoid(), torch.nn.Linear(H1, H2), torch.nn.Sigmoid(),
                                  torch.nn.Linear(H2, 1)).to(DEV)
        with pytest.raises(ValueError, match="fused_din_attention"):
            fused_din_attention(c["q"], c["k"].float(), c["mask"], att)
    c = A.make_case(2, 10, 32, 80, 40, 0, DEV)
    from deeprec_b200 import _native
    from deeprec_b200._native import stream_ptr
    out = torch.empty(2, 32, device=DEV)
    W = [c[n].float().contiguous() for n in ("W1", "b1", "W2", "b2", "w3")]
    p = A._p
    for L, mode in ((0, 0), (10, 2)):           # no position; an unknown mode
        assert _native.cuda().dr_cuda_din_att_fwd(p(c["q"]), p(c["k"]), 1, p(c["mask"]), 2, L, 32, p(W[0]), p(W[1]), 80, p(W[2]), p(W[3]),
                                                  40, p(W[4]), mode, p(out), stream_ptr()) == -2


def test_kernels_are_bit_identical_across_runs_and_graph_replay():
    for mode in (0, 1):
        c = A.make_case(2048, 50, 32, 80, 40, 9, DEV)
        gout = A.make_gout(c, mode, 9)
        _, o1, _, g1 = A.run_kernels(c, mode, gout)
        _, o2, _, g2 = A.run_kernels(c, mode, gout)
        assert torch.equal(o1, o2)
        for n in g1:
            assert torch.equal(g1[n], g2[n]), n
        res = {}
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(graph, stream=s):
                _, res["o"], _, res["g"] = A.run_kernels(c, mode, gout)
        torch.cuda.current_stream().wait_stream(s)
        for _ in range(2):
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(res["o"], o1)
            for n in g1:
                assert torch.equal(res["g"][n], g1[n]), n


def test_op_matches_the_kernels_and_is_repeatable_and_capturable():
    from deeprec_b200.nn import fused_din_attention
    torch.manual_seed(0)
    B, L, D = 512, 50, 32
    att = torch.nn.Sequential(torch.nn.Linear(4 * D, 80), torch.nn.Sigmoid(), torch.nn.Linear(80, 40), torch.nn.Sigmoid(),
                              torch.nn.Linear(40, 1)).to(DEV)
    mask = A.make_mask(B, L, 1).to(DEV)
    q0 = torch.randn(B, D, device=DEV)
    k0 = torch.randn(B, L, D, device=DEV).to(torch.bfloat16)

    def run(weights):
        att.zero_grad(set_to_none=False)
        q, k = q0.clone().requires_grad_(), k0.clone().requires_grad_()
        out = fused_din_attention(q, k, mask, att, weights=weights)
        (out.float() * torch.linspace(-1, 1, out.shape[-1], device=DEV)).sum().backward()
        return [out.detach().clone(), q.grad.clone(), k.grad.clone()] + [p.grad.clone() for p in att.parameters()]

    for weights in (False, True):
        for p in att.parameters():
            p.grad = torch.zeros_like(p)
        r1, r2 = run(weights), run(weights)
        assert r1[0].dtype == (torch.float32 if weights else q0.dtype)
        assert r1[2].dtype == torch.bfloat16
        for a, b in zip(r1, r2):
            assert torch.equal(a, b)
        assert float(att[4].bias.grad[0]) == 0.0
        assert bool((r1[2][~mask] == 0).all())
        # the oracle on the same inputs
        c = {"q": q0, "k": k0, "mask": mask, "W1": att[0].weight.detach(), "b1": att[0].bias.detach(), "W2": att[2].weight.detach(),
             "b2": att[2].bias.detach(), "w3": att[4].weight.detach().view(-1)}
        gout = torch.linspace(-1, 1, r1[0].shape[-1], device=DEV).expand_as(r1[0])
        ref = A.oracle(c, int(weights), gout)
        A.close(r1[0], ref["out"], "out")
        A.close(r1[1], ref["dq"], "dq")
        A.close(r1[2], ref["dk"], "dk")
        A.close(r1[3], ref["dW1"], "dW1")
        A.close(r1[5], ref["dW2"], "dW2")


@pytest.mark.parametrize("name", ("din", "dien"))
@pytest.mark.parametrize("graph", (False, True))
def test_engine_matches_a_torch_replica(name, graph):
    A.run_vs_replica(name, DEV, graph=graph)


@pytest.mark.parametrize("name", ("din", "dien"))
def test_engine_training_is_bit_identical_across_engines_and_graph_replay(name):
    p1, l1, t1 = A.train(name, DEV, graph=False)
    p2, l2, t2 = A.train(name, DEV, graph=False)
    assert torch.equal(p1, p2) and l1 == l2
    for a, b in zip(t1, t2):
        assert torch.equal(a, b)
    p3, l3, t3 = A.train(name, DEV, graph=True)
    assert torch.equal(p1, p3) and l1 == l3
    for a, b in zip(t1, t3):
        assert torch.equal(a, b)
