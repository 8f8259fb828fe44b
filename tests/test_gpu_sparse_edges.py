"""The generic kernel's sparse instantiation and the sparse single operators on the H100, at the shapes where their paths
switch (cases, float64 restatements and path mirrors: tests/sparse_edges.py).  Every window case runs on tier 1 and is
bit-identical to the CPU oracle on the whole state and within the rounding-error bound of the float64 restatement; so
are connection.compute and connection.update; and every bias the reference broadcasts gives the explicit bias' bits."""
import pytest
import torch

import cases
import geometry_edges as ge
import sparse_edges as se
from test_kernel_edges import _with
from test_sparse_edges import (BAD_BIASES, _bias_net, _biases, _oracle, assert_same_state, check_against_float64, check_bites,
                               check_op_against_float64)

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")

GPU_CASES = [c.at_gpu_size() for c in se.CASES]


@pytest.mark.parametrize("case", GPU_CASES, ids=lambda c: c.name)
def test_gpu_window_bit_exact_and_within_float64_bound(case):
    from bindsnet_b200 import _backend

    d = se.draw(case)
    a, net = se.run(B200, case, d, device="cuda")
    torch.cuda.synchronize()
    net.check_errors()
    assert _backend.last_tier == 1
    b, _ = _with(_oracle(), lambda: se.run(B200, case, d))
    for k in range(case.windows):
        assert_same_state(a[k], b[k], f"{case.name} window {k}")
    check_against_float64(case, d, a)
    check_bites(case, d, a)
    se.check_claims(case, se.paths(case, d))


@pytest.mark.parametrize("case", se.OP_CASES, ids=lambda c: c.name)
def test_gpu_op_bit_exact_and_within_float64_bound(case):
    d = se.draw_op(case)
    a = se.run_op(B200, case, d, device="cuda")
    torch.cuda.synchronize()
    b = _with(_oracle(), lambda: se.run_op(B200, case, d))
    for k in b:
        ge.assert_same(a[k], b[k], f"{case.name} {k}")
    check_op_against_float64(case, d, a)


@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
@pytest.mark.parametrize("form", list(_biases()))
def test_gpu_bias_forms_equal_the_explicit_bias(form, sparse):
    b, full = _biases()[form]
    outs = []
    for bias in (b, full):
        net, x = _bias_net(sparse, bias)
        net.to("cuda")
        x = x.cuda()
        net.run(inputs={"X": x}, time=5)
        out = net.connections[("X", "Y")].compute(x[0].bool())
        torch.cuda.synchronize()
        net.check_errors()
        outs.append((net.layers["Y"].v.cpu(), out.cpu()))
    for a, e in zip(*outs):
        assert torch.equal(a.view(torch.int32), e.view(torch.int32)), form


@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
@pytest.mark.parametrize("bad", list(BAD_BIASES))
def test_gpu_bad_bias_is_refused_before_anything_runs(bad, sparse):
    make, exc = BAD_BIASES[bad]
    net, x = _bias_net(sparse, torch.zeros(48))
    conn = net.connections[("X", "Y")]
    conn.b = torch.nn.Parameter(make(), requires_grad=False)
    net.to("cuda")
    x = x.cuda()
    v0 = net.layers["Y"].v.clone()
    with pytest.raises(exc):
        net.run(inputs={"X": x}, time=5)
    with pytest.raises(exc):
        conn.compute(x[0].bool())
    assert torch.equal(net.layers["Y"].v, v0), f"{bad}: the window ran"
