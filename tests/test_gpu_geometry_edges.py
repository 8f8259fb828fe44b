"""The generic kernel's Conv1dConnection, Conv3dConnection and LocalConnection3D paths (gathers and their staging, the
learning and normalize phases) and their single-operator kernels on the H100, at the shapes where their paths switch
(cases, float64 restatements and path mirrors: tests/geometry_edges.py).  Every case runs on tier 1, is bit-identical
to the kind's CPU oracle and within the rounding-error bound of the float64 restatement."""
import pytest
import torch

import cases
import geometry_edges as ge
from test_geometry_edges import check_against_float64, check_op_against_float64, oracle_for
from test_kernel_edges import _with

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")

GPU_WINDOW_CASES = [c.at_gpu_size() for c in ge.WINDOW_CASES]
GPU_GATHER_CASES = [c.at_gpu_size() for c in ge.GATHER_CASES]
GPU_OP_CASES = [c.at_gpu_size() for c in ge.OP_CASES]


@pytest.mark.parametrize("case", GPU_WINDOW_CASES, ids=lambda c: c.name)
def test_gpu_window_bit_exact_and_within_float64_bound(case):
    from bindsnet_b200 import _backend

    d = ge.draw_window(case)
    a, net = ge.run_window(B200, case, d, device="cuda")
    net.check_errors()
    assert _backend.last_tier == 1
    b, onet = _with(oracle_for(case.kind), lambda: ge.run_window(B200, case, d))
    for k in b:
        ge.assert_same(a[k], b[k], f"{case.name} {k}")
    check_against_float64(case, d, a, onet)


@pytest.mark.parametrize("case", GPU_GATHER_CASES, ids=lambda c: c.name)
def test_gpu_gather_bit_exact_and_within_float64_bound(case):
    from bindsnet_b200 import _backend

    d = ge.draw_gather(case)
    a = ge.run_gather(B200, case, d, device="cuda")
    torch.cuda.synchronize()
    assert _backend.last_tier == 1
    b = _with(oracle_for(case.kind), lambda: ge.run_gather(B200, case, d))
    ge.assert_same(a, b, case.name)
    v64, bound = ge.ref_gather(case, d)
    ge.assert_within_bound(a, v64, bound, case.name)


@pytest.mark.parametrize("case", GPU_OP_CASES, ids=lambda c: c.name)
def test_gpu_single_operators_bit_exact_and_within_float64_bound(case):
    d = ge.draw_op(case)
    a, w_in = ge.run_op(B200, case, d, device="cuda")
    torch.cuda.synchronize()
    b, _ = _with(oracle_for(case.kind), lambda: ge.run_op(B200, case, d))
    for k in b:
        ge.assert_same(a[k], b[k], f"{case.name} {k}")
    check_op_against_float64(case, d, a, w_in)
