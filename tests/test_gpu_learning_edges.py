"""The generic kernel's in-window learning paths (dense MSTDP / MSTDPET and their MulticompartmentConnection forms, the
rules of a Conv2dConnection and of a LocalConnection2D) and phase 1's convolutional and local gathers on the H100, at
the shapes where their paths switch and at full size where the CPU tier shrinks them (cases, float64 restatements and
path mirrors: tests/learning_edges.py).  Every case runs on tier 1, is bit-identical to the CPU oracle and within the
rounding-error bound of the float64 restatement."""
import pytest
import torch

import cases
import learning_edges as le
from test_kernel_edges import _assert_bit_identical, _assert_within_bound, _with
from test_learning_edges import check_against_float64, oracle_for

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")

GPU_WINDOW_CASES = [c.at_gpu_size() for c in le.WINDOW_CASES]
GPU_GATHER_CASES = [c.at_gpu_size() for c in le.GATHER_CASES]


@pytest.mark.parametrize("case", GPU_WINDOW_CASES, ids=lambda c: c.name)
def test_gpu_window_bit_exact_and_within_float64_bound(case):
    from bindsnet_b200 import _backend

    d = le.draw_window(case)
    a, net = le.run_window(B200, case, d, device="cuda")
    net.check_errors()
    assert _backend.last_tier == 1
    b, onet = _with(oracle_for(case.kind, case.rule), lambda: le.run_window(B200, case, d))
    assert a.keys() == b.keys()
    for k in a:
        _assert_bit_identical(a[k].float(), b[k].float(), f"{case.name} {k}")
    check_against_float64(case, d, a, onet)


@pytest.mark.parametrize("case", [c for c in GPU_WINDOW_CASES if c.reward_rule and c.B <= 128][:4], ids=lambda c: c.name)
def test_gpu_rule_state_across_windows_of_odd_and_even_length(case):
    from bindsnet_b200 import _backend

    case = le.replace(case, T=5)
    d = le.draw_window(case)
    a, net = le.run_window(B200, case, d, device="cuda", spans=[3, 2])
    net.check_errors()
    assert _backend.last_tier == 1
    b, _ = _with(oracle_for(case.kind, case.rule), lambda: le.run_window(B200, case, d))
    for k in a:
        _assert_bit_identical(a[k].float(), b[k].float(), f"{case.name} {k}")


@pytest.mark.parametrize("case", GPU_GATHER_CASES, ids=lambda c: c.name)
def test_gpu_gather_bit_exact_and_within_float64_bound(case):
    from bindsnet_b200 import _backend

    d = le.draw_gather(case)
    a = le.run_gather(B200, case, d, device="cuda")
    torch.cuda.synchronize()
    assert _backend.last_tier == 1
    b = _with(oracle_for(case.kind), lambda: le.run_gather(B200, case, d))
    _assert_bit_identical(a, b, case.name)
    v64, bound = le.ref_gather(B200, case, d)
    _assert_within_bound(a, v64, bound, case.name)
