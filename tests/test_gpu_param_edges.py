"""The generic kernel's per-synapse tensor (SYN) and per-neuron parameter (PN) instantiations on the H100, at the
shapes where their paths switch (cases, float64 restatements and path mirrors: tests/param_edges.py).  Every case runs
on tier 1 (the single-operator cases through conn_update_kernel<true>), is bit-identical to the CPU oracle on the whole
state and within the rounding-error bound of the float64 restatement."""
import pytest
import torch

import cases
import param_edges as pe
from test_kernel_edges import _with
from test_param_edges import _oracle, assert_same_state, check_pn_against_float64, check_syn_against_float64

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")

GPU_SYN_CASES = [c.at_gpu_size() for c in pe.SYN_CASES]
GPU_PN_CASES = [c.at_gpu_size() for c in pe.PN_CASES]


@pytest.mark.parametrize("case", GPU_SYN_CASES, ids=lambda c: c.name)
def test_gpu_syn_bit_exact_and_within_float64_bound(case):
    from bindsnet_b200 import _backend

    d = pe.draw_syn(case)
    a, net = pe.run_syn(B200, case, d, device="cuda")
    torch.cuda.synchronize()
    if not case.op:
        net.check_errors()
        assert _backend.last_tier == 1
    b, onet = _with(_oracle(), lambda: pe.run_syn(B200, case, d))
    assert_same_state(a, b, case.name)
    check_syn_against_float64(case, d, a, onet)


@pytest.mark.parametrize("case", GPU_PN_CASES, ids=lambda c: c.name)
def test_gpu_pn_bit_exact_and_within_float64_bound(case):
    from bindsnet_b200 import _backend

    d = pe.draw_pn(case)
    a, net = pe.run_pn(B200, case, d, device="cuda")
    net.check_errors()
    assert _backend.last_tier == 1
    b, onet = _with(_oracle(), lambda: pe.run_pn(B200, case, d))
    for k in range(case.windows):
        assert_same_state(a[k], b[k], f"{case.name} window {k}")
    check_pn_against_float64(case, d, a, onet.layers["P"])
