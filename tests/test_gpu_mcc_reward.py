"""MCC_learning.MSTDP / MSTDPET on the H100: the CUDA library's generic window bit for bit against the oracle
(tests/mcc_reward_oracle.c), the equivalence with learning.MSTDP / MSTDPET on a dense Connection, and a reservoir readout
at the benchmark's shape (N = 4000, B = 128, T = 50)."""
import pytest
import torch

import cases
import helpers
import mcc_reward_nets as rn
from test_mcc_reward import _readout_state

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _gpu_vs_oracle(case, one_step=False, stepwise=False, T=20):
    from bindsnet_b200 import _backend
    from mcc_reward_oracle import RewardOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = rn.live_net(B200, case, T=T)
        net.force_tier = 1
        if stepwise:
            net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["s", "refrac_count"], time=T), "Yr")
        if gpu:
            net.to("cuda")
            rn.run_two_windows(net, {k: v.cuda() for k, v in inputs.items()}, T, case, one_step=one_step)
            net.check_errors()
            assert _backend.last_tier == 1
        else:
            with RewardOracleBackend() as ob:
                rn.run_two_windows(net, inputs, T, case, one_step=one_step)
            assert ob.err == 0
        outs.append(rn.full_snapshot(net, T))
    return outs


@pytest.mark.parametrize("case", rn.LIVE_CASES)
def test_gpu_live_cases_bit_exact(case):
    a, b = _gpu_vs_oracle(case)
    helpers.assert_bit_identical(a, b, case)
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("mode", ["one_step", "stepwise"])
@pytest.mark.parametrize("case", ["w_b1", "pw_b4", "decay_range_et"])
def test_gpu_one_step_and_stepwise_bit_exact(case, mode):
    a, b = _gpu_vs_oracle(case, one_step=mode == "one_step", stepwise=mode == "stepwise", T=10)
    helpers.assert_bit_identical(a, b, f"{case} {mode}")


def _run_pair(rule, B, T, n_res, n_in):
    outs = []
    for mcc in (True, False):
        net, x = rn.reservoir_readout(B200, rule, B, T, n_res=n_res, n_in=n_in, mcc=mcc, seed=3, device="cuda")
        net.to("cuda")
        x = x.cuda()
        for k in range(2):
            net.run(inputs={"X": x}, time=T, one_spike_seed=7 + k, **rn.WINDOW_KWARGS[k])
        net.check_errors()
        outs.append(_readout_state(net))
    return outs


@pytest.mark.parametrize("rule,B", [("MSTDP", 1), ("MSTDP", 32), ("MSTDPET", 1)])
def test_gpu_mcc_rule_equals_dense_rule(rule, B):
    a, b = _run_pair(rule, B, 20, 300, 100)
    helpers.assert_bit_identical(a, b, f"MCC {rule} vs dense {rule}, B = {B}")
    assert a["O/s"].sum() + a["R/s"].sum() > 0


def test_gpu_reservoir_readout_at_bench_shape():
    """N = 4000, B = 128, T = 50: the MCC readout equals the dense one bit for bit, learns, and the window runs on tier 1."""
    from bindsnet_b200 import _backend

    a, b = _run_pair("MSTDP", 128, 50, 4000, 784)
    assert _backend.last_tier == 1
    helpers.assert_bit_identical(a, b, "MCC MSTDP vs dense MSTDP at N = 4000, B = 128")
    w0 = rn.reservoir_readout(B200, "MSTDP", 128, 1, seed=3)[0].connections[("R", "O")].w
    assert not torch.equal(torch.from_numpy(a["w"]), w0)
