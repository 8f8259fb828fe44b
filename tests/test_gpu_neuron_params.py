"""Per-neuron parameter tensors of LIFNodes, AdaptiveLIFNodes and DiehlAndCookNodes on the H100: the CUDA library's generic
window bit for bit against the oracle (tests/neuron_param_oracle.c), plus a DiehlAndCook2015-shaped network (n = 1600,
B = 128, T = 250) with per-neuron thresholds and theta increments and a recurrent E/I network at N = 4000, B = 128."""
import pytest
import torch

import cases
import helpers
import neuron_param_nets as pn
import synapse_nets as sn

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _gpu_vs_oracle(build, windows=2, **run_kw):
    from bindsnet_b200 import _backend
    from neuron_param_oracle import NeuronParamOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = build()
        torch.manual_seed(5)   # (the one_spike tie-break seed Network.run draws)
        if gpu:
            sn.to_device(net, "cuda")   # (and a rule's rate tensors, which Network.to leaves where they are)
            inputs = {k: v.cuda() for k, v in inputs.items()}
            for k in range(windows):
                net.run(inputs=pn.window_inputs(inputs, T, k), time=T, **run_kw)
            net.check_errors()
            assert _backend.last_tier == 1
        else:
            with NeuronParamOracleBackend() as ob:
                for k in range(windows):
                    net.run(inputs=pn.window_inputs(inputs, T, k), time=T, **run_kw)
            assert ob.err == 0
        outs.append(pn.snapshot(net))
    return outs


@pytest.mark.parametrize("case", pn.LIVE_CASES)
def test_gpu_cases_bit_exact(case):
    a, b = _gpu_vs_oracle(lambda: pn.live_net(B200, case, T=20))
    helpers.assert_bit_identical(a, b, case)
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("mode", ["one_step", "stepwise"])
@pytest.mark.parametrize("case", ["lif_b1", "dc", "traces"])
def test_gpu_one_step_and_stepwise_bit_exact(case, mode):
    def build():
        net, inputs, T = pn.live_net(B200, case, T=9)
        if mode == "stepwise":
            net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["s", "refrac_count"], time=T), "Yr")
        return net, inputs, T
    a, b = _gpu_vs_oracle(build, one_step=mode == "one_step")
    helpers.assert_bit_identical(a, b, f"{case} {mode}")


def _dc2015(n, B, T, **kw):
    net, x = pn.dc2015_like(B200, n, B, T, **kw)
    net.add_monitor(B200.monitors.Monitor(net.layers["Ae"], ["s"], time=T), "Ys")
    return net, {"X": x}, T


def test_gpu_dc2015_shape():
    """n = 1600, B = 128, one_spike, per-neuron thresholds and theta increments: a 10-step window bit for bit against the
    oracle, then T = 250 on the device (tier 1, the adaptive thresholds grow with each neuron's own increment)."""
    from bindsnet_b200 import _backend

    a, b = _gpu_vs_oracle(lambda: _dc2015(1600, 128, 10, seed=3), windows=1)
    helpers.assert_bit_identical(a, b, "DiehlAndCook2015-shaped, n = 1600, B = 128, T = 10")
    net, x = pn.dc2015_like(B200, 1600, 128, 250, seed=3, device="cuda")
    E = net.layers["Ae"]
    net.run(inputs={"X": x}, time=250)
    net.check_errors()
    assert _backend.last_tier == 1
    assert int(E.s.sum()) >= 0 and float(E.theta.sum()) > 0
    spiked = E.theta > 0   # theta ~ theta_plus[j] * (spikes of j), decayed by tc_theta_decay = 1e7
    ratio = (E.theta[spiked] / E.theta_plus[spiked])
    assert torch.allclose(ratio, ratio.round(), rtol=1e-4, atol=0.0)


@pytest.mark.parametrize("n,B,T", [(4000, 128, 250)])
def test_gpu_ei_large_constant_tensors_equal_scalars(n, B, T):
    """A recurrent E/I network (per-row sign bounds: SYN) whose LIF population's thresh, rest and tc_decay are tensors
    holding its scalars (PN), N = 4000, B = 128, T = 250: bit for bit the scalar population's run, on tier 1."""
    from bindsnet_b200 import _backend

    outs = []
    for tensors in (True, False):
        net, x = sn.ei_network(B200, n, B, T, seed=7, device="cuda")
        Y = net.layers["Y"]
        if tensors:
            Y.thresh = torch.full((n,), float(Y.thresh), device="cuda")
            Y.rest = torch.full((n,), float(Y.rest), device="cuda")
            Y.tc_decay = torch.full((n,), float(Y.tc_decay), device="cuda")
            Y.compute_decays(1.0)
        net.run(inputs={"X": x}, time=T)
        net.check_errors()
        assert _backend.last_tier == 1
        outs.append(sn.snapshot(net))
    helpers.assert_bit_identical(outs[0], outs[1], "E/I N = 4000, B = 128")
    assert outs[0]["L/Y/s"].sum() >= 0


def test_gpu_ei_heterogeneous_bit_exact():
    """The E/I network (SYN + PN) with heterogeneous neurons, N = 300, B = 16, against the oracle."""
    def build():
        T = 40
        net, x = sn.ei_network(B200, 300, 16, T, seed=7, n_in=200)
        Y = net.layers["Y"]
        g = torch.Generator().manual_seed(9)
        Y.thresh = -54.0 + 4.0 * torch.rand(300, generator=g)
        Y.rest = -66.0 + 2.0 * torch.rand(300, generator=g)
        Y.tc_decay = 60.0 + 80.0 * torch.rand(300, generator=g)
        Y.compute_decays(1.0)
        net.add_monitor(B200.monitors.Monitor(Y, ["s"], time=T), "Ys")
        return net, {"X": (torch.rand(2 * T, 16, 200, generator=g) < 0.1).to(torch.uint8)}, T
    a, b = _gpu_vs_oracle(build)
    helpers.assert_bit_identical(a, b, "E/I heterogeneous")
    assert a["M/Ys"].sum() > 0
