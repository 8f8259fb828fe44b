"""Weight(norm_frequency='time step') and per-target norm tensors on the H100: the CUDA library's generic window bit
for bit against the oracle (tests/weight_norm_oracle.c) on the CPU cases, the standalone normalisation, and the
DiehlAndCook2015 shape (Input(784) -> 1600 with inhibition, a 'time step' input Weight with norm 78.4, PostPre) at
B = 128, T = 250."""
import pytest
import torch

import cases
import helpers
import weight_norm_nets as wn

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _gpu_vs_oracle(case, one_step=False, **kw):
    from bindsnet_b200 import _backend
    from weight_norm_oracle import WeightNormOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T, run_kw = wn.build(B200, case, **kw)
        net.force_tier = 1
        if gpu:
            net.to("cuda")
            wn.run_windows(net, {k: v.cuda() for k, v in inputs.items()}, T, run_kw, one_step=one_step)
            net.check_errors()
            if not kw.get("custom"):
                assert _backend.last_tier == 1
        else:
            with WeightNormOracleBackend() as ob:
                wn.run_windows(net, inputs, T, run_kw, one_step=one_step)
            assert ob.err == 0
        outs.append(wn.full_snapshot(net, T))
    return outs


@pytest.mark.parametrize("case", wn.CASES)
def test_gpu_cases_bit_exact(case):
    a, b = _gpu_vs_oracle(case)
    helpers.assert_bit_identical(a, b, case)
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("case", ["ts_pp1", "tt_noop1"])
def test_gpu_one_step_bit_exact(case):
    a, b = _gpu_vs_oracle(case, one_step=True)
    helpers.assert_bit_identical(a, b, case)


@pytest.mark.parametrize("case", ["off", "ts_pp1", "pw"])
def test_gpu_scripted_tier_bit_exact(case):
    """A user-defined target population: the scripted tier's gather normalises a 'time step' Weight every step."""
    a, b = _gpu_vs_oracle(case, custom=True)
    helpers.assert_bit_identical(a, b, f"{case} scripted")


def test_gpu_large_batch_odd_shapes_bit_exact():
    a, b = _gpu_vs_oracle("t5", B=520, n_in=45, n=37)
    helpers.assert_bit_identical(a, b, "B=520")


@pytest.mark.parametrize("form", ["scalar", "tensor"])
def test_gpu_standalone_normalize_matches_oracle(form):
    from weight_norm_oracle import WeightNormOracleBackend

    F, _ = __import__("mcc_feature_nets").features(B200)
    g = torch.Generator().manual_seed(3)
    w = torch.randn(300, 70, generator=g)
    w[:, 5] = 0.0
    norm = 3.0 + torch.rand(70, generator=g) if form == "tensor" else 2.75
    outs = []
    for gpu in (True, False):
        X, Y = B200.nodes.Input(300), B200.nodes.LIFNodes(70)
        c = B200.topology.MulticompartmentConnection(source=X, target=Y, device="cpu",
                                                     pipeline=[F.Weight(name="w", value=w, norm=norm, norm_frequency="time step",
                                                                        range=[-10.0, 10.0])])
        s = (torch.rand(4, 300, generator=torch.Generator().manual_seed(1)) < 0.3).to(torch.uint8)
        if gpu:
            c.to("cuda")
            c.compute(s.cuda())
        else:
            with WeightNormOracleBackend():
                c.compute(s)
        outs.append(c.w.detach().cpu())
    assert torch.equal(outs[0], outs[1])


def test_gpu_dc_shape_bit_exact():
    from bindsnet_b200 import _backend
    from weight_norm_oracle import WeightNormOracleBackend

    outs = []
    for gpu in (True, False):
        net, x = wn.dc_graph(B200, 128, "time step", T=250)
        net.force_tier = 0
        if gpu:
            net.to("cuda")
            net.run(inputs={"X": x.cuda()}, time=250, one_spike_seed=7)
            net.check_errors()
            assert _backend.last_tier == 1
        else:
            with WeightNormOracleBackend() as ob:
                net.run(inputs={"X": x}, time=250, one_spike_seed=7)
            assert ob.err == 0
        outs.append(wn.full_snapshot(net, 250))
    helpers.assert_bit_identical(outs[0], outs[1], "dc")
    assert outs[0]["L/Ae/s"].sum() > 0 or outs[0]["L/Ae/theta"].sum() > 0
