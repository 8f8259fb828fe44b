"""Per-synapse wmin / wmax and learning-rate tensors of a dense Connection on the H100: the CUDA library's generic window
bit for bit against the oracle (tests/synapse_oracle.c), the equivalences (constant tensors = scalars, broadcast =
materialised), the single-operator update, and a recurrent E/I network at N = 4000, B = 128, T = 250."""
import pytest
import torch

import cases
import helpers
import synapse_nets as sn

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _gpu_vs_oracle(case, one_step=False, stepwise=False, T=20):
    from bindsnet_b200 import _backend
    from synapse_oracle import SynapseOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T, masks = sn.live_net(B200, case, T=T)
        if stepwise:
            net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["s", "refrac_count"], time=T), "Yr")
        if gpu:
            sn.to_device(net, "cuda")
            sn.run_two_windows(net, {k: v.cuda() for k, v in inputs.items()}, T, case, masks=masks, one_step=one_step)
            net.check_errors()
            assert _backend.last_tier == 1
        else:
            with SynapseOracleBackend() as ob:
                sn.run_two_windows(net, inputs, T, case, masks=masks, one_step=one_step)
            assert ob.err == 0
        outs.append(sn.snapshot(net))
    return outs


@pytest.mark.parametrize("case", sn.LIVE_CASES)
def test_gpu_cases_bit_exact(case):
    a, b = _gpu_vs_oracle(case)
    helpers.assert_bit_identical(a, b, case)
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("mode", ["one_step", "stepwise"])
@pytest.mark.parametrize("case", ["pp_tgt_mean", "wdep_src", "hebb_tgt", "mstdpet"])
def test_gpu_one_step_and_stepwise_bit_exact(case, mode):
    a, b = _gpu_vs_oracle(case, one_step=mode == "one_step", stepwise=mode == "stepwise", T=9)
    helpers.assert_bit_identical(a, b, f"{case} {mode}")


def _run(net, x, windows=2):
    for _ in range(windows):
        net.run(inputs={"X": x}, time=x.shape[0])
    net.check_errors()
    return sn.snapshot(net)


@pytest.mark.parametrize("B", [1, 32])
def test_gpu_equivalences(B):
    a = _run(*sn.ei_network(B200, 500, B, 30, seed=2, scalar_twin=True, device="cuda"))
    b = _run(*sn.constant_twin(B200, 500, B, 30, seed=2, device="cuda"))
    helpers.assert_bit_identical(a, b, "constant tensors vs scalars")
    c = _run(*sn.ei_network(B200, 500, B, 30, seed=4, device="cuda"))
    d = _run(*sn.ei_network(B200, 500, B, 30, seed=4, full_bounds=True, device="cuda"))
    helpers.assert_bit_identical(c, d, "per-row bounds vs their [n, n] copy")


def test_gpu_standalone_update_matches_oracle():
    from synapse_oracle import SynapseOracleBackend

    outs = []
    for gpu in (True, False):
        g = torch.Generator().manual_seed(8)
        X, Y = B200.nodes.Input(300, traces=True), B200.nodes.LIFNodes(200, traces=True)
        net = B200.Network(batch_size=5)
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        lo, hi = sn.bounds("src", 300, 200, g, inf=False)
        nu = sn.rates("full", "WeightDependentPostPre", 300, 200, g)
        c = B200.topology.Connection(X, Y, w=torch.rand(300, 200, generator=g), wmin=lo, wmax=hi, nu=nu,
                                     update_rule=B200.learning.WeightDependentPostPre, reduction=torch.sum)
        net.add_connection(c, "X", "Y")
        X.s, Y.s = torch.rand(5, 300, generator=g) < 0.3, torch.rand(5, 200, generator=g) < 0.3
        X.x, Y.x = torch.rand(5, 300, generator=g), torch.rand(5, 200, generator=g)
        if gpu:
            sn.to_device(net, "cuda")
            c.update()
            torch.cuda.synchronize()
        else:
            with SynapseOracleBackend():
                c.update()
        outs.append(c.w.detach().cpu().clone())
    assert torch.equal(outs[0], outs[1])


def test_gpu_rate_left_on_the_host_raises():
    """Network.to() does not move a rule's nu (the rule is not a Module): the window raises the reference's RuntimeError
    before anything runs."""
    net, inputs, T, _ = sn.live_net(B200, "wdep_full")
    net.to("cuda")
    w0 = net.connections[("X", "Y")].w.detach().clone()
    with pytest.raises(RuntimeError, match="same device"):
        net.run(inputs={k: v[:T].cuda() for k, v in inputs.items()}, time=T)
    assert torch.equal(net.connections[("X", "Y")].w, w0)


def test_gpu_ei_network_at_bench_shape():
    """N = 4000, B = 128, T = 250: runs on tier 1, every recurrent weight stays inside its row's sign bounds, and the
    per-row bounds give the same run as their materialised [N, N] copy."""
    from bindsnet_b200 import _backend

    outs = []
    for full in (False, True):
        net, x = sn.ei_network(B200, 4000, 128, 250, seed=1, device="cuda", full_bounds=full)
        net.run(inputs={"X": x}, time=250)
        net.check_errors()
        assert _backend.last_tier == 1
        yy = net.connections[("Y", "Y")]
        assert bool(((yy.w >= yy.wmin) & (yy.w <= yy.wmax)).all())
        outs.append({"w_in": net.connections[("X", "Y")].w.detach().cpu(), "w_rec": yy.w.detach().cpu(),
                     "s": net.layers["Y"].s.cpu()})
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k
