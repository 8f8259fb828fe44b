"""MCC_learning.PostPre with average_update on the H100: the CUDA library's generic window bit for bit against the
oracle (tests/mcc_average_oracle.c) on the CPU cases, the standalone update, and a DiehlAndCook-shaped layer at the
benchmark's shape (Input(784) -> 1600, k = 10, B = 128, T = 250)."""
import pytest
import torch

import cases
import helpers
import mcc_average_nets as an

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _gpu_vs_oracle(case, one_step=False, stepwise=False, B=None, n_in=40, n=30):
    from bindsnet_b200 import _backend
    from mcc_average_oracle import AverageOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = an.live_net(B200, case, B=B, n_in=n_in, n=n)
        net.force_tier = 1
        if stepwise:
            net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["s", "refrac_count"], time=T), "Yr")
        if gpu:
            net.to("cuda")
            an.run_windows(net, {k: v.cuda() for k, v in inputs.items()}, T, one_step=one_step)
            net.check_errors()
            assert _backend.last_tier == 1
        else:
            with AverageOracleBackend() as ob:
                an.run_windows(net, inputs, T, one_step=one_step)
            assert ob.err == 0
        outs.append(an.full_snapshot(net, T))
    return outs


@pytest.mark.parametrize("case", an.LIVE_CASES)
def test_gpu_live_cases_bit_exact(case):
    a, b = _gpu_vs_oracle(case)
    helpers.assert_bit_identical(a, b, case)
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("mode", ["one_step", "stepwise"])
@pytest.mark.parametrize("case", ["k3", "b4_sum", "pw"])
def test_gpu_one_step_and_stepwise_bit_exact(case, mode):
    a, b = _gpu_vs_oracle(case, one_step=mode == "one_step", stepwise=mode == "stepwise")
    helpers.assert_bit_identical(a, b, f"{case} {mode}")


def test_gpu_large_batch_odd_T_bit_exact():
    a, b = _gpu_vs_oracle("t5", B=520, n_in=70, n=40)
    helpers.assert_bit_identical(a, b, "B=520")


def test_gpu_standalone_update_bit_exact():
    from mcc_average_oracle import AverageOracleBackend

    outs = []
    for gpu in (True, False):
        F, ML = an.features(B200)
        g = torch.Generator().manual_seed(4)
        X, Y = B200.nodes.Input(70, traces=True), B200.nodes.LIFNodes(50, traces=True)
        net = B200.Network(dt=1.0, batch_size=3)
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        wt = F.Weight("w", 0.9 * torch.rand(70, 50, generator=g), learning_rule=ML.PostPre, nu=(0.07, 0.05), range=[0.0, 0.9])
        c = B200.topology.MulticompartmentConnection(source=X, target=Y, pipeline=[wt], average_update=3, continues_update=True)
        net.add_connection(c, "X", "Y")
        dev = "cuda" if gpu else "cpu"
        net.to(dev)
        with AverageOracleBackend() if not gpu else torch.no_grad():
            for _ in range(5):
                X.s = (torch.rand(3, 70, generator=g) < 0.3).to(dev)
                Y.s = (torch.rand(3, 50, generator=g) < 0.2).to(dev)
                X.x = torch.rand(3, 70, generator=g).to(dev)
                Y.x = torch.rand(3, 50, generator=g).to(dev)
                c.update(learning=True)
        r = wt.learning_rule
        outs.append({"w": c.w.cpu().numpy(), "pre": r.average_buffer_pre.cpu().numpy(), "post": r.average_buffer_post.cpu().numpy(),
                     "rows": r._avg_rows.cpu().numpy(), "cols": r._avg_cols.cpu().numpy()})
    helpers.assert_bit_identical(outs[0], outs[1], "standalone update")


@pytest.mark.parametrize("cont", [False, True])
def test_gpu_diehl_and_cook_shape_bit_exact(cont):
    """Input(784) -> 1600 DiehlAndCook one_spike layer through an averaged MCC PostPre (k = 10), B = 128, T = 250."""
    import bench_mcc_average as bm
    from mcc_average_oracle import AverageOracleBackend

    outs = []
    for gpu in (True, False):
        net, x = bm.build(B=128, k=10, cont=cont, T=250, device="cuda" if gpu else "cpu")
        if gpu:
            net.run({"X": x}, time=250, one_spike_seed=3)
            net.check_errors()
        else:
            with AverageOracleBackend(threads=0) as ob:
                net.run({"X": x}, time=250, one_spike_seed=3)
            assert ob.err == 0
        r = an.rule_of(net.connections[("X", "Ae")])
        outs.append({"w": net.connections[("X", "Ae")].w.cpu().numpy(), "theta": net.layers["Ae"].theta.cpu().numpy(),
                     "pre": r.average_buffer_pre.cpu().numpy(), "post": r.average_buffer_post.cpu().numpy()})
    helpers.assert_bit_identical(outs[0], outs[1], f"DiehlAndCook shape continues={cont}")
