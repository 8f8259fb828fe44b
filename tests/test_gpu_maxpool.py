"""MaxPool2dConnection on the H100: the CUDA library's window kernel and single operator bit for bit against the oracle
(tests/maxpool_oracle.c), on the cases tests/test_maxpool.py checks under emulation, plus a config-4-sized conv-pool
network at B = 128."""
import pytest
import torch

import cases
import maxpool_nets as mn
from test_maxpool import _restated

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _flat(states):
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


def _gpu_vs_oracle(build, **kw):
    from bindsnet_b200 import _backend
    from maxpool_oracle import MaxPoolOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = build()
        if gpu:
            net.to("cuda")
            inputs = {k: v.cuda() for k, v in inputs.items()}
            outs.append(_flat(mn.run_two_windows(net, inputs, T, **kw)))
            net.check_errors()
            assert _backend.lib().snn_b200_abi_version() == 13
        else:
            with MaxPoolOracleBackend() as ob:
                outs.append(_flat(mn.run_two_windows(net, inputs, T, **kw)))
            assert ob.err == 0
    a, b = outs
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), f"{k} differs from the oracle"
    return a


def _tier_of(build):
    import ctypes as C

    from bindsnet_b200 import _abi, _backend
    from bindsnet_b200.network import _plan

    net, _, T = build()
    net.to("cuda")
    plan, keep = _plan.build_net(net, net.batch_size, {}, {}, {}, {}, {})
    opts = _abi.SnnRunOpts()
    opts.T, opts.B = T, net.batch_size
    return int(_backend.lib().snn_b200_select_tier(C.byref(plan), C.byref(opts)))


@pytest.mark.parametrize("case", mn.LIVE_CASES)
def test_window_bit_exact(case):
    a = _gpu_vs_oracle(lambda: mn.conv_pool_net(B200, case))
    assert a["w1/Ps"].sum() > 0


@pytest.mark.parametrize("case", ["b1_d0.25_k2s2", "b4_d1_k2s1d2", "b4_d0_k3s2p1d2"])
def test_one_step_bit_exact(case):
    _gpu_vs_oracle(lambda: mn.conv_pool_net(B200, case), one_step=True)


@pytest.mark.parametrize("decay", [0.0, 1.0])
def test_ties_bit_exact(decay):
    _gpu_vs_oracle(lambda: mn.tie_net(B200, decay=decay))
    _gpu_vs_oracle(lambda: mn.tie_net(B200, B=770, T=7, decay=decay))


@pytest.mark.parametrize("one_step", [False, True])
@pytest.mark.parametrize("variant", [dict(one_spike=True), dict(target_first=True), dict(one_spike=True, target_first=True)])
def test_source_variants_bit_exact(variant, one_step):
    a = _gpu_vs_oracle(lambda: mn.variant_net(B200, **variant), one_step=one_step, one_spike_seed=5)
    assert a["w1/Ss"].sum() > 0 and a["w1/Ps"].sum() > 0


@pytest.mark.parametrize("one_step", [False, True])
@pytest.mark.parametrize("T", [13, 14])
def test_consecutive_windows_bit_exact(T, one_step):
    _gpu_vs_oracle(lambda: mn.variant_net(B200, T=T), reset=False, one_step=one_step)


def test_stepwise_rates_monitor_bit_exact():
    from maxpool_oracle import MaxPoolOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = mn.conv_pool_net(B200, "b4_d0.25_k3s1", T=12)
        net.add_monitor(B200.monitors.Monitor(net.connections[("C1", "P")], ["firing_rates"], time=T), "fr")
        x = inputs["X"][0]
        if gpu:
            net.to("cuda")
            net.run(inputs={"X": x.cuda()}, time=T)
            net.check_errors()
        else:
            with MaxPoolOracleBackend():
                net.run(inputs={"X": x}, time=T)
        outs.append({"fr": net.monitors["fr"].get("firing_rates").cpu(), **mn.state(net)})
    for k in outs[1]:
        assert torch.equal(outs[0][k], outs[1][k]), k


@pytest.mark.parametrize("geom", list(mn.GEOMS))
def test_standalone_compute_matches_max_pool2d(geom):
    k, st, p, d = mn.GEOMS[geom]
    g = torch.Generator().manual_seed(3)
    C_, H, W, B = 3, 9, 10, 600
    X = B200.nodes.Input(shape=[C_, H, W])
    X.set_batch_size(B)
    P = B200.nodes.LIFNodes(shape=list(mn.pooled_shape(C_, H, W, geom)))
    conn = B200.topology.MaxPool2dConnection(X, P, kernel_size=k, stride=st, padding=p, dilation=d, decay=0.3).to("cuda")
    fr = conn.firing_rates.cpu().clone()
    for step in range(4):
        s = torch.rand(B, C_, H, W, generator=g) < 0.4
        out = conn.compute(s.cuda())
        fr, ref = _restated(fr, s, 0.3, k, st, p, d)
        assert torch.equal(conn.firing_rates.cpu(), fr), step
        assert torch.equal(out.cpu(), ref), step


def test_config4_sized_conv_pool_b128():
    build = lambda: mn.c4_pool_net(B200, B=128, T=40)
    assert _tier_of(build) == 1
    a = _gpu_vs_oracle(build)
    assert a["w1/Ps"].sum() > 0 and a["w1/Ys"].sum() > 0
