"""MaxPoo3dConnection on the H100: the CUDA library's window kernel and single operator bit for bit against the oracle
(tests/maxpool3d_oracle.c), on the cases tests/test_maxpool3d.py checks under emulation, the degenerate-depth twin of a
MaxPool2dConnection, and the benchmark's network (bench_maxpool3d.py) at B = 32, T = 250 and B = 128, T = 40."""
import pytest
import torch

import cases
import maxpool3d_nets as mn
from test_maxpool3d import VARIANTS, _restated

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _flat(states):
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


def _gpu_vs_oracle(build, **kw):
    from bindsnet_b200 import _backend
    from maxpool3d_oracle import MaxPool3dOracleBackend

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
            with MaxPool3dOracleBackend() as ob:
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


@pytest.mark.parametrize("case", ["b1_c2_d0.25_k2s2", "b4_c2_d0.25_d211", "b4_c2_d0.25_k123s121"])
def test_one_step_bit_exact(case):
    _gpu_vs_oracle(lambda: mn.conv_pool_net(B200, case), one_step=True)


@pytest.mark.parametrize("decay", [0.0, 1.0])
def test_ties_bit_exact(decay):
    _gpu_vs_oracle(lambda: mn.tie_net(B200, decay=decay))
    _gpu_vs_oracle(lambda: mn.tie_net(B200, B=520, T=7, decay=decay))


@pytest.mark.parametrize("B,T", [(3, 7), (33, 6)])
def test_batch_sizes_bit_exact(B, T):
    _gpu_vs_oracle(lambda: mn.tie_net(B200, B=B, T=T, decay=0.25))


def test_one_spike_source_bit_exact():
    a = _gpu_vs_oracle(lambda: mn.one_spike_net(B200))
    assert a["w1/Ss"].sum() > 0 and a["w1/Ps"].sum() > 0


@pytest.mark.parametrize("one_step", [False, True])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_source_variants_bit_exact(variant, one_step):
    a = _gpu_vs_oracle(lambda: mn.variant_net(B200, **VARIANTS[variant]), one_step=one_step, one_spike_seed=5)
    assert a["w1/Ss"].sum() > 0 and a["w1/Ps"].sum() > 0


@pytest.mark.parametrize("one_step", [False, True])
@pytest.mark.parametrize("T", [13, 14])
def test_consecutive_windows_bit_exact(T, one_step):
    _gpu_vs_oracle(lambda: mn.variant_net(B200, T=T), reset=False, one_step=one_step)


def test_stepwise_rates_monitor_bit_exact():
    from maxpool3d_oracle import MaxPool3dOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = mn.conv_pool_net(B200, "b4_c2_d0.25_k3s1", T=12)
        net.add_monitor(B200.monitors.Monitor(net.connections[("C1", "P")], ["firing_rates"], time=T), "fr")
        x = inputs["X"][0]
        if gpu:
            net.to("cuda")
            net.run(inputs={"X": x.cuda()}, time=T)
            net.check_errors()
        else:
            with MaxPool3dOracleBackend():
                net.run(inputs={"X": x}, time=T)
        outs.append({"fr": net.monitors["fr"].get("firing_rates").cpu(), **mn.state(net)})
    for k in outs[1]:
        assert torch.equal(outs[0][k], outs[1][k]), k


@pytest.mark.parametrize("one_step", [False, True])
@pytest.mark.parametrize("one_spike", [False, True])
def test_twin_of_max_pool_2d_bit_identical(one_spike, one_step):
    from maxpool_nets import run_two_windows

    outs = []
    for three_d in (True, False):
        net, inputs, T = mn.twin_net(B200, three_d, one_spike=one_spike)
        net.to("cuda")
        outs.append(_flat(run_two_windows(net, {k: v.cuda() for k, v in inputs.items()}, T, one_step=one_step, one_spike_seed=3)))
        net.check_errors()
    a, b = outs
    for k in a:
        assert torch.equal(a[k].flatten(), b[k].flatten()), k
    assert a["w1/Ps"].sum() > 0


@pytest.mark.parametrize("geom", list(mn.GEOMS))
def test_standalone_compute_matches_max_pool3d(geom):
    kw = mn.pool_kwargs(geom)
    vol = mn.GEOMS[geom][4]
    g = torch.Generator().manual_seed(3)
    C_, B = 3, 600
    X = B200.nodes.Input(shape=[C_, *vol])
    X.set_batch_size(B)
    P = B200.nodes.LIFNodes(shape=list(mn.pooled_shape(C_, vol, geom)))
    conn = B200.topology.MaxPoo3dConnection(X, P, decay=0.3, **kw).to("cuda")
    fr = conn.firing_rates.cpu().clone()
    for step in range(4):
        s = torch.rand(B, C_, *vol, generator=g) < 0.4
        out = conn.compute(s.cuda())
        fr, ref = _restated(fr, s, 0.3, kw["kernel_size"], kw["stride"], kw["padding"], kw["dilation"])
        assert torch.equal(conn.firing_rates.cpu(), fr), step
        assert torch.equal(out.cpu(), ref), step


@pytest.mark.parametrize("B,T", [(32, 250), (128, 40)])
def test_benchmark_network_bit_exact(B, T):
    """The whole batch on the device; the first four samples on the oracle (learning is off and no layer couples the
    samples, so each sample's window is its own computation), compared sample for sample."""
    from maxpool3d_oracle import MaxPool3dOracleBackend

    k = 4
    assert _tier_of(lambda: mn.bench_net(B200, B=B, T=T)) == 1
    net, inputs, _ = mn.bench_net(B200, B=B, T=T)
    net.to("cuda")
    net.run(inputs={"X": inputs["X"][0].cuda()}, time=T)
    net.check_errors()
    gpu = mn.state(net)
    sub, sub_inputs, _ = mn.bench_net(B200, B=k, T=T)
    with MaxPool3dOracleBackend() as ob:
        sub.run(inputs={"X": inputs["X"][0, :, :k].clone()}, time=T)
    assert ob.err == 0
    cpu = mn.state(sub)
    for name, v in cpu.items():
        g = gpu[name]
        g = g[:, :k] if name in ("Ps", "Ys") else g if name.endswith("/w") else g[:k]
        assert torch.equal(g, v), f"{name} differs from the oracle"
    assert cpu["Ps"].sum() > 0 and cpu["Ys"].sum() > 0
