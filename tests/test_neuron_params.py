"""Per-neuron parameter tensors of LIFNodes, AdaptiveLIFNodes and DiehlAndCookNodes (reference: nodes.py:96-107,
500-559, 921-978, 1069-1144: thresh, rest, tc_decay, theta_plus, tc_theta_decay, tc_trace and an additive trace_scale
given as tensors), run on the generic window kernel.  CPU tests: the oracle against the live reference's stored results,
the emulated kernel against the oracle bit for bit, equivalences (constant tensors = scalars, per-channel = materialised),
refusals and tier selection.  "The oracle" here is tests/neuron_param_oracle.c.  The stored reference results are
regenerated with ``python tests/golden/gen_live.py test_neuron_params``."""
import os
import sys

import pytest
import torch

import cases
import helpers
import neuron_param_nets as pn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

@reference_side(pn.LIVE_CASES)
def _live(ns, case):
    net, inputs, T = pn.live_net(ns, case)
    return pn.run_two_windows(net, inputs, T, reference=True)


@pytest.mark.parametrize("case", pn.LIVE_CASES)
def test_oracle_matches_live_reference(case):
    from neuron_param_oracle import NeuronParamOracleBackend

    ref = load(_live, case)
    net, inputs, T = pn.live_net(B200, case)
    with NeuronParamOracleBackend() as ob:
        ours = pn.run_two_windows(net, inputs, T)
    assert ob.err == 0
    for k in ("0", "1"):
        assert torch.equal(ours[f"{k}/Ys"], ref[f"{k}/Ys"]), f"window {k}: spike rasters differ"
        assert ours[f"{k}/Ys"].sum() > 0
        for name in [n for n in ref if n.startswith(f"{k}/") and n != f"{k}/Ys"]:
            torch.testing.assert_close(ours[name], ref[name], rtol=1e-5, atol=1e-4, msg=f"{name}")


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _with_env(env, fn):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return fn()
    finally:
        for k, v in old.items():
            os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)


def _emu_vs_oracle(build, env, windows=2, **run_kw):
    """``build()`` -> (net, inputs, T); both backends run ``windows`` windows without a reset."""
    import emu
    from neuron_param_oracle import NeuronParamOracleBackend

    outs = []
    for backend in (emu.EmuBackend, NeuronParamOracleBackend):
        net, inputs, T = build()
        torch.manual_seed(5)   # (the one_spike tie-break seed Network.run draws)

        def go():
            with backend() as be:
                for k in range(windows):
                    net.run(inputs=pn.window_inputs(inputs, T, k), time=T, **run_kw)
                assert be.err == 0
        _with_env(env if backend is emu.EmuBackend else {}, go)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
        outs.append(pn.snapshot(net))
    return outs


def _dc_one_spike(B=3, T=12):
    g = torch.Generator().manual_seed(3)
    net = B200.Network(dt=1.0, batch_size=B, learning=True)
    X = B200.nodes.Input(pn.N_IN, traces=True)
    Y = pn.population(B200, "DiehlAndCookNodes", pn.N, g, one_spike=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    net.add_connection(B200.topology.Connection(X, Y, w=3.0 * torch.rand(pn.N_IN, pn.N, generator=g), update_rule=B200.learning.PostPre,
                                                nu=(1e-2, 1e-2), reduction=torch.sum, wmin=0.0, wmax=3.0), "X", "Y")
    net.add_monitor(B200.monitors.Monitor(Y, ["s"], time=T), "Ys")
    return net, {"X": (torch.rand(2 * T, B, pn.N_IN, generator=g) < 0.3).to(torch.uint8)}, T


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["lif_b4", "dc", "alif", "conv_chan", "traces", "ei", "dc_one_spike"])
def test_emulated_kernel_bit_exact(case, env):
    build = _dc_one_spike if case == "dc_one_spike" else (lambda: pn.live_net(B200, case, T=10))
    a, b = _emu_vs_oracle(build, ENVS[env])
    helpers.assert_bit_identical(a, b, f"{case} {env}")
    assert a["L/Y/s"].sum() + a.get("M/Ys", a["L/Y/s"]).sum() > 0


@pytest.mark.parametrize("mode", ["one_step", "stepwise"])
@pytest.mark.parametrize("case", ["lif_b1", "dc", "traces"])
def test_emulated_kernel_one_step_and_stepwise_bit_exact(case, mode):
    def build():
        net, inputs, T = pn.live_net(B200, case, T=7)
        if mode == "stepwise":   # a monitor on a state the kernel does not record: one-step windows
            net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["s", "refrac_count"], time=T), "Yr")
        return net, inputs, T
    a, b = _emu_vs_oracle(build, ENVS["sms3"], one_step=mode == "one_step")
    helpers.assert_bit_identical(a, b, f"{case} {mode}")


def test_emulated_kernel_large_batch_odd_T():
    """B = 520, odd T, two windows without a reset, one_spike on."""
    a, b = _emu_vs_oracle(lambda: _dc_one_spike(B=520, T=7), ENVS["sms3"])
    helpers.assert_bit_identical(a, b, "B = 520, T = 7")


def test_scripted_tier_with_a_user_defined_layer():
    """The scripted tier (a user-defined population in the network): the built-in layers' one-step windows read the
    per-neuron block."""
    from test_scripted_tier import MyLIF

    def build():
        net, inputs, T = pn.live_net(B200, "lif_b4", T=6)
        U = MyLIF(12)
        net.add_layer(U, "U")
        g = torch.Generator().manual_seed(4)
        net.add_connection(B200.topology.Connection(net.layers["Y"], U, w=3.0 * torch.rand(pn.N, 12, generator=g)), "Y", "U")
        return net, inputs, T
    a, b = _emu_vs_oracle(build, ENVS["sms3"])
    helpers.assert_bit_identical(a, b, "scripted tier")


def test_single_layer_forward():
    """``layer.forward(x)`` (a one-layer, one-step window) reads the per-neuron block like Network.run."""
    import emu
    from neuron_param_oracle import NeuronParamOracleBackend

    outs = []
    for backend in (emu.EmuBackend, NeuronParamOracleBackend):
        g = torch.Generator().manual_seed(6)
        Y = pn.population(B200, "DiehlAndCookNodes", 40, g)
        net = B200.Network(dt=1.0, batch_size=3)
        net.add_layer(Y, "Y")
        with backend():
            for _ in range(5):
                Y.forward(20.0 * torch.rand(3, 40, generator=g))
        outs.append({"v": Y.v.numpy().copy(), "s": Y.s.numpy().copy(), "theta": Y.theta.numpy().copy()})
    helpers.assert_bit_identical(outs[0], outs[1], "single-layer forward")


# ---- 3. equivalences, bit for bit ------------------------------------------------------------------------------------

def _run_emu(net, x, windows=2, **kw):
    import emu

    torch.manual_seed(5)   # (the one_spike tie-break seed Network.run draws)
    with emu.EmuBackend() as be:
        for k in range(windows):
            net.run(inputs={"X": x}, time=x.shape[0], **kw)
        assert be.err == 0
    return pn.snapshot(net)


@pytest.mark.parametrize("one_spike", [False, True])
def test_constant_tensors_equal_scalars(one_spike):
    """Tensors filled with the scalars give the scalar network's results bit for bit on the generic tier."""
    a = _run_emu(*pn.dc2015_like(B200, 64, 3, 9, n_in=48, seed=2, constant=True, one_spike=one_spike))
    net, x = pn.dc2015_like(B200, 64, 3, 9, n_in=48, seed=2, constant=True, one_spike=one_spike)
    E = net.layers["Ae"]
    E.thresh, E.theta_plus = torch.tensor(-52.0), torch.tensor(0.05)
    net.force_tier = 1
    b = _run_emu(net, x)
    helpers.assert_bit_identical(a, b, "constant tensors vs scalars")


def test_per_channel_equals_materialised():
    """A [C, 1, 1] threshold equals its materialised [C, H, W] copy bit for bit."""
    a = _run_emu(*_conv_net(False))
    b = _run_emu(*_conv_net(True))
    helpers.assert_bit_identical(a, b, "[C, 1, 1] vs [C, H, W]")


def _conv_net(materialised):
    net, inputs, T = pn.live_net(B200, "conv_chan", T=8)
    Y = net.layers["Y"]
    if materialised:
        Y.thresh = Y.thresh.expand(3, 4, 4).contiguous()
    return net, inputs["X"][:T]


# ---- 4. refusals and tier selection ----------------------------------------------------------------------------------

def _state(net):
    return {k: v.copy() for k, v in pn.snapshot(net).items()}


@pytest.mark.parametrize("name,exc", [("refrac", RuntimeError), ("reset", RuntimeError), ("lbound", RuntimeError),
                                      ("trace_scale", RuntimeError)])
def test_refused_tensor_parameters(name, exc):
    """refrac / reset / lbound / a non-additive trace_scale reach the reference's masked_fill_, which takes a 0-dim value:
    its first step raises RuntimeError.  Here the plan raises it, before any state changes."""
    import emu

    for kind in ("LIFNodes", "DiehlAndCookNodes", "AdaptiveLIFNodes"):
        net, inputs, T = pn.live_net(B200, "lif_b1" if kind == "LIFNodes" else "alif")
        Y = net.layers["Y"]
        if kind == "DiehlAndCookNodes":
            Y.one_spike = True
        value = torch.linspace(-70.0, -66.0, pn.N)
        if name == "trace_scale":
            Y.trace_scale = torch.linspace(0.5, 1.0, pn.N)
        elif name == "lbound":
            Y.lbound = value
        else:
            setattr(Y, name, value)
        before = _state(net)
        with emu.EmuBackend(), pytest.raises(exc, match="masked_fill_"):
            net.run(inputs=pn.window_inputs(inputs, T, 0), time=T)
        helpers.assert_bit_identical(before, _state(net), f"{kind}.{name}")


def test_reset_with_tensor_rest_raises():
    """reset_state_variables() calls v.fill_(rest), which raises RuntimeError for a tensor rest in the reference;
    set_batch_size (rest * ones) works."""
    net, inputs, T = pn.live_net(B200, "lif_b4")
    Y = net.layers["Y"]
    before = _state(net)
    with pytest.raises(RuntimeError, match="fill_"):
        net.reset_state_variables()
    with pytest.raises(RuntimeError, match="fill_"):
        Y.reset_state_variables()
    helpers.assert_bit_identical(before, _state(net), "reset")
    Y.set_batch_size(2)
    assert torch.equal(Y.v, Y.rest * torch.ones(2, pn.N))


def test_shapes():
    """A tensor that would grow the state raises NotImplementedError; one that does not broadcast, RuntimeError."""
    import emu

    for thresh, exc in ((torch.full((2, pn.N), -55.0), NotImplementedError), (torch.full((7,), -55.0), RuntimeError)):
        net, inputs, T = pn.live_net(B200, "lif_b1")
        net.layers["Y"].thresh = thresh
        with emu.EmuBackend(), pytest.raises(exc):
            net.run(inputs=pn.window_inputs(inputs, T, 0), time=T)


def test_other_populations_keep_their_message():
    """Populations other than the three keep today's refusal, word for word."""
    import emu

    g = torch.Generator().manual_seed(1)
    for cls in (B200.nodes.IFNodes, B200.nodes.CurrentLIFNodes, B200.nodes.BoostedLIFNodes, B200.nodes.McCullochPitts):
        net = B200.Network(dt=1.0, batch_size=1)
        X = B200.nodes.Input(8)
        Y = cls(6, thresh=torch.full((6,), -50.0))
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        net.add_connection(B200.topology.Connection(X, Y, w=torch.rand(8, 6, generator=g)), "X", "Y")
        with emu.EmuBackend(), pytest.raises(NotImplementedError,
                                             match=r"per-neuron tensor for 'thresh' is not supported by the CUDA core yet \(scalar only\)"):
            net.run(inputs={"X": torch.zeros(3, 1, 8, dtype=torch.uint8)}, time=3)


def test_not_with_the_pooling_instantiation():
    import emu

    net = B200.Network(dt=1.0, batch_size=1, learning=False)
    X = B200.nodes.Input(shape=[1, 4, 4])
    Y = B200.nodes.LIFNodes(shape=[1, 4, 4], thresh=torch.linspace(-55.0, -50.0, 16).view(1, 4, 4))
    Z = B200.nodes.LIFNodes(shape=[1, 2, 2])
    net.add_layer(X, "X"); net.add_layer(Y, "Y"); net.add_layer(Z, "Z")
    net.add_connection(B200.topology.Connection(X, Y, w=torch.rand(16, 16)), "X", "Y")
    net.add_connection(B200.topology.MaxPool2dConnection(Y, Z, kernel_size=2, stride=2, decay=0.5), "Y", "Z")
    with emu.EmuBackend(), pytest.raises(NotImplementedError, match="per-neuron"):
        net.run(inputs={"X": torch.zeros(2, 1, 1, 4, 4, dtype=torch.uint8)}, time=2)


def test_tier_selection():
    """tier 0 and 1 select the generic kernel; a forced fused tier (and a delta window) is SNN_ERR_UNSUPPORTED; an
    older-style plan without the flag ignores pn_mask; a malformed block is SNN_ERR_BAD_ARG."""
    import emu
    from bindsnet_b200 import _abi, _backend
    from bindsnet_b200.network import _plan

    net, x = pn.dc2015_like(B200, 32, 2, 4, n_in=16, seed=1)
    B200.Network.run   # (the host builds plans through _plan.build_net)
    with emu.EmuBackend():
        d, keep = _plan.build_net(net, 2, {"X": x.contiguous()}, {}, {}, {}, {})
        assert d.layers[1].kind == _abi.SNN_NODE_DC | _abi.SNN_NODE_PN
        assert d.layers[1].pn_mask == (1 << _abi.SNN_PN_THRESH) | (1 << _abi.SNN_PN_THETA_PLUS)
        lib = emu.lib()
        for tier, want in ((0, 1), (1, 1), (2, 0), (3, 0)):
            o = _abi.SnnRunOpts(); o.T, o.B, o.tier = 4, 2, tier
            assert lib.snn_b200_select_tier(d, o) == want, tier
        o = _abi.SnnRunOpts(); o.T, o.B, o.tier = 4, 2, 0
        dw = torch.zeros(16 * 32); o.delta_w = dw.data_ptr()
        assert lib.snn_b200_select_tier(d, o) == 0
        o.delta_w = None
        mask = d.layers[1].pn_mask
        d.layers[1].pn_mask = mask | (1 << _abi.SNN_PN_TRACE_SCALE)   # traces_additive is off
        assert lib.snn_b200_select_tier(d, o) == 0
        d.layers[1].pn_mask = mask
        d.layers[2].kind |= _abi.SNN_NODE_PN   # a LIF layer with the flag and no rows: fine
        assert lib.snn_b200_select_tier(d, o) == 1
        d.layers[0].kind |= _abi.SNN_NODE_PN   # the flag on an Input layer
        assert lib.snn_b200_select_tier(d, o) == 0
        del keep
    assert _backend is not None


def test_reference_network_through_the_binding():
    """The reference's own network with per-neuron tensors runs through reference_binding on the oracle and reproduces
    the stored live results of its first window."""
    from bindsnet_b200 import reference_binding as rb
    from neuron_param_oracle import lib

    try:
        ref_ns = cases.namespace("reference")
    except ImportError:
        pytest.skip("the reference copy is not built")
    for case in ("lif_b4", "dc", "traces"):
        ref = load(_live, case)
        net, inputs, T = pn.live_net(ref_ns, case)
        rb.run_window(net, pn.window_inputs(inputs, T, 0), time=T, library=lib())
        Y = net.layers["Y"]
        torch.testing.assert_close(Y.v, ref["0/Y/v"], rtol=1e-5, atol=1e-4)
        torch.testing.assert_close(Y.x, ref["0/Y/x"], rtol=1e-5, atol=1e-4)
