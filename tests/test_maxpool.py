"""MaxPool2dConnection (reference: topology.py:1124-1211) on the generic window kernel.  CPU tests: the oracle
(tests/maxpool_oracle.c, the CPU oracle extended by the pooling connection) against the live reference's stored results,
the emulated kernel against the oracle bit for bit, the standalone compute against F.max_pool2d, refusals and tier
selection.  The stored reference results are regenerated with ``python tests/golden/gen_live.py test_maxpool``."""
import ctypes as C
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import cases
import maxpool_nets as mn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")
TIE_DECAYS = [0.0, 1.0]


def _flat(states):
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

@reference_side(mn.LIVE_CASES)
def _live_conv_pool(ns, case):
    net, inputs, T = mn.conv_pool_net(ns, case)
    return _flat(mn.run_two_windows(net, inputs, T))


@reference_side(TIE_DECAYS)
def _live_ties(ns, decay):
    net, inputs, T = mn.tie_net(ns, decay=decay)
    return _flat(mn.run_two_windows(net, inputs, T))


@reference_side([0])
def _live_rates_monitor(ns, _):
    """A Monitor on the connection's firing_rates (the window then runs step by step here)."""
    net, inputs, T = mn.conv_pool_net(ns, "b4_d0.25_k3s1", T=12)
    pool = net.connections[("C1", "P")]
    net.add_monitor(ns.monitors.Monitor(pool, ["firing_rates"], time=T), "fr")
    net.run(inputs={"X": inputs["X"][0]}, time=T)
    return {"fr": net.monitors["fr"].get("firing_rates").detach().clone(), **mn.state(net)}


def _check_against(ref, ours, what):
    for k, v in ref.items():
        o = ours[k]
        assert o.shape == v.shape, (what, k)
        if k.endswith("/fr") or k.endswith("s") or k == "fr":
            assert torch.equal(o.float(), v.float()), f"{what}: {k} differs"
        else:
            torch.testing.assert_close(o.float(), v.float(), rtol=1e-5, atol=1e-4, msg=f"{what}: {k}")


@pytest.mark.parametrize("case", mn.LIVE_CASES)
def test_oracle_matches_live_reference(case):
    from maxpool_oracle import MaxPoolOracleBackend

    net, inputs, T = mn.conv_pool_net(B200, case)
    with MaxPoolOracleBackend() as ob:
        ours = _flat(mn.run_two_windows(net, inputs, T))
    assert ob.err == 0
    _check_against(load(_live_conv_pool, case), ours, case)
    assert ours["w1/Ps"].sum() > 0 and ours["w1/Ys"].sum() > 0


@pytest.mark.parametrize("decay", TIE_DECAYS)
def test_oracle_ties_match_live_reference(decay):
    from maxpool_oracle import MaxPoolOracleBackend

    net, inputs, T = mn.tie_net(B200, decay=decay)
    with MaxPoolOracleBackend():
        ours = _flat(mn.run_two_windows(net, inputs, T))
    _check_against(load(_live_ties, decay), ours, f"ties decay={decay}")
    # the case is built to tie: in most windows of the last step some two elements have the same rate
    fr = ours["w1/XP/fr"].view(4, 3, 4, 2, 4, 2).permute(0, 1, 2, 4, 3, 5).reshape(4, 3, 4, 4, 4)
    ties = (fr.unsqueeze(-1) == fr.unsqueeze(-2)).sum((-1, -2)) > 4
    assert ties.float().mean() > 0.5


def test_rates_monitor_matches_live_reference():
    import emu

    ref = load(_live_rates_monitor, 0)
    net, inputs, T = mn.conv_pool_net(B200, "b4_d0.25_k3s1", T=12)
    net.add_monitor(B200.monitors.Monitor(net.connections[("C1", "P")], ["firing_rates"], time=T), "fr")
    with emu.EmuBackend() as be:
        net.run(inputs={"X": inputs["X"][0]}, time=T)
    assert be.err == 0
    ours = {"fr": net.monitors["fr"].get("firing_rates"), **mn.state(net)}
    _check_against(ref, ours, "stepwise")


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _emu_vs_oracle(build, env=None, **kw):
    import emu
    from maxpool_oracle import MaxPoolOracleBackend

    outs = []
    for backend in (emu.EmuBackend, MaxPoolOracleBackend):
        net, inputs, T = build()
        net.force_tier = 1
        old = {k: os.environ.get(k) for k in (env or {})}
        os.environ.update(env if backend is emu.EmuBackend and env else {})
        try:
            with backend() as be:
                outs.append(_flat(mn.run_two_windows(net, inputs, T, **kw)))
            assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
    a, b = outs
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), f"{k} differs"
    return a


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["b4_d0.25_k3s1", "b1_d0_k3s2p1", "b4_d0_k3s2p1d2", "b4_d0.25_k23s12p10"])
def test_emulated_kernel_bit_exact(case, env):
    a = _emu_vs_oracle(lambda: mn.conv_pool_net(B200, case), ENVS[env])
    assert a["w1/Ps"].sum() > 0


@pytest.mark.parametrize("case", ["b1_d0.25_k2s2", "b4_d1_k2s1d2"])
def test_emulated_kernel_one_step_bit_exact(case):
    _emu_vs_oracle(lambda: mn.conv_pool_net(B200, case), ENVS["sms3"], one_step=True)


@pytest.mark.parametrize("decay", TIE_DECAYS)
def test_emulated_kernel_ties_bit_exact(decay):
    _emu_vs_oracle(lambda: mn.tie_net(B200, decay=decay), ENVS["sms7"])
    _emu_vs_oracle(lambda: mn.tie_net(B200, decay=decay), ENVS["sms3"], one_step=True)


@pytest.mark.parametrize("T", [5, 6])
def test_emulated_kernel_large_batch_bit_exact(T):
    """B = 770 (> 768) and an odd and an even window length (the rates' slot parity)."""
    a = _emu_vs_oracle(lambda: mn.tie_net(B200, B=770, T=T, decay=0.25), ENVS["sms3"])
    assert a["w1/Ps"].sum() > 0


VARIANTS = {"one_spike_source": dict(one_spike=True), "target_first": dict(target_first=True),
            "one_spike_target_first": dict(one_spike=True, target_first=True)}


@pytest.mark.parametrize("one_step", [False, True])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_emulated_kernel_source_variants_bit_exact(variant, one_step):
    """A DiehlAndCookNodes(one_spike) source, whose rates advance in phase 2, and a source added after its target, which
    the target reads one step late in one-step mode too."""
    a = _emu_vs_oracle(lambda: mn.variant_net(B200, **VARIANTS[variant]), ENVS["sms3"], one_step=one_step, one_spike_seed=5)
    assert a["w1/Ss"].sum() > 0 and a["w1/Ps"].sum() > 0


@pytest.mark.parametrize("one_step", [False, True])
@pytest.mark.parametrize("T", [13, 14])
def test_emulated_kernel_consecutive_windows_bit_exact(T, one_step):
    """Two windows without a reset: the second window's prologue folds the first window's last spikes into the rates."""
    a = _emu_vs_oracle(lambda: mn.variant_net(B200, T=T), ENVS["sms7"], reset=False, one_step=one_step)
    assert a["w0/S/s"].sum() > 0 and not torch.equal(a["w0/SP/fr"], torch.zeros_like(a["w0/SP/fr"]))


def test_stepwise_equals_window():
    import emu

    outs = []
    for stepwise in (True, False):
        net, inputs, T = mn.conv_pool_net(B200, "b4_d0.25_k3s2p1", T=10)
        if stepwise:
            net.add_monitor(B200.monitors.Monitor(net.connections[("C1", "P")], ["firing_rates"], time=T), "fr")
        with emu.EmuBackend():
            net.run(inputs={"X": inputs["X"][0]}, time=T)
        outs.append(mn.state(net))
    for k in outs[1]:
        assert torch.equal(outs[0][k], outs[1][k]), k


@pytest.mark.parametrize("one_step", [False, True])
def test_scripted_tier_equals_window(one_step):
    import emu
    from maxpool_oracle import MaxPoolOracleBackend

    def build(user):
        net, inputs, T = mn.tie_net(B200, B=3, T=12, decay=0.25)
        if user:
            old = net.layers["P"]
            from test_scripted_tier import MyLIF   # a user-defined population: the network runs on the scripted tier

            P = MyLIF(None, shape=[3, 4, 4], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=0)
            net.layers["P"] = P
            net.add_layer(P, "P")
            conn = net.connections[("X", "P")]
            conn.target = P
            net.monitors["Ps"].obj = P
            assert old is not P
        return net, inputs, T

    outs = []
    for user, backend in ((True, emu.EmuBackend), (True, MaxPoolOracleBackend), (False, emu.EmuBackend)):
        net, inputs, T = build(user)
        assert net._scripted_required() == user
        with backend():
            net.run(inputs=inputs, time=T, one_step=one_step)
        outs.append(mn.state(net))
    for o in outs[1:]:
        for k in outs[0]:
            assert torch.equal(outs[0][k].float(), o[k].float()), k
    assert outs[0]["Ps"].sum() > 0


# ---- 3. the standalone compute ---------------------------------------------------------------------------------------

def _restated(fr, s, decay, k, st, p, d):
    """topology.py:1163-1185 in torch, on float32 CPU tensors."""
    fr = fr - decay * fr
    fr = fr + s.float()
    _, idx = F.max_pool2d(fr, kernel_size=k, stride=st, padding=p, dilation=d, return_indices=True)
    return fr, s.flatten(2).gather(2, idx.flatten(2)).view_as(idx).float()


@pytest.mark.parametrize("geom", list(mn.GEOMS))
def test_standalone_compute_matches_max_pool2d(geom):
    import emu

    k, st, p, d = mn.GEOMS[geom]
    g = torch.Generator().manual_seed(3)
    C_, H, W, B = 3, 9, 10, 5
    X = B200.nodes.Input(shape=[C_, H, W])
    X.set_batch_size(B)
    P = B200.nodes.LIFNodes(shape=list(mn.pooled_shape(C_, H, W, geom)))
    conn = B200.topology.MaxPool2dConnection(X, P, kernel_size=k, stride=st, padding=p, dilation=d, decay=0.3)
    assert conn.firing_rates.shape == (B, C_, H, W)
    fr = conn.firing_rates.clone()
    with emu.EmuBackend():
        for step in range(6):
            s = torch.rand(B, C_, H, W, generator=g) < 0.4
            out = conn.compute(s)
            fr, ref = _restated(fr, s, 0.3, k, st, p, d)
            assert torch.equal(conn.firing_rates, fr), step
            assert torch.equal(out, ref), step


# ---- 4. refusals -----------------------------------------------------------------------------------------------------

def _pool_net(ns, B=2, src_shape=(2, 6, 6), tgt_shape=(2, 3, 3), learning=False, **kw):
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=list(src_shape))
    P = ns.nodes.LIFNodes(shape=list(tgt_shape))
    net.add_layer(X, "X"); net.add_layer(P, "P")
    kw.setdefault("decay", 0.5)
    net.add_connection(ns.topology.MaxPool2dConnection(X, P, kernel_size=2, stride=2, **kw), "X", "P")
    x = (torch.rand(4, B, *src_shape, generator=torch.Generator().manual_seed(1)) < 0.3).to(torch.uint8)
    return net, {"X": x}


def _reference():
    """The live reference where build() copied it (oracle/_ref), else None: our side of a check runs either way."""
    try:
        return cases.namespace("reference")
    except ImportError:
        return None


def _raises_like_reference(build, exc):
    """The reference raises ``exc`` for this network, and so does ours (before anything runs)."""
    import emu

    ref = _reference()
    if ref is not None:
        net, inputs = build(ref)
        with pytest.raises(exc):
            net.run(inputs=inputs, time=4)
    net, inputs = build(B200)
    with emu.EmuBackend(), pytest.raises(exc):
        net.run(inputs=inputs, time=4)


def test_decay_none_raises_type_error():
    _raises_like_reference(lambda ns: _pool_net(ns, decay=None), TypeError)


def _squeeze_c1(ns):
    return _pool_net(ns, B=3, src_shape=(1, 6, 6), tgt_shape=(1, 3, 3))


def _squeeze_h1(ns):
    net = ns.Network(dt=1.0, batch_size=3, learning=False)
    X, P = ns.nodes.Input(shape=[2, 1, 6]), ns.nodes.LIFNodes(shape=[2, 1, 3])
    net.add_layer(X, "X"); net.add_layer(P, "P")
    net.add_connection(ns.topology.MaxPool2dConnection(X, P, kernel_size=(1, 2), stride=(1, 2), decay=0.5), "X", "P")
    return net, {"X": (torch.rand(4, 3, 2, 1, 6) < 0.3).to(torch.uint8)}


@pytest.mark.parametrize("build", [_squeeze_c1, _squeeze_h1])
def test_squeeze_quirk_shapes_raise(build):
    """fr += s.float().squeeze() drops a size-1 channel / row dimension of s at B > 1 but not of the buffer."""
    _raises_like_reference(build, RuntimeError)


def test_batch_one_size_one_dims_run():
    """At B = 1 the squeeze only drops the batch dimension: the reference runs, and so do we."""
    import emu
    from maxpool_oracle import MaxPoolOracleBackend

    outs = []
    for backend in (emu.EmuBackend, MaxPoolOracleBackend):
        net, inputs = _pool_net(B200, B=1, src_shape=(1, 6, 6), tgt_shape=(1, 3, 3))
        with backend():
            net.run(inputs=inputs, time=4)
        outs.append(net.connections[("X", "P")].firing_rates.clone())
    assert torch.equal(*outs) and outs[0].sum() > 0


def test_batch_change_without_reset_raises():
    """The buffer keeps the batch size of construction until reset_state_variables()."""
    def build(ns):
        net, inputs = _pool_net(ns, B=1)
        return net, {"X": (torch.rand(4, 3, 2, 6, 6) < 0.3).to(torch.uint8)}

    _raises_like_reference(build, RuntimeError)


def test_window_in_the_padding_raises():
    """Dilation 3 with padding 1 over two rows: the only window's rows are -1 and 2, both outside the image."""
    def build(ns):
        net = ns.Network(dt=1.0, batch_size=2, learning=False)
        X, P = ns.nodes.Input(shape=[2, 2, 6]), ns.nodes.LIFNodes(shape=[2, 1, 6])
        net.add_layer(X, "X"); net.add_layer(P, "P")
        net.add_connection(ns.topology.MaxPool2dConnection(X, P, kernel_size=(2, 1), padding=(1, 0), dilation=(3, 1), decay=0.5),
                           "X", "P")
        return net, {"X": (torch.rand(4, 2, 2, 2, 6) < 0.5).to(torch.uint8)}

    _raises_like_reference(build, RuntimeError)
    with pytest.raises(RuntimeError, match="padding"):
        B200.topology.pool_out_shape(build(B200)[0].connections[("X", "P")])


def test_source_not_chw_raises():
    def build(ns):
        net = ns.Network(dt=1.0, batch_size=2, learning=False)
        X, P = ns.nodes.Input(shape=[6, 6]), ns.nodes.LIFNodes(shape=[3, 3])
        net.add_layer(X, "X"); net.add_layer(P, "P")
        net.add_connection(ns.topology.MaxPool2dConnection(X, P, kernel_size=2, stride=2, decay=0.5), "X", "P")
        return net, {"X": (torch.rand(4, 2, 6, 6) < 0.5).to(torch.uint8)}

    _raises_like_reference(build, RuntimeError)


def test_wrong_target_shape_raises():
    _raises_like_reference(lambda ns: _pool_net(ns, tgt_shape=(2, 9)), RuntimeError)


def test_learning_window_raises_attribute_error():
    _raises_like_reference(lambda ns: _pool_net(ns, learning=True), AttributeError)


def test_masks_raise_attribute_error():
    import emu

    for ns in (_reference(), B200):
        if ns is None:
            continue
        net, inputs = _pool_net(ns)
        ctx = emu.EmuBackend() if ns is B200 else torch.no_grad()
        with ctx, pytest.raises(AttributeError):
            net.run(inputs=inputs, time=4, masks={("X", "P"): torch.zeros(2, 2, dtype=torch.bool)})


@pytest.mark.parametrize("rule", ["PostPre", "Hebbian", "WeightDependentPostPre"])
def test_other_rules_refused(rule):
    for ns in (_reference(), B200):
        if ns is None:
            continue
        X, P = ns.nodes.Input(shape=[2, 6, 6], traces=True), ns.nodes.LIFNodes(shape=[2, 3, 3], traces=True)
        with pytest.raises(NotImplementedError, match="not supported for this Connection type"):
            ns.topology.MaxPool2dConnection(X, P, kernel_size=2, stride=2, decay=0.5, update_rule=getattr(ns.learning, rule),
                                            wmin=0.0, wmax=1.0)


def test_geometry_errors_raise_runtime_error():
    _raises_like_reference(lambda ns: _pool_net(ns, src_shape=(2, 6, 6), tgt_shape=(2, 3, 3), padding=2), RuntimeError)


def test_one_and_three_dimensional_pooling_refused():
    X, P = B200.nodes.Input(shape=[2, 6]), B200.nodes.LIFNodes(shape=[2, 3])
    for cls in (B200.topology.MaxPool1dConnection, B200.topology.MaxPoo3dConnection):
        with pytest.raises(NotImplementedError):
            cls(X, P, kernel_size=2, decay=0.5)


def test_mixed_with_sparse_or_features_refused():
    import emu

    F_, _ = __import__("mcc_feature_nets").features(B200)
    for extra in ("sparse", "feature"):
        net, inputs = _pool_net(B200)
        Y = B200.nodes.LIFNodes(5)
        net.add_layer(Y, "Y")
        if extra == "sparse":
            c = B200.topology.SparseConnection(net.layers["P"], Y, w=torch.rand(18, 5))
        else:
            c = B200.topology.MulticompartmentConnection(net.layers["P"], Y, pipeline=[F_.Mask("m", torch.rand(18, 5) < 0.5),
                                                                                       F_.Weight("w", torch.rand(18, 5))])
        net.add_connection(c, "P", "Y")
        with emu.EmuBackend(), pytest.raises(NotImplementedError, match="MaxPool2dConnection"):
            net.run(inputs=inputs, time=4)


def test_construction_attributes_match_reference():
    for ns in (_reference(), B200):
        if ns is None:
            continue
        X, P = ns.nodes.Input(shape=[2, 6, 6]), ns.nodes.LIFNodes(shape=[2, 3, 3])
        c = ns.topology.MaxPool2dConnection(X, P, kernel_size=2, stride=(2, 2), padding=0, dilation=1, decay=0.5)
        assert (c.kernel_size, c.stride, c.padding, c.dilation, c.decay) == ((2, 2), (2, 2), (0, 0), (1, 1), 0.5)
        assert c.firing_rates.numel() == 0                       # source not added to a network yet
        c.normalize()
        with pytest.raises(TypeError):                           # nu is passed positionally by the constructor
            ns.topology.MaxPool2dConnection(X, P, kernel_size=2, decay=0.5, nu=1e-2)


# ---- 5. tier selection -----------------------------------------------------------------------------------------------

def test_tier_selection():
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    net, inputs = _pool_net(B200, B=2)

    def tier(force):
        plan, keep = _plan.build_net(net, 2, {}, {}, {}, {}, {})
        opts = _abi.SnnRunOpts()
        opts.T, opts.B, opts.tier = 4, 2, force
        return int(emu.lib().snn_b200_select_tier(C.byref(plan), C.byref(opts)))

    assert tier(0) == 1 and tier(1) == 1 and tier(2) == 0 and tier(3) == 0
    net.force_tier = 2
    with emu.EmuBackend(), pytest.raises(RuntimeError, match="not implemented"):
        net.run(inputs=inputs, time=4)
    net.force_tier = 0
    with emu.EmuBackend():
        net.run(inputs=inputs, time=4)
    assert emu.last_tier == 1


# ---- 6. the reference's own objects through the ABI -----------------------------------------------------------------

def test_reference_binding_runs_the_references_network():
    """bindsnet_b200.reference_binding fills the plan from a live reference network with a MaxPool2dConnection; the
    pooling oracle library then computes what the reference's own run computes."""
    ref = _reference()
    if ref is None:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb
    import maxpool_oracle

    twins = [mn.tie_net(ref, B=3, T=12, decay=0.25) for _ in range(2)]
    (a, inputs, T), (b, _, _) = twins
    a.run(inputs={"X": inputs["X"].clone()}, time=T)
    assert rb.run_window(b, {"X": inputs["X"].clone()}, time=T, library=maxpool_oracle.lib()) == 0
    sa, sb = mn.state(a), mn.state(b)
    for k in ("XP/fr", "P/s", "P/v", "P/refrac_count"):
        assert torch.equal(sa[k], sb[k]), k
    assert sa["P/s"].sum() > 0


class _NoRun:
    """A library stand-in whose window entry point must never be reached."""

    @property
    def snn_oracle_run_window(self):
        raise AssertionError("the plan was executed")


def test_reference_binding_checks_the_rates_buffer():
    """A reference network built at batch size 1 and bound for a run at B = 4: the reference never resizes firing_rates
    (its own run raises RuntimeError), so the binding refuses the plan before anything reads or writes the buffer.  So it
    does for a buffer on another device and for a learning window."""
    ref = _reference()
    if ref is None:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb

    net, inputs = _pool_net(ref, B=1)
    x4 = (torch.rand(4, 4, 2, 6, 6, generator=torch.Generator().manual_seed(2)) < 0.3).to(torch.uint8)
    with pytest.raises(RuntimeError):
        net.run(inputs={"X": x4.clone()}, time=4)
    net, inputs = _pool_net(ref, B=1)
    fr = net.connections[("X", "P")].firing_rates
    with pytest.raises(RuntimeError, match="firing_rates"):
        rb.run_window(net, {"X": x4}, time=4, library=_NoRun())
    assert tuple(fr.shape) == (1, 2, 6, 6) and not fr.any()

    net, inputs = _pool_net(ref, B=2)
    conn = net.connections[("X", "P")]
    conn.firing_rates = conn.firing_rates.to("meta")
    with pytest.raises(RuntimeError, match="device"):
        rb.run_window(net, inputs, time=4, library=_NoRun())

    net, inputs = _pool_net(ref, B=2, learning=True)
    with pytest.raises(AttributeError):
        rb.run_window(net, inputs, time=4, library=_NoRun())


def test_abi_v13_pooling_fields_match_the_header():
    import re

    from bindsnet_b200 import _abi

    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "snn_b200.h")).read()
    assert int(re.search(r"#define\s+SNN_ABI_VERSION\s+(\d+)", header).group(1)) == _abi.SNN_ABI_VERSION == 13
    assert int(re.search(r"#define\s+SNN_CONN_MAXPOOL2D\s+(\d+)", header).group(1)) == _abi.SNN_CONN_MAXPOOL2D
    body = header[header.index("typedef struct snn_conn"):header.index("} snn_conn_t;")]
    assert re.search(r"float \*pool_rates;\s*float pool_decay;\s*$", body)
    assert [f[0] for f in _abi.SnnConn._fields_][-2:] == ["pool_rates", "pool_decay"]
