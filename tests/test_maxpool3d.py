"""MaxPoo3dConnection (reference: topology.py:1214-1301) on the generic window kernel.  CPU tests: the oracle
(tests/maxpool3d_oracle.c, the CPU oracle extended by Conv3dConnection and the 3-D pooling connection) against the live
reference's stored results, the emulated kernel against the oracle bit for bit, a degenerate-depth pool against its
MaxPool2dConnection twin, the standalone compute against F.max_pool3d, refusals and tier selection.  The stored
reference results are regenerated with ``python tests/golden/gen_live.py test_maxpool3d``."""
import ctypes as C
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import cases
import maxpool3d_nets as mn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")
TIE_DECAYS = [0.0, 1.0]
VARIANTS = {"one_spike_source": dict(one_spike=True), "target_first": dict(target_first=True),
            "one_spike_target_first": dict(one_spike=True, target_first=True)}


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
def _live_one_spike(ns, _):
    net, inputs, T = mn.one_spike_net(ns)
    return _flat(mn.run_two_windows(net, inputs, T))


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
    from maxpool3d_oracle import MaxPool3dOracleBackend

    net, inputs, T = mn.conv_pool_net(B200, case)
    with MaxPool3dOracleBackend() as ob:
        ours = _flat(mn.run_two_windows(net, inputs, T))
    assert ob.err == 0
    _check_against(load(_live_conv_pool, case), ours, case)
    assert ours["w1/Ps"].sum() > 0 and ours["w1/Ys"].sum() > 0


@pytest.mark.parametrize("decay", TIE_DECAYS)
def test_oracle_ties_match_live_reference(decay):
    from maxpool3d_oracle import MaxPool3dOracleBackend

    net, inputs, T = mn.tie_net(B200, decay=decay)
    with MaxPool3dOracleBackend():
        ours = _flat(mn.run_two_windows(net, inputs, T))
    _check_against(load(_live_ties, decay), ours, f"ties decay={decay}")
    # the case is built to tie: in most windows of the last step some two of the eight elements have the same rate
    fr = ours["w1/XP/fr"].view(4, 3, 2, 2, 2, 2, 2, 2).permute(0, 1, 2, 4, 6, 3, 5, 7).reshape(4, 3, 8, 8)
    ties = (fr.unsqueeze(-1) == fr.unsqueeze(-2)).sum((-1, -2)) > 8
    assert ties.float().mean() > 0.5


def test_one_spike_source_matches_live_reference():
    """A DiehlAndCookNodes(one_spike) source whose winner is the only candidate (mn.one_spike_net)."""
    from maxpool3d_oracle import MaxPool3dOracleBackend

    net, inputs, T = mn.one_spike_net(B200)
    with MaxPool3dOracleBackend():
        ours = _flat(mn.run_two_windows(net, inputs, T))
    _check_against(load(_live_one_spike, 0), ours, "one_spike source")
    assert ours["w1/Ss"].sum() > 0 and ours["w1/Ps"].sum() > 0


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _with_env(env, fn):
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        return fn()
    finally:
        for k, v in old.items():
            os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)


def _emu_vs_oracle(build, env=None, **kw):
    import emu
    from maxpool3d_oracle import MaxPool3dOracleBackend

    outs = []
    for backend in (emu.EmuBackend, MaxPool3dOracleBackend):
        net, inputs, T = build()
        net.force_tier = 1

        def run():
            with backend() as be:
                outs.append(_flat(mn.run_two_windows(net, inputs, T, **kw)))
            assert be.err == 0

        _with_env(env if backend is emu.EmuBackend else None, run)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
    a, b = outs
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), f"{k} differs"
    return a


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["b4_c2_d0.25_k3s1", "b1_c1_d0_k3s2p1", "b4_c2_d1_d112", "b2_c3_d0.25_k233s2p1d112"])
def test_emulated_kernel_bit_exact(case, env):
    a = _emu_vs_oracle(lambda: mn.conv_pool_net(B200, case), ENVS[env])
    assert a["w1/Ps"].sum() > 0


@pytest.mark.parametrize("case", ["b1_c2_d0.25_k2s2", "b4_c2_d0.25_d211", "b4_c2_d0.25_k123s121"])
def test_emulated_kernel_one_step_bit_exact(case):
    _emu_vs_oracle(lambda: mn.conv_pool_net(B200, case), ENVS["sms3"], one_step=True)


@pytest.mark.parametrize("decay", TIE_DECAYS)
def test_emulated_kernel_ties_bit_exact(decay):
    _emu_vs_oracle(lambda: mn.tie_net(B200, decay=decay), ENVS["sms7"])
    _emu_vs_oracle(lambda: mn.tie_net(B200, decay=decay), ENVS["sms3"], one_step=True)


@pytest.mark.parametrize("B,T", [(3, 7), (33, 6), (520, 5)])
def test_emulated_kernel_batch_sizes_bit_exact(B, T):
    """B = 3, 33 and 520, odd and even window lengths (the rates' slot parity)."""
    a = _emu_vs_oracle(lambda: mn.tie_net(B200, B=B, T=T, decay=0.25), ENVS["sms3"])
    assert a["w1/Ps"].sum() > 0


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
    """A Monitor on firing_rates runs the window step by step (one-step windows): the same state as the whole window."""
    import emu

    outs = []
    for stepwise in (True, False):
        net, inputs, T = mn.conv_pool_net(B200, "b4_c2_d0.25_k3s2p1", T=10)
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
    from maxpool3d_oracle import MaxPool3dOracleBackend

    def build(user):
        net, inputs, T = mn.tie_net(B200, B=3, T=12, decay=0.25)
        if user:
            from test_scripted_tier import MyLIF   # a user-defined population: the network runs on the scripted tier

            P = MyLIF(None, shape=[3, 2, 2, 2], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=0)
            net.add_layer(P, "P")
            net.connections[("X", "P")].target = P
            net.monitors["Ps"].obj = P
        return net, inputs, T

    outs = []
    for user, backend in ((True, emu.EmuBackend), (True, MaxPool3dOracleBackend), (False, emu.EmuBackend)):
        net, inputs, T = build(user)
        assert net._scripted_required() == user
        with backend():
            net.run(inputs=inputs, time=T, one_step=one_step)
        outs.append(mn.state(net))
    for o in outs[1:]:
        for k in outs[0]:
            assert torch.equal(outs[0][k].float(), o[k].float()), k
    assert outs[0]["Ps"].sum() > 0


# ---- 3. the degenerate-depth twin of a MaxPool2dConnection -----------------------------------------------------------

def _twin_states(backend_cls, one_spike, one_step=False):
    from maxpool_nets import run_two_windows   # the twin's input is [2 windows, T, B, 2, H, W]

    outs = []
    for three_d in (True, False):
        net, inputs, T = mn.twin_net(B200, three_d, one_spike=one_spike)
        with backend_cls():
            outs.append(_flat(run_two_windows(net, inputs, T, one_step=one_step, one_spike_seed=3)))
    return outs


@pytest.mark.parametrize("one_step", [False, True])
@pytest.mark.parametrize("one_spike", [False, True])
def test_twin_of_max_pool_2d_bit_identical(one_spike, one_step):
    """A [1, 1, H, W] source pooled with kernel (1, kh, kw) computes what the MaxPool2dConnection on [1, H, W] computes."""
    import emu

    a, b = _twin_states(emu.EmuBackend, one_spike, one_step)
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k].flatten(), b[k].flatten()), k
    assert a["w1/Ps"].sum() > 0


# ---- 4. the standalone compute ---------------------------------------------------------------------------------------

def _restated(fr, s, decay, k, st, p, d):
    """topology.py:1255-1277 in torch, on float32 CPU tensors."""
    fr = fr - decay * fr
    fr = fr + s.float()
    _, idx = F.max_pool3d(fr, kernel_size=k, stride=st, padding=p, dilation=d, return_indices=True)
    return fr, s.flatten(2).gather(2, idx.flatten(2)).view_as(idx).float()


@pytest.mark.parametrize("geom", list(mn.GEOMS))
def test_standalone_compute_matches_max_pool3d(geom):
    import emu

    kw = mn.pool_kwargs(geom)
    vol = mn.GEOMS[geom][4]
    g = torch.Generator().manual_seed(3)
    C_, B = 3, 5
    X = B200.nodes.Input(shape=[C_, *vol])
    X.set_batch_size(B)
    P = B200.nodes.LIFNodes(shape=list(mn.pooled_shape(C_, vol, geom)))
    conn = B200.topology.MaxPoo3dConnection(X, P, decay=0.3, **kw)
    assert conn.firing_rates.shape == (B, C_, *vol)
    fr = conn.firing_rates.clone()
    with emu.EmuBackend():
        for step in range(5):
            s = torch.rand(B, C_, *vol, generator=g) < 0.4
            out = conn.compute(s)
            fr, ref = _restated(fr, s, 0.3, kw["kernel_size"], kw["stride"], kw["padding"], kw["dilation"])
            assert torch.equal(conn.firing_rates, fr), step
            assert torch.equal(out, ref), step


def test_oracle_compute_matches_max_pool3d():
    from bindsnet_b200.network import _plan
    import maxpool3d_oracle

    geom = "k233s2p1d112"
    kw, vol = mn.pool_kwargs(geom), mn.GEOMS[geom][4]
    X = B200.nodes.Input(shape=[2, *vol])
    X.set_batch_size(3)
    P = B200.nodes.LIFNodes(shape=list(mn.pooled_shape(2, vol, geom)))
    conn = B200.topology.MaxPoo3dConnection(X, P, decay=0.5, **kw)
    s = torch.rand(3, 2, *vol, generator=torch.Generator().manual_seed(4)) < 0.5
    fr, ref = _restated(conn.firing_rates.clone(), s, 0.5, kw["kernel_size"], kw["stride"], kw["padding"], kw["dilation"])
    d = _plan._conn_desc(conn, 3)
    out = torch.empty(3, P.n)
    su8 = s.to(torch.uint8).reshape(3, -1).contiguous()
    assert maxpool3d_oracle.lib().snn_oracle_conn_compute(C.byref(d), X.n, P.n, 3, su8.data_ptr(), out.data_ptr()) == 0
    assert torch.equal(conn.firing_rates, fr) and torch.equal(out.view_as(ref), ref)


# ---- 5. refusals -----------------------------------------------------------------------------------------------------

def _pool_net(ns, B=2, src_shape=(2, 4, 6, 6), tgt_shape=(2, 2, 3, 3), learning=False, **kw):
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=list(src_shape))
    P = ns.nodes.LIFNodes(shape=list(tgt_shape))
    net.add_layer(X, "X"); net.add_layer(P, "P")
    kw.setdefault("decay", 0.5)
    kw.setdefault("kernel_size", 2)
    kw.setdefault("stride", 2)
    net.add_connection(ns.topology.MaxPoo3dConnection(X, P, **kw), "X", "P")
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


@pytest.mark.parametrize("src,tgt", [((1, 4, 6, 6), (1, 2, 3, 3)), ((2, 1, 6, 6), (2, 1, 3, 3))])
def test_squeeze_quirk_shapes_raise(src, tgt):
    """fr += s.float().squeeze() drops a size-1 channel / depth dimension of s at B > 1 but not of the buffer."""
    kw = dict(kernel_size=(1, 2, 2), stride=(1, 2, 2)) if src[1] == 1 else {}
    _raises_like_reference(lambda ns: _pool_net(ns, B=4, src_shape=src, tgt_shape=tgt, **kw), RuntimeError)


def test_batch_one_size_one_dims_run():
    """At B = 1 the squeeze only drops the batch dimension: the reference runs, and so do we."""
    import emu
    from maxpool3d_oracle import MaxPool3dOracleBackend

    outs = []
    for backend in (emu.EmuBackend, MaxPool3dOracleBackend):
        net, inputs = _pool_net(B200, B=1, src_shape=(1, 4, 6, 6), tgt_shape=(1, 2, 3, 3))
        with backend():
            net.run(inputs=inputs, time=4)
        outs.append(net.connections[("X", "P")].firing_rates.clone())
    assert torch.equal(*outs) and outs[0].sum() > 0


def test_batch_change_without_reset_raises():
    def build(ns):
        net, inputs = _pool_net(ns, B=1)
        return net, {"X": (torch.rand(4, 3, 2, 4, 6, 6) < 0.3).to(torch.uint8)}

    _raises_like_reference(build, RuntimeError)


def test_wrong_target_shape_raises():
    _raises_like_reference(lambda ns: _pool_net(ns, tgt_shape=(2, 18)), RuntimeError)


@pytest.mark.parametrize("padding", [(2, 0, 0), (0, 2, 0), (0, 0, 2)])
def test_padding_above_half_the_kernel_raises(padding):
    _raises_like_reference(lambda ns: _pool_net(ns, tgt_shape=(2, 3, 3, 3), padding=padding), RuntimeError)


def test_window_in_the_padding_raises():
    """Depth dilation 3 with padding 1 over two planes: the only window's planes are -1 and 2, both outside the volume."""
    def build(ns):
        return _pool_net(ns, src_shape=(2, 2, 4, 4), tgt_shape=(2, 1, 4, 4), kernel_size=(2, 1, 1), stride=1, padding=(1, 0, 0),
                         dilation=(3, 1, 1))

    _raises_like_reference(build, RuntimeError)
    with pytest.raises(RuntimeError, match="padding"):
        B200.topology.pool_out_shape(build(B200)[0].connections[("X", "P")])


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
        X, P = ns.nodes.Input(shape=[2, 4, 6, 6], traces=True), ns.nodes.LIFNodes(shape=[2, 2, 3, 3], traces=True)
        with pytest.raises(NotImplementedError, match="not supported for this Connection type"):
            ns.topology.MaxPoo3dConnection(X, P, kernel_size=2, stride=2, decay=0.5, update_rule=getattr(ns.learning, rule),
                                           wmin=0.0, wmax=1.0)


@pytest.mark.parametrize("shape", [[2, 6], [2, 6, 6], [1, 2, 4, 6, 6]])
def test_non_four_dimensional_source_refused(shape):
    """A deliberate difference from the reference: a source that is not [C, D, H, W] is refused at construction."""
    X, P = B200.nodes.Input(shape=shape), B200.nodes.LIFNodes(shape=[2, 3])
    with pytest.raises(NotImplementedError, match=r"\[C, D, H, W\]"):
        B200.topology.MaxPoo3dConnection(X, P, kernel_size=2, decay=0.5)


def test_one_dimensional_kinds_stay_refused():
    X, P = B200.nodes.Input(shape=[2, 6]), B200.nodes.LIFNodes(shape=[2, 3])
    for cls in (B200.topology.MaxPool1dConnection, B200.topology.LocalConnection1D):
        with pytest.raises(NotImplementedError):
            cls(X, P, 2)


def test_mixed_with_sparse_features_or_neuron_tensors_refused():
    import emu

    F_, _ = __import__("mcc_feature_nets").features(B200)
    for extra in ("sparse", "feature"):
        net, inputs = _pool_net(B200)
        Y = B200.nodes.LIFNodes(5)
        net.add_layer(Y, "Y")
        if extra == "sparse":
            c = B200.topology.SparseConnection(net.layers["P"], Y, w=torch.rand(36, 5))
        else:
            c = B200.topology.MulticompartmentConnection(net.layers["P"], Y, pipeline=[F_.Mask("m", torch.rand(36, 5) < 0.5),
                                                                                       F_.Weight("w", torch.rand(36, 5))])
        net.add_connection(c, "P", "Y")
        with emu.EmuBackend(), pytest.raises(NotImplementedError, match="MaxPoo3dConnection"):
            net.run(inputs=inputs, time=4)
    net = B200.Network(dt=1.0, batch_size=2, learning=False)
    X = B200.nodes.Input(shape=[2, 4, 6, 6])
    P = B200.nodes.LIFNodes(shape=[2, 2, 3, 3], thresh=torch.full((2, 2, 3, 3), -55.0))
    net.add_layer(X, "X"); net.add_layer(P, "P")
    net.add_connection(B200.topology.MaxPoo3dConnection(X, P, kernel_size=2, stride=2, decay=0.5), "X", "P")
    with emu.EmuBackend(), pytest.raises(NotImplementedError, match="MaxPoo3dConnection"):
        net.run(inputs={"X": torch.zeros(4, 2, 2, 4, 6, 6, dtype=torch.uint8)}, time=4)


def test_construction_attributes_match_reference():
    for ns in (_reference(), B200):
        if ns is None:
            continue
        X, P = ns.nodes.Input(shape=[2, 4, 6, 6]), ns.nodes.LIFNodes(shape=[2, 2, 3, 3])
        c = ns.topology.MaxPoo3dConnection(X, P, kernel_size=2, stride=(2, 2, 1), padding=0, dilation=(1, 2, 1), decay=0.5)
        assert (c.kernel_size, c.stride, c.padding, c.dilation, c.decay) == ((2, 2, 2), (2, 2, 1), (0, 0, 0), (1, 2, 1), 0.5)
        assert c.firing_rates.numel() == 0                       # source not added to a network yet
        c.normalize()


def test_reset_keeps_the_buffer_on_its_device():
    net, _ = _pool_net(B200, B=3)
    conn = net.connections[("X", "P")]
    conn.firing_rates = conn.firing_rates.to("meta")
    conn.reset_state_variables()
    assert conn.firing_rates.device.type == "meta" and tuple(conn.firing_rates.shape) == (3, 2, 4, 6, 6)


def test_not_a_learned_connection_of_the_multi_gpu_runner():
    from bindsnet_b200.distributed import ShardedWindowRunner

    net, _ = _pool_net(B200)
    assert ShardedWindowRunner(net)._learned() == []


# ---- 6. tier selection and the library's own checks ------------------------------------------------------------------

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


def test_library_refuses_bad_plans():
    """The library's own checks on the depth fields and the rest of the kind's contract."""
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    net, _ = _pool_net(B200, B=2)
    m = torch.zeros(1, dtype=torch.uint8)
    bad = (("din", 5), ("dout", 3), ("kd", 0), ("sd", 0), ("pd", 2), ("pd", -1), ("dd", 0), ("dd", 4), ("cout", 1),
           ("w", m.data_ptr()), ("b", m.data_ptr()), ("pool_rates", None))
    for field, value in bad:
        plan, keep = _plan.build_net(net, 2, {}, {}, {}, {}, {})
        setattr(plan.conns[0], field, value)
        opts = _abi.SnnRunOpts()
        opts.T, opts.B = 4, 2
        assert int(emu.lib().snn_b200_workspace_bytes(C.byref(plan), C.byref(opts))) == 0, field
        assert int(emu.lib().snn_b200_run_window(C.byref(plan), C.byref(opts), None, 0, None)) == _abi.SNN_ERR_BAD_ARG, field
    for field, value in (("mask", m.data_ptr()), ("rule", _abi.SNN_RULE_POSTPRE), ("has_norm", 1)):
        plan, keep = _plan.build_net(net, 2, {}, {}, {}, {}, {})
        setattr(plan.conns[0], field, value)
        opts = _abi.SnnRunOpts()
        opts.T, opts.B = 4, 2
        assert int(emu.lib().snn_b200_run_window(C.byref(plan), C.byref(opts), None, 0, None)) == _abi.SNN_ERR_UNSUPPORTED, field


def test_abi_fields_match_the_header():
    import re

    from bindsnet_b200 import _abi

    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "snn_b200.h")).read()
    assert int(re.search(r"#define\s+SNN_ABI_VERSION\s+(\d+)", header).group(1)) == _abi.SNN_ABI_VERSION == 13
    assert int(re.search(r"#define\s+SNN_CONN_MAXPOOL3D\s+(\d+)", header).group(1)) == _abi.SNN_CONN_MAXPOOL3D == 9
    assert re.search(r"int32_t din, dout, kd, sd, pd, dd;", header)
    assert [f[0] for f in _abi._Conv3dFields._fields_] == ["din", "dout", "kd", "sd", "pd", "dd"]
    assert C.sizeof(_abi.SnnConn) == 320 and _abi.SnnConn.pool_rates.offset == 304


# ---- 7. the reference's own objects through the ABI -----------------------------------------------------------------

def test_reference_binding_runs_the_references_network():
    """bindsnet_b200.reference_binding fills the plan from a live reference network with a Conv3dConnection and a
    MaxPoo3dConnection; the oracle library then computes what the reference's own run computes."""
    ref = _reference()
    if ref is None:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb
    import maxpool3d_oracle

    case = "b2_c3_d0.25_k233s2p1d112"
    (a, inputs, T), (b, _, _) = mn.conv_pool_net(ref, case), mn.conv_pool_net(ref, case)
    a.run(inputs={"X": inputs["X"][0].clone()}, time=T)
    assert rb.run_window(b, {"X": inputs["X"][0].clone()}, time=T, library=maxpool3d_oracle.lib()) == 0
    sa, sb = mn.state(a), mn.state(b)
    for k in ("C1P/fr", "P/s", "P/v", "P/refrac_count", "Y/s"):
        assert torch.equal(sa[k], sb[k]), k
    assert sa["P/s"].sum() > 0


class _NoRun:
    """A library stand-in whose window entry point must never be reached."""

    @property
    def snn_oracle_run_window(self):
        raise AssertionError("the plan was executed")


def test_reference_binding_checks_the_rates_buffer():
    ref = _reference()
    if ref is None:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb

    net, inputs = _pool_net(ref, B=1)
    x4 = (torch.rand(4, 4, 2, 4, 6, 6, generator=torch.Generator().manual_seed(2)) < 0.3).to(torch.uint8)
    fr = net.connections[("X", "P")].firing_rates
    with pytest.raises(RuntimeError, match="firing_rates"):
        rb.run_window(net, {"X": x4}, time=4, library=_NoRun())
    assert tuple(fr.shape) == (1, 2, 4, 6, 6) and not fr.any()

    net, inputs = _pool_net(ref, B=2)
    conn = net.connections[("X", "P")]
    conn.firing_rates = conn.firing_rates.to("meta")
    with pytest.raises(RuntimeError, match="device"):
        rb.run_window(net, inputs, time=4, library=_NoRun())

    net, inputs = _pool_net(ref, B=2, learning=True)
    with pytest.raises(AttributeError):
        rb.run_window(net, inputs, time=4, library=_NoRun())
