"""LocalConnection2D (reference: topology.py:1623-1767) and its PostPre / WeightDependentPostPre / Hebbian rules on the
generic window kernel.  CPU tests: the oracle (tests/local2d_oracle.c, the CPU oracle extended by the local connection)
against the live reference's stored results, the emulated kernel against the oracle bit for bit, the standalone
operators against a torch restatement, refusals and tier selection.  The stored reference results are regenerated with
``python tests/golden/gen_live.py test_local2d``."""
import ctypes as C
import os
import sys

import pytest
import torch

import cases
import local2d_nets as ln
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")
CASES = list(ln.LIVE_CASES)


def _flat(states):
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


def _reference():
    try:
        return cases.namespace("reference")
    except ImportError:
        return None


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

@reference_side(CASES)
def _live(ns, case):
    net, inputs, T = ln.build_case(ns, case)
    return _flat(ln.run_windows(net, inputs, T, ln.windows_of(case)))


def _check_against(ref, ours, what):
    for k, v in ref.items():
        o = ours[k]
        assert o.shape == v.shape, (what, k)
        if k.endswith("s"):
            assert torch.equal(o.float(), v.float()), f"{what}: {k} differs"
        elif k.endswith("/w"):
            torch.testing.assert_close(o, v, rtol=1e-4, atol=0.0, equal_nan=True, msg=f"{what}: {k}")
        else:
            torch.testing.assert_close(o.float(), v.float(), rtol=1e-5, atol=1e-4, equal_nan=True, msg=f"{what}: {k}")


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_live_reference(case):
    from local2d_oracle import Local2dOracleBackend

    net, inputs, T = ln.build_case(B200, case)
    with Local2dOracleBackend() as ob:
        ours = _flat(ln.run_windows(net, inputs, T, ln.windows_of(case)))
    assert ob.err == 0
    _check_against(load(_live, case), ours, case)
    assert ours["w0/Ys"].sum() > 0
    if ln.LIVE_CASES[case] and ln.LIVE_CASES[case].get("zero_row"):
        assert torch.isnan(ours["w0/XY/w"][1, 7]).all() and not torch.isnan(ours["w0/XY/w"][0]).any()


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _emu_vs_oracle(build, env=None, n=2, **kw):
    import emu
    from local2d_oracle import Local2dOracleBackend

    outs = []
    for backend in (emu.EmuBackend, Local2dOracleBackend):
        net, inputs, T = build()
        old = {k: os.environ.get(k) for k in (env or {})}
        os.environ.update(env if backend is emu.EmuBackend and env else {})
        try:
            with backend() as be:
                outs.append(_flat(ln.run_windows(net, inputs, T, n, **kw)))
            assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
    a, b = outs
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]) or (a[k].is_floating_point() and torch.equal(a[k].isnan(), b[k].isnan())
                                          and torch.equal(a[k].nan_to_num(), b[k].nan_to_num())), f"{k} differs"
    return a


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["example_b1", "c2_PostPre", "c2_WeightDependentPostPre", "c2_Hebbian", "c2_NoOp"])
def test_emulated_kernel_bit_exact(case, env):
    a = _emu_vs_oracle(lambda: ln.build_case(B200, case), ENVS[env])
    assert a["w1/Ys"].sum() > 0


def test_emulated_kernel_zero_row_bit_exact():
    _emu_vs_oracle(lambda: ln.build_case(B200, "c2_zero_row"), ENVS["sms3"], n=1)


@pytest.mark.parametrize("rule", ["PostPre", "Hebbian"])
def test_emulated_kernel_one_step_bit_exact(rule):
    _emu_vs_oracle(lambda: ln.multi_net(B200, rule=rule), ENVS["sms3"], one_step=True)


def test_stepwise_equals_oracle():
    """A monitor on the target's traces makes the window run step by step (one one-step window per step)."""
    def build():
        net, inputs, T = ln.multi_net(B200, rule="WeightDependentPostPre", T=10)
        net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["x"], time=T), "Yx")
        return net, inputs, T

    _emu_vs_oracle(build, ENVS["sms3"])


@pytest.mark.parametrize("T", [7, 8])
def test_emulated_kernel_large_batch_bit_exact(T):
    """B = 520 and an odd and an even window length."""
    a = _emu_vs_oracle(lambda: ln.multi_net(B200, rule="PostPre", B=520, T=T), ENVS["sms3"])
    assert a["w1/Ys"].sum() > 0


def test_tiles_straddle_filters():
    """P = 15 target positions per filter: the 32-neuron tiles of the target start inside filters, and 7 SMs spread the
    learning phase's elements over many CTAs."""
    _emu_vs_oracle(lambda: ln.multi_net(B200, rule="Hebbian", B=3, T=9), ENVS["sms7"])


def test_scripted_tier_equals_window():
    import emu
    from local2d_oracle import Local2dOracleBackend
    from test_scripted_tier import MyLIF

    def build(user):
        net, inputs, T = ln.multi_net(B200, rule="PostPre", B=3, T=12)
        if user:   # a user-defined population as the last layer: the network runs on the scripted tier
            Z = MyLIF(6, traces=True, thresh=-62.0)
            net.layers["Z"] = Z
            net.add_layer(Z, "Z")
            net.connections[("Y", "Z")].target = Z
            net.monitors["Zs"].obj = Z
        return net, inputs, T

    outs = []
    for user, backend in ((True, emu.EmuBackend), (True, Local2dOracleBackend), (False, emu.EmuBackend)):
        net, inputs, T = build(user)
        assert net._scripted_required() == user
        with backend():
            net.run(inputs={"X": inputs["X"][0]}, time=T)
        outs.append(ln.state(net))
    for o in outs[1:]:
        for k in outs[0]:
            assert torch.equal(outs[0][k].float(), o[k].float()), k
    assert outs[0]["Ys"].sum() > 0


def test_nonfinite_weight_under_silent_input():
    """The spike gather never reads the weight of a silent input: an inf there leaves the target's input finite (the
    reference's s_unfold * w makes it NaN; DESIGN.md section 8).  Emulated kernel and oracle agree."""
    import emu

    for backend in (emu.EmuBackend, __import__("local2d_oracle").Local2dOracleBackend):
        X = B200.nodes.Input(shape=[1, 6, 6])
        Y = B200.nodes.LIFNodes(shape=[2, 2, 2])
        net = B200.Network(batch_size=1, learning=False)
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        lc = B200.topology.LocalConnection2D(X, Y, kernel_size=3, stride=3, n_filters=2)
        with torch.no_grad():
            lc.w[0, :, 0] = float("inf")
        net.add_connection(lc, "X", "Y")
        s = torch.ones(1, 1, 6, 6, dtype=torch.bool)
        s[0, 0, ::3, ::3] = False       # the first position of every window is silent
        with backend():
            out = lc.compute(s)
        assert torch.isfinite(out).all()
        torch.testing.assert_close(out.view(-1), lc.w[0, :, 1:].sum(-1), rtol=1e-6, atol=1e-6)


# ---- 3. the standalone operators -------------------------------------------------------------------------------------

def _restated_compute(s, w, k, st, F_):
    """topology.py:1717-1740 in torch: unfold the source, one weight per (channel, target, window position)."""
    B, Cin = s.shape[:2]
    u = s.float().unfold(2, k[0], st[0]).unfold(3, k[1], st[1])              # [B, Cin, Ho, Wo, kh, kw]
    u = u.reshape(B, Cin, -1, k[0] * k[1]).repeat(1, 1, F_, 1)               # [B, Cin, N, K]
    return (u * w).sum(-1).sum(1)


def _restated_update(conn, rule, B):
    """learning.py:258-320 / 717-791 / 1186-1250 in torch: the reshaped unfold, row n' reads row n' % P."""
    k, st, F_ = conn.kernel_size, conn.stride, conn.n_filters
    X, Y = conn.source, conn.target

    def unf(v):
        u = v.float().unfold(2, k[0], st[0]).unfold(3, k[1], st[1])
        return u.reshape(B, conn.conv_prod, -1).repeat(1, F_, 1)             # [B, N, Cin * K]

    pre = (Y.x.reshape(B, -1, 1) * unf(X.s)).sum(0)
    post = (Y.s.float().reshape(B, -1, 1) * unf(X.x)).sum(0)
    w = conn.w.clone().view(pre.shape)
    nu0, nu1 = float(rule.nu[0]), float(rule.nu[1])
    if type(rule).__name__ == "WeightDependentPostPre":
        w = w + (-(nu0 * pre * (w - 0.0)) + nu1 * post * (1.0 - w))
    elif type(rule).__name__ == "Hebbian":
        w = w + nu0 * pre + nu1 * post
    else:
        w = w - nu0 * pre + nu1 * post
    return w.clamp(0.0, 1.0).view(conn.w.shape)


def _pair_layers(B, Cin=2, H=9, W=11):
    X = B200.nodes.Input(shape=[Cin, H, W], traces=True)
    Y = B200.nodes.LIFNodes(shape=[3, 4, 4], traces=True)
    for L in (X, Y):
        L.set_batch_size(B)
        L.compute_decays(1.0)
    return X, Y


@pytest.mark.parametrize("rule", ["PostPre", "WeightDependentPostPre", "Hebbian"])
def test_standalone_operators_match_torch(rule):
    import emu

    g = torch.Generator().manual_seed(21)
    B = 3
    X, Y = _pair_layers(B)
    conn = B200.topology.LocalConnection2D(X, Y, kernel_size=(3, 2), stride=(2, 3), n_filters=3, nu=(0.01, 0.02), wmin=0.0, wmax=1.0,
                                           norm=2.0, reduction=torch.sum, update_rule=getattr(B200.learning, rule))
    assert conn.w.shape == (2, 48, 6) and conn.conv_size == (4, 4)
    with emu.EmuBackend():
        for step in range(3):
            s = torch.rand(B, 2, 9, 11, generator=g) < 0.4
            out = conn.compute(s)
            torch.testing.assert_close(out.view(B, -1), _restated_compute(s, conn.w, conn.kernel_size, conn.stride, 3), rtol=1e-5, atol=1e-5)
            X.s = s.clone()
            X.x = torch.rand(B, 2, 9, 11, generator=g)
            Y.s = torch.rand(B, 3, 4, 4, generator=g) < 0.3
            Y.x = torch.rand(B, 3, 4, 4, generator=g)
            ref = _restated_update(conn, conn.update_rule, B)
            conn.update_rule.update()
            torch.testing.assert_close(conn.w, ref, rtol=1e-5, atol=1e-6)
        conn.normalize()
    rows = conn.w.view(-1, 6).sum(-1)
    torch.testing.assert_close(rows, torch.full_like(rows, 2.0), rtol=1e-5, atol=1e-5)


# ---- 4. refusals and errors ------------------------------------------------------------------------------------------

def _lc_net(ns, B=2, tgt_shape=(2, 2, 2), learning=False, rule=None, **kw):
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=[1, 6, 6], traces=True)
    Y = ns.nodes.LIFNodes(shape=list(tgt_shape), traces=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    if rule is not None:
        kw["update_rule"] = getattr(ns.learning, rule)
    net.add_connection(ns.topology.LocalConnection2D(X, Y, kernel_size=3, stride=3, n_filters=2, **kw), "X", "Y")
    return net, {"X": (torch.rand(4, B, 1, 6, 6, generator=torch.Generator().manual_seed(1)) < 0.3).to(torch.uint8)}


def _raises_like_reference(build, exc):
    import emu

    ref = _reference()
    if ref is not None:
        with pytest.raises(exc):
            net, inputs = build(ref)
            net.run(inputs=inputs, time=4)
    with emu.EmuBackend(), pytest.raises(exc):
        net, inputs = build(B200)
        net.run(inputs=inputs, time=4)


def test_w_kwarg_raises_attribute_error():
    _raises_like_reference(lambda ns: _lc_net(ns, w=torch.rand(1, 8, 9)), AttributeError)


def test_wrong_target_size_raises_runtime_error():
    _raises_like_reference(lambda ns: _lc_net(ns, tgt_shape=(3, 2, 2)), RuntimeError)


def test_kernel_larger_than_source_raises_runtime_error():
    def build(ns):
        net = ns.Network(dt=1.0, batch_size=1, learning=False)
        X, Y = ns.nodes.Input(shape=[1, 4, 4]), ns.nodes.LIFNodes(shape=[2, 0, 0])
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        net.add_connection(ns.topology.LocalConnection2D(X, Y, kernel_size=5, stride=1, n_filters=2), "X", "Y")
        return net, {"X": torch.zeros(4, 1, 1, 4, 4, dtype=torch.uint8)}

    import emu

    with emu.EmuBackend(), pytest.raises(RuntimeError):
        net, inputs = build(B200)
        net.run(inputs=inputs, time=4)


@pytest.mark.parametrize("rule", ["MSTDP", "MSTDPET"])
def test_reward_rules_refused(rule):
    X, Y = B200.nodes.Input(shape=[1, 6, 6], traces=True), B200.nodes.LIFNodes(shape=[2, 2, 2], traces=True)
    with pytest.raises(NotImplementedError):
        B200.topology.LocalConnection2D(X, Y, kernel_size=3, stride=3, n_filters=2, update_rule=getattr(B200.learning, rule))


def test_masks_refused():
    import emu

    net, inputs = _lc_net(B200)
    with emu.EmuBackend(), pytest.raises(NotImplementedError, match="dense Connection only"):
        net.run(inputs=inputs, time=4, masks={("X", "Y"): torch.zeros(1, 8, 9, dtype=torch.bool)})


def test_one_and_three_dimensional_local_connections_refused():
    X, Y = B200.nodes.Input(shape=[1, 6, 6]), B200.nodes.LIFNodes(shape=[2, 2, 2])
    for cls in (B200.topology.LocalConnection1D, B200.topology.LocalConnection3D):
        with pytest.raises(NotImplementedError):
            cls(X, Y, kernel_size=3, stride=3, n_filters=2)


def test_mixed_with_sparse_or_features_refused():
    import emu

    F_, _ = __import__("mcc_feature_nets").features(B200)
    for extra in ("sparse", "feature"):
        net, inputs = _lc_net(B200)
        Z = B200.nodes.LIFNodes(5)
        net.add_layer(Z, "Z")
        if extra == "sparse":
            c = B200.topology.SparseConnection(net.layers["Y"], Z, w=torch.rand(8, 5))
        else:
            c = B200.topology.MulticompartmentConnection(net.layers["Y"], Z, pipeline=[F_.Mask("m", torch.rand(8, 5) < 0.5),
                                                                                       F_.Weight("w", torch.rand(8, 5))])
        net.add_connection(c, "Y", "Z")
        with emu.EmuBackend(), pytest.raises(NotImplementedError, match="LocalConnection2D"):
            net.run(inputs=inputs, time=4)


def test_construction_attributes_match_reference():
    for ns in (_reference(), B200):
        if ns is None:
            continue
        X, Y = ns.nodes.Input(shape=[2, 9, 11]), ns.nodes.LIFNodes(shape=[3, 4, 4])
        torch.manual_seed(4)
        c = ns.topology.LocalConnection2D(X, Y, kernel_size=(3, 2), stride=(2, 3), n_filters=3, wmin=0.2, wmax=0.7)
        assert (c.kernel_size, c.stride, c.n_filters, c.in_channels, c.conv_size, c.conv_prod, c.kernel_prod) == \
            ((3, 2), (2, 3), 3, 2, (4, 4), 16, 6)
        assert c.w.shape == (2, 48, 6) and float(c.w.min()) >= 0.2 and float(c.w.max()) <= 0.7
        torch.manual_seed(4)
        assert torch.equal(c.w, torch.rand(2, 48, 6).clamp(0.2, 0.7))
        assert c.b.numel() == 0


# ---- 5. tier selection -----------------------------------------------------------------------------------------------

def test_tier_selection():
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    net, inputs = _lc_net(B200, B=2, learning=True, rule="PostPre", nu=(1e-2, 1e-2), reduction=torch.sum)

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


# ---- 6. the target reset ---------------------------------------------------------------------------------------------

def test_reset_resets_the_target():
    import emu

    net, inputs = _lc_net(B200, B=1)
    with emu.EmuBackend():
        net.run(inputs=inputs, time=4, inject_v={"Y": torch.full((8,), 3.0)})
    Y = net.layers["Y"]
    assert not torch.equal(Y.v, torch.full_like(Y.v, Y.rest))
    net.connections[("X", "Y")].reset_state_variables()
    assert torch.equal(Y.v, torch.full_like(Y.v, Y.rest)) and not Y.x.any() and not Y.s.any()


# ---- 7. the reference's own objects through the ABI -----------------------------------------------------------------

@pytest.mark.parametrize("case", ["example_b1", "c2_WeightDependentPostPre"])
def test_reference_binding_runs_the_references_network(case):
    ref = _reference()
    if ref is None:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb
    import local2d_oracle

    (a, inputs, T), (b, _, _) = ln.build_case(ref, case), ln.build_case(ref, case)
    a.run(inputs={"X": inputs["X"][0].clone()}, time=T)
    assert rb.run_window(b, {"X": inputs["X"][0].clone()}, time=T, library=local2d_oracle.lib()) == 0
    sa, sb = ln.state(a), ln.state(b)
    for k in (k for k in sa if "/" in k):   # (the binding runs the window; the reference's monitors are not its business)
        if k.endswith("s"):
            assert torch.equal(sa[k], sb[k]), k
        else:
            torch.testing.assert_close(sb[k], sa[k], rtol=1e-4, atol=1e-4, msg=k)
    assert sa["Ys"].sum() > 0
