"""Conv1dConnection (reference: topology.py:540-683) and its PostPre / WeightDependentPostPre / Hebbian rules on the
generic window kernel.  CPU tests: the oracle (tests/conv1d_oracle.c, the CPU oracle extended by the 1-D convolution)
against the live reference's stored results, the emulated kernel against the oracle bit for bit, the equivalence with a
Conv2dConnection of kernel (1, k), the standalone operators against F.conv1d and a torch restatement of the rules,
refusals, tier selection, the reference's own networks through the binding and the multi-GPU combine.  The stored
reference results are regenerated with ``python tests/golden/gen_live.py test_conv1d``."""
import ctypes as C
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import cases
import conv1d_nets as cn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")
CASES = list(cn.LIVE_CASES)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _flat(states):
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


def _reference():
    try:
        return cases.namespace("reference")
    except ImportError:
        return None


def _same(a, b):
    return torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num()))


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

@reference_side(CASES)
def _live(ns, case):
    net, inputs, T = cn.build_case(ns, case)
    return _flat(cn.run_windows(net, inputs, T, cn.windows_of(case)))


def _check_against(ref, ours, what):
    for k, v in ref.items():
        o = ours[k]
        assert o.shape == v.shape, (what, k)
        if k.endswith("s"):
            assert torch.equal(o.float(), v.float()), f"{what}: {k} differs"
        elif k.endswith("/w"):
            torch.testing.assert_close(o, v, rtol=1e-4, atol=1e-6, equal_nan=True, msg=f"{what}: {k}")
        else:
            torch.testing.assert_close(o.float(), v.float(), rtol=1e-5, atol=1e-4, equal_nan=True, msg=f"{what}: {k}")


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_live_reference(case):
    from conv1d_oracle import Conv1dOracleBackend

    net, inputs, T = cn.build_case(B200, case)
    w0 = net.connections[("X", "Y")].w.detach().clone()
    with Conv1dOracleBackend() as ob:
        ours = _flat(cn.run_windows(net, inputs, T, cn.windows_of(case)))
    assert ob.err == 0
    ref = load(_live, case)
    assert ref.keys() == ours.keys()
    _check_against(ref, ours, case)
    assert ours["w0/Ys"].sum() > 0
    if cn.LIVE_CASES[case].get("zero_row"):
        assert torch.isnan(ours["w0/XY/w"][1, 0]).all() and not torch.isnan(ours["w0/XY/w"][0]).any()
    elif cn.LIVE_CASES[case].get("learning", True):
        assert not torch.equal(ours["w0/XY/w"], w0)


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _emu_vs_oracle(build, env=None, n=2, **kw):
    import emu
    from conv1d_oracle import Conv1dOracleBackend

    outs = []
    for backend in (emu.EmuBackend, Conv1dOracleBackend):
        net, inputs, T = build()
        old = {k: os.environ.get(k) for k in (env or {})}
        os.environ.update(env if backend is emu.EmuBackend and env else {})
        try:
            with backend() as be:
                outs.append(_flat(cn.run_windows(net, inputs, T, n, **kw)))
            assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
    a, b = outs
    assert a.keys() == b.keys()
    for k in a:
        assert _same(a[k], b[k]), f"{k} differs"
    return a


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["example_b1", "c2_PostPre", "c2_WeightDependentPostPre", "c2_Hebbian", "c2_NoOp", "c2_mean"])
def test_emulated_kernel_bit_exact(case, env):
    a = _emu_vs_oracle(lambda: cn.build_case(B200, case, T=10 if case.startswith("example") else 24), ENVS[env])
    assert a["w1/Ys"].sum() > 0


@pytest.mark.parametrize("case", ["c2_bias", "c2_nolearn", "wide_k40"])
def test_emulated_kernel_other_cases_bit_exact(case):
    a = _emu_vs_oracle(lambda: cn.build_case(B200, case), ENVS["sms3"])
    assert a["w1/Ys"].sum() > 0


def test_emulated_kernel_zero_row_bit_exact():
    _emu_vs_oracle(lambda: cn.build_case(B200, "c2_zero_row"), ENVS["sms3"], n=1)


@pytest.mark.parametrize("rule", ["PostPre", "Hebbian"])
def test_emulated_kernel_one_step_bit_exact(rule):
    _emu_vs_oracle(lambda: cn.multi_net(B200, rule=rule), ENVS["sms3"], one_step=True)


def test_stepwise_equals_oracle():
    """A monitor on the target's traces makes the window run step by step (one one-step window per step)."""
    def build():
        net, inputs, T = cn.multi_net(B200, rule="WeightDependentPostPre", T=10)
        net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["x"], time=T), "Yx")
        return net, inputs, T

    _emu_vs_oracle(build, ENVS["sms3"])


@pytest.mark.parametrize("T", [7, 8])
def test_emulated_kernel_large_batch_bit_exact(T):
    """B = 520 (lanes over 32 samples at a time, 17 groups) and an odd and an even window length."""
    a = _emu_vs_oracle(lambda: cn.multi_net(B200, rule="PostPre", B=520, T=T), ENVS["sms3"])
    assert a["w1/Ys"].sum() > 0


@pytest.mark.parametrize("B", [3, 5, 33])
def test_emulated_kernel_sample_groups_bit_exact(B):
    """Batch sizes that leave lanes of the learning phase's warps idle (3, 5: groups of 4 / 8 lanes per element) and one
    that spans two groups of 32 samples (33)."""
    _emu_vs_oracle(lambda: cn.multi_net(B200, rule="Hebbian", B=B, T=9), ENVS["sms7"])


def test_two_windows_without_reset():
    _emu_vs_oracle(lambda: cn.multi_net(B200, rule="PostPre", T=9), ENVS["sms3"], reset=False)


def test_staged_and_unstaged_bits_and_taps():
    """The example geometry: a 25-word source sample and 56 taps per filter, so every tile stages its bit rows and taps;
    wide_k40 at B = 3 stages both too; a [3, 6000] source at B = 32 (5664 words) does not stage its bit rows, and
    4096 / (3 * 1400) taps do not fit the tap stage."""
    net, _, _ = cn.example_net(B200)
    p = cn.gather_paths(net.connections[("X", "Y")], 1)
    assert p["st_bits"] and p["st_taps_all"]

    def big():
        g = torch.Generator().manual_seed(3)
        net = B200.Network(dt=1.0, batch_size=32, learning=True)
        X = B200.nodes.Input(shape=[3, 6000], traces=True)
        Y = B200.nodes.LIFNodes(shape=[2, 4], traces=True, thresh=-60.0)
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        net.add_connection(B200.topology.Conv1dConnection(X, Y, kernel_size=1400, stride=1500, nu=(1e-4, 1e-3), wmin=0.0, wmax=1.0,
                                                          reduction=torch.sum, update_rule=B200.learning.PostPre,
                                                          w=0.01 * torch.rand(2, 3, 1400, generator=g)), "X", "Y")
        net.add_monitor(B200.monitors.Monitor(Y, ["s"], time=4), "Ys")
        return net, {"X": (torch.rand(2, 4, 32, 3, 6000, generator=g) < 0.1).to(torch.uint8)}, 4

    net, _, _ = big()
    p = cn.gather_paths(net.connections[("X", "Y")], 32)
    assert not p["st_bits"] and p["st_taps_some_off"]
    a = _emu_vs_oracle(big, ENVS["sms3"])
    assert a["w1/Ys"].sum() > 0


def test_scripted_tier_equals_window():
    import emu
    from conv1d_oracle import Conv1dOracleBackend
    from test_scripted_tier import MyLIF

    def build(user):
        net, inputs, T = cn.multi_net(B200, rule="PostPre", B=3, T=12)
        if user:   # a user-defined population as the last layer: the network runs on the scripted tier
            Z = MyLIF(6, traces=True, thresh=-62.0)
            net.layers["Z"] = Z
            net.add_layer(Z, "Z")
            net.connections[("Y", "Z")].target = Z
            net.monitors["Zs"].obj = Z
        return net, inputs, T

    outs = []
    for user, backend in ((True, emu.EmuBackend), (True, Conv1dOracleBackend), (False, emu.EmuBackend)):
        net, inputs, T = build(user)
        assert net._scripted_required() == user
        with backend():
            net.run(inputs={"X": inputs["X"][0]}, time=T)
        outs.append(cn.state(net))
    for o in outs[1:]:
        for k in outs[0]:
            assert torch.equal(outs[0][k].float(), o[k].float()), k
    assert outs[0]["Ys"].sum() > 0


# ---- 3. Conv1d with one input channel is Conv2d with kernel (1, k) ---------------------------------------------------

def _twin(kind, rule, B=4, T=16, seed=31):
    g = torch.Generator().manual_seed(seed)
    net = B200.Network(dt=1.0, batch_size=B, learning=True)
    X = B200.nodes.Input(shape=[1, 30] if kind == 1 else [1, 1, 30], traces=True)
    Y = B200.nodes.LIFNodes(shape=[3, 14] if kind == 1 else [3, 1, 14], traces=True, thresh=-60.0)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    w = 0.6 * torch.rand(3, 1, 5, generator=g)
    kw = dict(nu=(2e-3, 5e-3), wmin=0.0, wmax=1.0, norm=2.5, reduction=torch.sum, update_rule=getattr(B200.learning, rule))
    if rule == "NoOp":
        kw["weight_decay"] = 0.01
    if kind == 1:
        conv = B200.topology.Conv1dConnection(X, Y, kernel_size=5, stride=2, padding=1, w=w, **kw)
    else:
        conv = B200.topology.Conv2dConnection(X, Y, kernel_size=(1, 5), stride=(1, 2), padding=(0, 1), w=w.unsqueeze(2), **kw)
    net.add_connection(conv, "X", "Y")
    net.add_monitor(B200.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 30, generator=g) < 0.3).to(torch.uint8)
    return net, {"X": x.view(2, T, B, 1, 30) if kind == 1 else x.view(2, T, B, 1, 1, 30)}, T


@pytest.mark.parametrize("rule", ["PostPre", "WeightDependentPostPre", "Hebbian", "NoOp"])
def test_single_channel_equals_conv2d_twin(rule):
    import emu

    outs = []
    for kind in (1, 2):
        net, inputs, T = _twin(kind, rule)
        with emu.EmuBackend():
            st = _flat(cn.run_windows(net, inputs, T, 2))
        outs.append(st)
    a, b = outs
    for k in a:
        assert torch.equal(a[k].flatten(), b[k].flatten()), k
    assert a["w1/Ys"].sum() > 0 and torch.isfinite(a["w1/XY/w"]).all()


# ---- 4. the standalone operators -------------------------------------------------------------------------------------

def _restated_update(conn, rule, B):
    """learning.py:422-455 / 873-918 / 1316-1346 in torch: the reshaped unfold of the padded source."""
    X, Y = conn.source, conn.target
    k, s, p, cin, cout = conn.kernel_size, conn.stride, conn.padding, conn.in_channels, conn.out_channels

    def unf(v):
        return F.pad(v.float(), (p, p)).unfold(-1, k, s).reshape(B, -1, cin * k)

    pre = torch.bmm(Y.x.view(B, cout, -1), unf(X.s)).sum(0)
    post = torch.bmm(Y.s.float().view(B, cout, -1), unf(X.x)).sum(0)
    w = conn.w.clone().view(pre.shape)
    nu0, nu1 = float(rule.nu[0]), float(rule.nu[1])
    if type(rule).__name__ == "WeightDependentPostPre":
        w = w + (-(nu0 * pre * (w - 0.0)) + nu1 * post * (1.0 - w))
    elif type(rule).__name__ == "Hebbian":
        w = w + nu0 * pre + nu1 * post
    else:
        w = w - nu0 * pre + nu1 * post
    return w.clamp(0.0, 1.0).view(conn.w.shape)


@pytest.mark.parametrize("rule", ["PostPre", "WeightDependentPostPre", "Hebbian"])
def test_standalone_operators_match_torch(rule):
    import emu
    from conv1d_oracle import Conv1dOracleBackend

    g = torch.Generator().manual_seed(21)
    B = 3
    X = B200.nodes.Input(shape=[3, 11], traces=True)
    Y = B200.nodes.LIFNodes(shape=[2, 5], traces=True)
    for L in (X, Y):
        L.set_batch_size(B)
        L.compute_decays(1.0)
    conn = B200.topology.Conv1dConnection(X, Y, kernel_size=4, stride=2, padding=1, nu=(0.01, 0.02), wmin=0.0, wmax=1.0, norm=2.0,
                                          reduction=torch.sum, update_rule=getattr(B200.learning, rule), b=torch.rand(2, generator=g))
    for step in range(3):
        s = torch.rand(B, 3, 11, generator=g) < 0.4
        with emu.EmuBackend():
            out = conn.compute(s)
        with Conv1dOracleBackend():
            assert torch.equal(out, conn.compute(s))
        torch.testing.assert_close(out, F.conv1d(s.float(), conn.w, conn.b, stride=2, padding=1), rtol=1e-5, atol=1e-5)
        X.s = s.clone()
        X.x = torch.rand(B, 3, 11, generator=g)
        Y.s = torch.rand(B, 2, 5, generator=g) < 0.3
        Y.x = torch.rand(B, 2, 5, generator=g)
        ref = _restated_update(conn, conn.update_rule, B)
        w_before = conn.w.detach().clone()
        with Conv1dOracleBackend():
            conn.update_rule.update()
        w_oracle = conn.w.detach().clone()
        with torch.no_grad():
            conn.w.copy_(w_before)
        with emu.EmuBackend():
            conn.update_rule.update()
        assert torch.equal(conn.w, w_oracle)
        torch.testing.assert_close(conn.w, ref, rtol=1e-5, atol=1e-6)
    with emu.EmuBackend():
        conn.normalize()
    rows = conn.w.view(-1, 4).sum(-1)
    torch.testing.assert_close(rows, torch.full_like(rows, 2.0), rtol=1e-5, atol=1e-5)


# ---- 5. refusals and errors ------------------------------------------------------------------------------------------

def _small(ns, B=2, rule="NoOp", learning=True, tgt=(2, 4), src=(1, 9), **kw):
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=list(src), traces=True)
    Y = ns.nodes.LIFNodes(shape=list(tgt), traces=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    net.add_connection(ns.topology.Conv1dConnection(X, Y, kernel_size=3, stride=2, update_rule=getattr(ns.learning, rule), **kw), "X", "Y")
    return net, {"X": (torch.rand(4, B, *src, generator=torch.Generator().manual_seed(1)) < 0.3).to(torch.uint8)}


def _unchanged_after(exc, net, inputs, match=None, **run_kw):
    import emu

    before = {k: v.clone() for k, v in cn.state(net).items()}
    with emu.EmuBackend(), pytest.raises(exc, match=match):
        net.run(inputs=inputs, time=4, **run_kw)
    after = cn.state(net)
    for k in before:
        assert _same(before[k], after[k]), k


@pytest.mark.parametrize("src,tgt", [((1, 6, 6), (2, 2, 2)), ((1, 9), (2, 2, 2)), ((9,), (2, 4))])
def test_populations_other_than_c_l_refused(src, tgt):
    X, Y = B200.nodes.Input(shape=list(src)), B200.nodes.LIFNodes(shape=list(tgt))
    with pytest.raises(NotImplementedError, match=r"\[C, L\]"):
        B200.topology.Conv1dConnection(X, Y, 3)
    with pytest.raises(NotImplementedError, match=r"\[C, L\]"):
        B200.topology.Conv1dConnection(None, None, 3)


def test_dilation_refused():
    for ns in (_reference(), B200):
        if ns is not None:
            with pytest.raises(NotImplementedError):
                _small(ns, dilation=2)


def test_wrong_target_shape_raises_assertion_error():
    for ns in (_reference(), B200):
        if ns is not None:
            with pytest.raises(AssertionError):
                _small(ns, tgt=(2, 5))


def test_non_float32_weights_and_tensor_bounds_refused():
    with pytest.raises(NotImplementedError):
        _small(B200, w_dtype=torch.float16)
    with pytest.raises(NotImplementedError):
        _small(B200, rule="PostPre", nu=(torch.ones(2, 1, 3), torch.ones(2, 1, 3)), wmin=0.0, wmax=1.0)
    net, inputs = _small(B200, rule="PostPre", nu=(1e-2, 1e-2), wmin=torch.zeros(2, 1, 3), wmax=1.0)
    _unchanged_after(NotImplementedError, net, inputs, match="wmin/wmax")


def test_empty_output_raises_runtime_error():
    def build(ns):
        net = ns.Network(dt=1.0, batch_size=1, learning=False)
        X, Y = ns.nodes.Input(shape=[1, 4]), ns.nodes.LIFNodes(shape=[2, 0])
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        net.add_connection(ns.topology.Conv1dConnection(X, Y, kernel_size=5), "X", "Y")
        return net, {"X": torch.zeros(4, 1, 1, 4, dtype=torch.uint8)}

    ref = _reference()
    if ref is not None:
        with pytest.raises(RuntimeError):
            net, inputs = build(ref)
            net.run(inputs=inputs, time=4)
    net, inputs = build(B200)
    _unchanged_after(RuntimeError, net, inputs)


def test_bad_bias_shape_raises_runtime_error():
    net, inputs = _small(B200, learning=False, b=torch.zeros(3))
    _unchanged_after(RuntimeError, net, inputs, match="bias")


def test_squeeze_reduction_at_batch_size_above_one_refused():
    net, inputs = _small(B200, B=1, rule="PostPre", nu=(1e-2, 1e-2), wmin=0.0, wmax=1.0)
    net.batch_size = 2
    for L in net.layers.values():
        L.set_batch_size(2)
    with pytest.raises(RuntimeError, match="torch.squeeze"):
        import emu
        with emu.EmuBackend():
            net.run(inputs={"X": torch.zeros(4, 2, 1, 9, dtype=torch.uint8)}, time=4)


@pytest.mark.parametrize("rule", ["MSTDP", "MSTDPET"])
def test_reward_rules_refused(rule):
    with pytest.raises(NotImplementedError, match="Conv1dConnection"):
        _small(B200, rule=rule)


def test_masks_refused():
    net, inputs = _small(B200, learning=False)
    _unchanged_after(NotImplementedError, net, inputs, match="dense Connection only", masks={("X", "Y"): torch.zeros(2, 1, 3, dtype=torch.bool)})


def test_mixed_with_sparse_or_features_refused():
    import emu

    F_, _ = __import__("mcc_feature_nets").features(B200)
    for extra in ("sparse", "feature"):
        net, inputs = _small(B200, learning=False)
        Z = B200.nodes.LIFNodes(5)
        net.add_layer(Z, "Z")
        if extra == "sparse":
            c = B200.topology.SparseConnection(net.layers["Y"], Z, w=torch.rand(8, 5))
        else:
            c = B200.topology.MulticompartmentConnection(net.layers["Y"], Z, pipeline=[F_.Mask("m", torch.rand(8, 5) < 0.5),
                                                                                       F_.Weight("w", torch.rand(8, 5))])
        net.add_connection(c, "Y", "Z")
        with emu.EmuBackend(), pytest.raises(NotImplementedError, match="Conv1dConnection"):
            net.run(inputs=inputs, time=4)


def test_other_one_dimensional_kinds_stay_refused():
    X, Y = B200.nodes.Input(shape=[1, 9]), B200.nodes.LIFNodes(shape=[2, 4])
    for cls in (B200.topology.MaxPool1dConnection, B200.topology.LocalConnection1D, B200.topology.LocalConnection3D):
        with pytest.raises(NotImplementedError):
            cls(X, Y, 3)


def test_construction_attributes_match_reference():
    for ns in (_reference(), B200):
        if ns is None:
            continue
        X, Y = ns.nodes.Input(shape=[2, 20]), ns.nodes.LIFNodes(shape=[3, 10])
        for kw, draw in ((dict(wmin=0.2, wmax=0.7), lambda: 0.5 * torch.rand(3, 2, 4) + 0.2),
                         (dict(wmax=0.7), lambda: torch.rand(3, 2, 4).clamp(max=0.7))):
            torch.manual_seed(4)
            c = ns.topology.Conv1dConnection(X, Y, kernel_size=4, stride=2, padding=1, **kw)
            assert (c.kernel_size, c.stride, c.padding, c.dilation, c.in_channels, c.out_channels) == (4, 2, 1, 1, 2, 3)
            torch.manual_seed(4)
            torch.testing.assert_close(c.w.data, draw(), rtol=0, atol=1e-7)
            assert torch.equal(c.b.data, torch.zeros(3))


# ---- 6. tier selection -----------------------------------------------------------------------------------------------

def test_tier_selection():
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    net, inputs = _small(B200, rule="PostPre", nu=[1e-2, 1e-2], wmin=0.0, wmax=1.0, reduction=torch.sum)

    def tier(force, delta=False):
        plan, keep = _plan.build_net(net, 2, {}, {}, {}, {}, {})
        opts = _abi.SnnRunOpts()
        opts.T, opts.B, opts.tier = 4, 2, force
        dw = torch.zeros(2, 1, 3)
        if delta:
            opts.delta_w = dw.data_ptr()
        return int(emu.lib().snn_b200_select_tier(C.byref(plan), C.byref(opts)))

    assert tier(0) == 1 and tier(1) == 1 and tier(2) == 0 and tier(3) == 0 and tier(0, delta=True) == 0
    net.force_tier = 2
    with emu.EmuBackend(), pytest.raises(RuntimeError, match="not implemented"):
        net.run(inputs=inputs, time=4)
    net.force_tier = 0
    with emu.EmuBackend():
        net.run(inputs=inputs, time=4)
    assert emu.last_tier == 1


# ---- 7. the reference's own objects through the ABI -----------------------------------------------------------------

@pytest.mark.parametrize("case", ["example_b1", "c2_WeightDependentPostPre", "c2_Hebbian"])
def test_reference_binding_runs_the_references_network(case):
    ref = _reference()
    if ref is None:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb
    import conv1d_oracle

    (a, inputs, T), (b, _, _) = cn.build_case(ref, case), cn.build_case(ref, case)
    a.run(inputs={"X": inputs["X"][0].clone()}, time=T)
    assert rb.run_window(b, {"X": inputs["X"][0].clone()}, time=T, library=conv1d_oracle.lib()) == 0
    sa, sb = cn.state(a), cn.state(b)
    for k in (k for k in sa if "/" in k):   # (the binding runs the window; the reference's monitors are not its business)
        if k.endswith("s"):
            assert torch.equal(sa[k], sb[k]), k
        else:
            torch.testing.assert_close(sb[k], sa[k], rtol=1e-4, atol=1e-4, msg=k)
    assert sa["Ys"].sum() > 0


# ---- 8. the multi-GPU combine: sum + clamp on the flattened filters, then the connection's own normalize ------------

def _dist_make(B):
    return cn.multi_net(B200, rule="PostPre", B=B, T=12)[0]


def _dist_inputs():
    return cn.multi_net(B200, B=8, T=12)[1]["X"]


def _dist_worker(rank, world, port, out):
    import torch.distributed as dist

    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from bindsnet_b200.distributed import ShardedWindowRunner
    from conv1d_oracle import Conv1dOracleBackend
    from test_distributed import _patch_cpu_combine

    _patch_cpu_combine()
    shard = _dist_inputs()[:, :, rank * 4:(rank + 1) * 4]
    net = _dist_make(4)
    with Conv1dOracleBackend():
        runner = ShardedWindowRunner(net)
        for window in range(2):
            if window:
                net.reset_state_variables()
            runner.run({"X": shard[window]}, time=12)
    torch.save({f"{s}->{t}": c.w.detach().clone() for (s, t), c in net.connections.items()}, os.path.join(out, f"rank{rank}.pt"))
    dist.destroy_process_group()


def test_two_rank_combine_normalizes_conv1d_filters(tmp_path):
    import numpy as np
    import torch.multiprocessing as mp
    from conv1d_oracle import Conv1dOracleBackend

    port = 34500 + (os.getpid() % 1000)
    mp.spawn(_dist_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    assert all(torch.equal(r0[k], r1[k]) for k in r0), "ranks diverged"

    x = _dist_inputs()
    nets = [_dist_make(4), _dist_make(4)]
    keys = list(nets[0].connections)
    w = {k: nets[0].connections[k].w.detach().clone() for k in keys}
    with Conv1dOracleBackend():
        for window in range(2):
            sums = {k: torch.zeros_like(w[k]) for k in keys}
            for r, net in enumerate(nets):
                with torch.no_grad():
                    for k in keys:
                        net.connections[k].w.copy_(w[k])
                if window:
                    net.reset_state_variables()
                net.run({"X": x[window, :, r * 4:(r + 1) * 4]}, time=12, b200_normalize=False)
                for k in keys:
                    sums[k] += net.connections[k].w.detach() - w[k]
            c = nets[0].connections[("X", "Y")]
            with torch.no_grad():
                c.w.copy_(torch.clamp(w[("X", "Y")] + sums[("X", "Y")], float(c.wmin), float(c.wmax)))
            c.normalize()   # per (out, in) filter, not per column of a [n_src, n_tgt] matrix
            w[("X", "Y")] = c.w.detach().clone()
    assert np.array_equal(r0["X->Y"].numpy(), w[("X", "Y")].numpy())
    sums = r0["X->Y"].view(6, -1).sum(1)
    torch.testing.assert_close(sums, torch.full_like(sums, 2.0), rtol=1e-5, atol=1e-5)
