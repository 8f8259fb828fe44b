"""LocalConnection3D (reference: topology.py:1770-1917) and its PostPre / WeightDependentPostPre / Hebbian rules on the
generic window kernel.  CPU tests: the oracle (tests/local3d_oracle.c, the CPU oracle extended by both local connections)
against the live reference's stored results, the emulated kernel against the oracle bit for bit, the LocalConnection2D
twin, the standalone operators against a torch restatement, refusals, tier selection, the reference's own networks and the
multi-GPU combine.  The stored reference results are regenerated with ``python tests/golden/gen_live.py test_local3d``."""
import ctypes as C
import os
import sys

import pytest
import torch

import cases
import local3d_nets as ln
from live_golden import load, reference_side

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))

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
    return ln.shrink(_flat(ln.run_windows(net, inputs, T, ln.windows_of(case))))


def _check_against(ref, ours, what):
    for k, v in ref.items():
        o = ours[k]
        assert o.shape == v.shape, (what, k)
        if k.endswith("s"):
            assert torch.equal(o.float(), v.float()), f"{what}: {k} differs"
        elif "/w" in k:
            torch.testing.assert_close(o, v, rtol=1e-4, atol=0.0, equal_nan=True, msg=f"{what}: {k}")
        else:
            torch.testing.assert_close(o.float(), v.float(), rtol=1e-5, atol=1e-4, equal_nan=True, msg=f"{what}: {k}")


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_live_reference(case):
    from local3d_oracle import Local3dOracleBackend

    net, inputs, T = ln.build_case(B200, case)
    with Local3dOracleBackend() as ob:
        ours = _flat(ln.run_windows(net, inputs, T, ln.windows_of(case)))
    assert ob.err == 0
    _check_against(load(_live, case), ln.shrink(ours), case)
    assert ours["w0/Ys"].sum() > 0
    if ln.LIVE_CASES[case] and ln.LIVE_CASES[case].get("zero_row"):
        assert torch.isnan(ours["w0/XY/w"][1, 7]).all() and not torch.isnan(ours["w0/XY/w"][0]).any()


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _equal(a, b):
    return torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num()))


def _emu_vs_oracle(build, env=None, n=2, **kw):
    import emu
    from local3d_oracle import Local3dOracleBackend

    outs = []
    for backend in (emu.EmuBackend, Local3dOracleBackend):
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
        assert _equal(a[k], b[k]), f"{k} differs"
    return a


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["c2_PostPre", "c2_WeightDependentPostPre", "c2_Hebbian", "c2_NoOp", "c2_mean"])
def test_emulated_kernel_bit_exact(case, env):
    a = _emu_vs_oracle(lambda: ln.build_case(B200, case), ENVS[env])
    assert a["w1/Ys"].sum() > 0


def test_emulated_kernel_example_bit_exact():
    """The example's layer sizes (kernel 16^3, 25 filters) on an 18^3 source, a short window."""
    a = _emu_vs_oracle(lambda: ln.example_net(B200, T=5, S=18), ENVS["sms3"])
    assert a["w0/Ys"].sum() > 0


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


@pytest.mark.parametrize("B,T", [(3, 7), (33, 5), (520, 7)])
def test_emulated_kernel_batch_sizes_bit_exact(B, T):
    """B = 3 / 33 / 520 with odd window lengths: one, two and many 32-sample groups of the learning phase."""
    a = _emu_vs_oracle(lambda: ln.multi_net(B200, rule="PostPre", B=B, T=T), ENVS["sms3"])
    assert a["w1/Ys"].sum() > 0


def test_two_windows_without_reset():
    _emu_vs_oracle(lambda: ln.multi_net(B200, rule="Hebbian", T=9), ENVS["sms3"], reset=False)


def test_tiles_straddle_filters():
    """P = 36 target positions per filter: the 32-neuron tiles of the target start inside filters, and 7 SMs spread the
    learning phase's row segments over many CTAs."""
    _emu_vs_oracle(lambda: ln.multi_net(B200, rule="Hebbian", B=3, T=9), ENVS["sms7"])


def _wide(B):
    """A [1, 20, 20, 20] source (250 bit words per sample) with a small kernel: at B = 3 a phase-1 chunk stages its bit
    rows (750 words), at B = 33 it does not (at least 17 samples, 4250 words > SNN_CONV_STAGE_WORDS)."""
    return lambda: ln.multi_net(B200, rule="WeightDependentPostPre", B=B, T=5, shape=(1, 20, 20, 20), kernel=(2, 3, 4),
                                stride=(3, 3, 3), filters=2)


@pytest.mark.parametrize("B", [3, 33])
def test_staged_and_unstaged_bit_rows(B):
    a = _emu_vs_oracle(_wide(B), ENVS["sms3"])
    assert a["w1/Ys"].sum() > 0


def test_kernel_rows_wider_than_a_word():
    """kw = 36 along the contiguous axis: every kernel row of the gather spans a bit-word boundary, and K = 72 elements
    per channel give a row segment of the learning phase that ends inside a row."""
    a = _emu_vs_oracle(lambda: ln.multi_net(B200, rule="PostPre", B=2, T=6, shape=(1, 3, 2, 45), kernel=(2, 1, 36), stride=(1, 1, 4),
                                            filters=2), ENVS["shuffle"])
    assert a["w1/Ys"].sum() > 0


def test_scripted_tier_equals_window():
    import emu
    from local3d_oracle import Local3dOracleBackend
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
    for user, backend in ((True, emu.EmuBackend), (True, Local3dOracleBackend), (False, emu.EmuBackend)):
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
    from local3d_oracle import Local3dOracleBackend

    for backend in (emu.EmuBackend, Local3dOracleBackend):
        X = B200.nodes.Input(shape=[1, 4, 6, 6])
        Y = B200.nodes.LIFNodes(shape=[2, 2, 2, 2])
        B200.Network(batch_size=1, learning=False)
        lc = B200.topology.LocalConnection3D(X, Y, kernel_size=(2, 3, 3), stride=(2, 3, 3), n_filters=2)
        with torch.no_grad():
            lc.w[0, :, 0] = float("inf")
        s = torch.ones(1, 1, 4, 6, 6, dtype=torch.bool)
        s[0, 0, ::2, ::3, ::3] = False       # the first position of every window is silent
        with backend():
            out = lc.compute(s)
        assert torch.isfinite(out).all()
        torch.testing.assert_close(out.view(-1), lc.w[0, :, 1:].sum(-1), rtol=1e-6, atol=1e-6)


# ---- 3. the LocalConnection2D twin -----------------------------------------------------------------------------------

def _twin(ns3, rule, dims):
    """LocalConnection3D on [2, 1, 9, 11] with kernel (1, 3, 4) and stride (1, 2, 3) when dims == 3, the
    LocalConnection2D on [2, 9, 11] with kernel (3, 4) and stride (2, 3) otherwise; the same weights, inputs and targets."""
    g = torch.Generator().manual_seed(17)
    B, T = 3, 10
    net = ns3.Network(dt=1.0, batch_size=B, learning=True)
    X = ns3.nodes.Input(shape=[2, 1, 9, 11] if dims == 3 else [2, 9, 11], traces=True)
    Y = ns3.nodes.LIFNodes(shape=[3, 1, 4, 3] if dims == 3 else [3, 4, 3], traces=True, thresh=-60.0, refrac=2)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    kw = dict(nu=(2e-3, 5e-3), wmin=0.0, wmax=1.0, norm=3.0, reduction=torch.sum, update_rule=getattr(ns3.learning, rule))
    if rule == "NoOp":
        kw["weight_decay"] = 0.01
    if dims == 3:
        lc = ns3.topology.LocalConnection3D(X, Y, kernel_size=(1, 3, 4), stride=(1, 2, 3), n_filters=3, **kw)
    else:
        lc = ns3.topology.LocalConnection2D(X, Y, kernel_size=(3, 4), stride=(2, 3), n_filters=3, **kw)
    with torch.no_grad():
        lc.w.copy_(0.5 * torch.rand(lc.w.shape, generator=g))
    net.add_connection(lc, "X", "Y")
    net.add_monitor(ns3.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 2, 9, 11, generator=g) < 0.3).to(torch.uint8)
    return net, {"X": x.unsqueeze(4) if dims == 3 else x}, T


@pytest.mark.parametrize("backend", ["emu", "oracle"])
@pytest.mark.parametrize("rule", ln.RULES)
def test_twin_of_local_connection_2d_bit_identical(rule, backend):
    """A LocalConnection3D whose first spatial axis is 1 is bit-identical to its LocalConnection2D twin: the gather, each
    rule's pairing and normalize reduce exactly to the 2-D ones."""
    import emu
    from local3d_oracle import Local3dOracleBackend

    be = emu.EmuBackend if backend == "emu" else Local3dOracleBackend
    outs = []
    for dims in (3, 2):
        net, inputs, T = _twin(B200, rule, dims)
        with be():
            st = ln.run_windows(net, inputs, T, 2)
        outs.append([{k: v.reshape(-1) for k, v in s.items()} for s in st])
    for a, b in zip(*outs):
        assert a.keys() == b.keys()
        for k in a:
            assert _equal(a[k], b[k]), f"{rule}: {k} differs from the LocalConnection2D twin"
    assert outs[0][0]["Ys"].sum() > 0


# ---- 4. the standalone operators -------------------------------------------------------------------------------------

def _unfold(v, k, st):
    """The reference's three unfolds of a [B, C, H, W, D] tensor, flattened to [B, C, P, K] (topology.py:1885-1891)."""
    B, Cin = v.shape[:2]
    u = v.float().unfold(-3, k[0], st[0]).unfold(-3, k[1], st[1]).unfold(-3, k[2], st[2])
    return u.reshape(B, Cin, -1, k[0] * k[1] * k[2])


def _restated_compute(s, w, k, st, F_):
    """topology.py:1866-1896 in torch: one weight per (channel, target, window position)."""
    return (_unfold(s, k, st).repeat(1, 1, F_, 1) * w).sum(-1).sum(1)


def _restated_update(conn, rule, B):
    """learning.py:322-388 / 793-871 / 1249-1314 in torch: the reshaped unfold, row n' reads row n' % P."""
    k, st, F_ = conn.kernel_size, conn.stride, conn.n_filters
    X, Y = conn.source, conn.target

    def unf(v):
        return _unfold(v, k, st).reshape(B, conn.conv_prod, -1).repeat(1, F_, 1)   # [B, N, Cin * K]

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


@pytest.mark.parametrize("backend", ["emu", "oracle"])
@pytest.mark.parametrize("rule", ["PostPre", "WeightDependentPostPre", "Hebbian"])
def test_standalone_operators_match_torch(rule, backend):
    import emu
    from local3d_oracle import Local3dOracleBackend

    g = torch.Generator().manual_seed(21)
    B = 3
    X = B200.nodes.Input(shape=[2, 7, 5, 11], traces=True)
    Y = B200.nodes.LIFNodes(shape=[3, 3, 4, 3], traces=True)
    for L in (X, Y):
        L.set_batch_size(B)
        L.compute_decays(1.0)
    conn = B200.topology.LocalConnection3D(X, Y, kernel_size=(3, 2, 4), stride=(2, 1, 3), n_filters=3, nu=(0.01, 0.02), wmin=0.0,
                                           wmax=1.0, norm=2.0, reduction=torch.sum, update_rule=getattr(B200.learning, rule))
    assert conn.w.shape == (2, 108, 24) and conn.conv_size == (3, 4, 3)
    with (emu.EmuBackend if backend == "emu" else Local3dOracleBackend)():
        for step in range(3):
            s = torch.rand(B, 2, 7, 5, 11, generator=g) < 0.4
            out = conn.compute(s)
            torch.testing.assert_close(out.view(B, -1), _restated_compute(s, conn.w, conn.kernel_size, conn.stride, 3), rtol=1e-5, atol=1e-5)
            X.s = s.clone()
            X.x = torch.rand(B, 2, 7, 5, 11, generator=g)
            Y.s = torch.rand(B, 3, 3, 4, 3, generator=g) < 0.3
            Y.x = torch.rand(B, 3, 3, 4, 3, generator=g)
            ref = _restated_update(conn, conn.update_rule, B)
            conn.update_rule.update()
            torch.testing.assert_close(conn.w, ref, rtol=1e-5, atol=1e-6)
        conn.normalize()
    rows = conn.w.view(-1, 24).sum(-1)
    torch.testing.assert_close(rows, torch.full_like(rows, 2.0), rtol=1e-5, atol=1e-5)


# ---- 5. refusals and errors ------------------------------------------------------------------------------------------

def _lc_net(ns, B=2, tgt_shape=(2, 2, 2, 2), learning=False, rule=None, src=(1, 4, 6, 6), kernel=(2, 3, 3), stride=(2, 3, 3), **kw):
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=list(src), traces=True)
    Y = ns.nodes.LIFNodes(shape=list(tgt_shape), traces=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    if rule is not None:
        kw["update_rule"] = getattr(ns.learning, rule)
    net.add_connection(ns.topology.LocalConnection3D(X, Y, kernel_size=kernel, stride=stride, n_filters=2, **kw), "X", "Y")
    return net, {"X": (torch.rand(4, B, *src, generator=torch.Generator().manual_seed(1)) < 0.3).to(torch.uint8)}


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
    _raises_like_reference(lambda ns: _lc_net(ns, w=torch.rand(1, 16, 18)), AttributeError)


def test_wrong_target_size_raises_runtime_error():
    _raises_like_reference(lambda ns: _lc_net(ns, tgt_shape=(3, 2, 2, 2)), RuntimeError)


def test_kernel_larger_than_source_raises_runtime_error():
    """int((3 - 5) / 2) + 1 == 1: the conv size is 1 along that axis, but the kernel does not fit; unfold fails."""
    _raises_like_reference(lambda ns: _lc_net(ns, src=(1, 3, 6, 6), kernel=(5, 3, 3), tgt_shape=(2, 1, 2, 2)), RuntimeError)


def test_non_four_dimensional_source_refused_before_arguments():
    """A source that is not [C, H, W, D] raises NotImplementedError before the other arguments are looked at; with a
    [C, H, W, D] source the missing stride / n_filters raise the reference's TypeError."""
    for shape in ([1, 6, 6], [1, 9]):
        X, Y = B200.nodes.Input(shape=shape), B200.nodes.LIFNodes(shape=[2, 2, 2])
        with pytest.raises(NotImplementedError):
            B200.topology.LocalConnection3D(X, Y, 3)
        with pytest.raises(NotImplementedError):
            B200.topology.LocalConnection3D(X, Y, kernel_size=3, stride=3, n_filters=2)
    with pytest.raises(NotImplementedError):
        B200.topology.LocalConnection3D(B200.nodes.Input(shape=[1, 4, 4, 4]), torch.zeros(3), 2, 2, 2)
    for ns in (_reference(), B200):
        if ns is None:
            continue
        X, Y = ns.nodes.Input(shape=[1, 4, 6, 6]), ns.nodes.LIFNodes(shape=[2, 2, 2, 2])
        with pytest.raises(TypeError, match="missing 2 required positional arguments: 'stride' and 'n_filters'"):
            ns.topology.LocalConnection3D(X, Y, 3)
        with pytest.raises(TypeError, match="missing 1 required positional argument: 'n_filters'"):
            ns.topology.LocalConnection3D(X, Y, 3, 2)


@pytest.mark.parametrize("rule", ["MSTDP", "MSTDPET"])
def test_reward_rules_refused(rule):
    X, Y = B200.nodes.Input(shape=[1, 4, 6, 6], traces=True), B200.nodes.LIFNodes(shape=[2, 2, 2, 2], traces=True)
    with pytest.raises(NotImplementedError):
        B200.topology.LocalConnection3D(X, Y, kernel_size=(2, 3, 3), stride=(2, 3, 3), n_filters=2, update_rule=getattr(B200.learning, rule))


def test_masks_refused():
    import emu

    net, inputs = _lc_net(B200)
    with emu.EmuBackend(), pytest.raises(NotImplementedError, match="dense Connection only"):
        net.run(inputs=inputs, time=4, masks={("X", "Y"): torch.zeros(1, 16, 18, dtype=torch.bool)})


def test_non_float32_and_tensor_parameters_refused():
    import emu

    X, Y = B200.nodes.Input(shape=[1, 4, 6, 6], traces=True), B200.nodes.LIFNodes(shape=[2, 2, 2, 2], traces=True)
    with pytest.raises(NotImplementedError):
        B200.topology.LocalConnection3D(X, Y, kernel_size=(2, 3, 3), stride=(2, 3, 3), n_filters=2, w_dtype=torch.float16)
    for kw in (dict(wmin=torch.zeros(1, 16, 18)), dict(wmax=torch.ones(1, 16, 18)),
               dict(rule="PostPre", learning=True, nu=(torch.full((1, 16, 18), 1e-3), torch.full((1, 16, 18), 1e-3)))):
        with emu.EmuBackend(), pytest.raises(NotImplementedError):   # (tensor nu: when the rule is built)
            net, inputs = _lc_net(B200, **kw)
            net.run(inputs=inputs, time=4)


def test_mixed_with_sparse_features_or_neuron_tensors_refused():
    import emu

    F_, _ = __import__("mcc_feature_nets").features(B200)
    for extra in ("sparse", "feature"):
        net, inputs = _lc_net(B200)
        Z = B200.nodes.LIFNodes(5)
        net.add_layer(Z, "Z")
        if extra == "sparse":
            c = B200.topology.SparseConnection(net.layers["Y"], Z, w=torch.rand(16, 5))
        else:
            c = B200.topology.MulticompartmentConnection(net.layers["Y"], Z, pipeline=[F_.Mask("m", torch.rand(16, 5) < 0.5),
                                                                                       F_.Weight("w", torch.rand(16, 5))])
        net.add_connection(c, "Y", "Z")
        with emu.EmuBackend(), pytest.raises(NotImplementedError, match="LocalConnection3D"):
            net.run(inputs=inputs, time=4)
    net = B200.Network(dt=1.0, batch_size=2, learning=False)
    X = B200.nodes.Input(shape=[1, 4, 6, 6])
    Y = B200.nodes.LIFNodes(shape=[2, 2, 2, 2], thresh=torch.full((2, 2, 2, 2), -55.0))
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    net.add_connection(B200.topology.LocalConnection3D(X, Y, kernel_size=(2, 3, 3), stride=(2, 3, 3), n_filters=2), "X", "Y")
    with emu.EmuBackend(), pytest.raises(NotImplementedError, match="LocalConnection3D"):
        net.run(inputs={"X": torch.zeros(4, 2, 1, 4, 6, 6, dtype=torch.uint8)}, time=4)


def test_construction_attributes_match_reference():
    for ns in (_reference(), B200):
        if ns is None:
            continue
        X, Y = ns.nodes.Input(shape=[2, 7, 5, 11]), ns.nodes.LIFNodes(shape=[3, 3, 4, 3])
        torch.manual_seed(4)
        c = ns.topology.LocalConnection3D(X, Y, kernel_size=(3, 2, 4), stride=(2, 1, 3), n_filters=3, wmin=0.2, wmax=0.7)
        assert (tuple(c.kernel_size), tuple(c.stride), c.n_filters, c.in_channels, c.conv_size, c.conv_prod, c.kernel_prod) == \
            ((3, 2, 4), (2, 1, 3), 3, 2, (3, 4, 3), 36, 24)
        assert c.w.shape == (2, 108, 24) and float(c.w.min()) >= 0.2 and float(c.w.max()) <= 0.7
        torch.manual_seed(4)
        assert torch.equal(c.w, torch.rand(2, 108, 24).clamp(0.2, 0.7))
        assert c.b is None or c.b.numel() == 0
        c2 = ns.topology.LocalConnection3D(X, Y, kernel_size=2, stride=3, n_filters=1)
        assert tuple(c2.kernel_size) == (2, 2, 2) and tuple(c2.stride) == (3, 3, 3) and c2.conv_size == (2, 2, 4)


# ---- 6. tier selection -----------------------------------------------------------------------------------------------

def test_tier_selection():
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    net, inputs = _lc_net(B200, B=2, learning=True, rule="PostPre", nu=(1e-2, 1e-2), reduction=torch.sum)

    def tier(force, **opt):
        plan, keep = _plan.build_net(net, 2, {}, {}, {}, {}, {})
        opts = _abi.SnnRunOpts()
        opts.T, opts.B, opts.tier = 4, 2, force
        for k, v in opt.items():
            setattr(opts, k, v)
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
    """The library's own checks: a geometry that does not match the layers, a bias, a mask, a reward rule."""
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    net, _ = _lc_net(B200, B=2, learning=True, rule="PostPre", nu=(1e-2, 1e-2), reduction=torch.sum)
    m = torch.zeros(1, dtype=torch.uint8)
    for field, value, rc in (("dout", 3, _abi.SNN_ERR_BAD_ARG), ("kd", 5, _abi.SNN_ERR_BAD_ARG), ("pd", 1, _abi.SNN_ERR_BAD_ARG),
                             ("b", m.data_ptr(), _abi.SNN_ERR_BAD_ARG), ("mask", m.data_ptr(), _abi.SNN_ERR_UNSUPPORTED),
                             ("rule", _abi.SNN_RULE_MSTDP, _abi.SNN_ERR_UNSUPPORTED)):
        plan, keep = _plan.build_net(net, 2, {}, {}, {}, {}, {})
        setattr(plan.conns[0], field, value)
        opts = _abi.SnnRunOpts()
        opts.T, opts.B = 4, 2
        assert int(emu.lib().snn_b200_workspace_bytes(C.byref(plan), C.byref(opts))) == 0, field
        assert int(emu.lib().snn_b200_run_window(C.byref(plan), C.byref(opts), None, 0, None)) == rc, field


# ---- 7. the target reset ---------------------------------------------------------------------------------------------

def test_reset_resets_the_target():
    import emu

    net, inputs = _lc_net(B200, B=1)
    with emu.EmuBackend():
        net.run(inputs=inputs, time=4, inject_v={"Y": torch.full((16,), 3.0)})
    Y = net.layers["Y"]
    assert not torch.equal(Y.v, torch.full_like(Y.v, Y.rest))
    net.connections[("X", "Y")].reset_state_variables()
    assert torch.equal(Y.v, torch.full_like(Y.v, Y.rest)) and not Y.x.any() and not Y.s.any()


# ---- 8. the reference's own objects through the ABI -----------------------------------------------------------------

@pytest.mark.parametrize("case", ["c2_WeightDependentPostPre", "c2_Hebbian"])
def test_reference_binding_runs_the_references_network(case):
    ref = _reference()
    if ref is None:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb
    import local3d_oracle

    (a, inputs, T), (b, _, _) = ln.build_case(ref, case), ln.build_case(ref, case)
    a.run(inputs={"X": inputs["X"][0].clone()}, time=T)
    assert rb.run_window(b, {"X": inputs["X"][0].clone()}, time=T, library=local3d_oracle.lib()) == 0
    sa, sb = ln.state(a), ln.state(b)
    for k in (k for k in sa if "/" in k):   # (the binding runs the window; the reference's monitors are not its business)
        if k.endswith("s"):
            assert torch.equal(sa[k], sb[k]), k
        else:
            torch.testing.assert_close(sb[k], sa[k], rtol=1e-4, atol=1e-4, msg=k)
    assert sa["Ys"].sum() > 0


# ---- 9. the multi-GPU combine: sum + clamp on w, then the connection's own row normalize ------------------------------

def _dist_make(B):
    return ln.multi_net(B200, rule="PostPre", B=B, T=12)[0]


def _dist_inputs():
    return ln.multi_net(B200, B=8, T=12)[1]["X"]


def _dist_worker(rank, world, port, out):
    import torch.distributed as dist

    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from bindsnet_b200.distributed import ShardedWindowRunner
    from local3d_oracle import Local3dOracleBackend
    from test_distributed import _patch_cpu_combine

    _patch_cpu_combine()
    shard = _dist_inputs()[:, :, rank * 4:(rank + 1) * 4]
    net = _dist_make(4)
    with Local3dOracleBackend():
        runner = ShardedWindowRunner(net)
        for window in range(2):
            if window:
                net.reset_state_variables()
            runner.run({"X": shard[window]}, time=12)
    torch.save({f"{s}->{t}": c.w.detach().clone() for (s, t), c in net.connections.items()}, os.path.join(out, f"rank{rank}.pt"))
    dist.destroy_process_group()


def test_two_rank_combine_normalizes_local3d_rows(tmp_path):
    import numpy as np
    import torch.multiprocessing as mp
    from local3d_oracle import Local3dOracleBackend

    port = 35500 + (os.getpid() % 1000)
    mp.spawn(_dist_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    assert all(torch.equal(r0[k], r1[k]) for k in r0), "ranks diverged"

    x = _dist_inputs()
    nets = [_dist_make(4), _dist_make(4)]
    keys = list(nets[0].connections)
    w = {k: nets[0].connections[k].w.detach().clone() for k in keys}
    with Local3dOracleBackend():
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
            c.normalize()   # per [cin * n, K] row, not per column of an [n_src, n_tgt] matrix
            w[("X", "Y")] = c.w.detach().clone()
    assert np.array_equal(r0["X->Y"].numpy(), w[("X", "Y")].numpy())
    rows = r0["X->Y"].view(-1, 24).sum(1)
    torch.testing.assert_close(rows, torch.full_like(rows, 3.0), rtol=1e-5, atol=1e-5)
