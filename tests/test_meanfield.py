"""MeanFieldConnection (reference: topology.py:1920-2006) on the generic window kernel.  CPU tests: construction parity
with the reference, the oracle (tests/meanfield_oracle.c, the CPU oracle extended by the mean-field connection) against
the live reference's stored results, the emulated kernel against the oracle bit for bit, the standalone compute,
refusals and tier selection.  The stored reference results are regenerated with
``python tests/golden/gen_live.py test_meanfield``."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

import cases
import meanfield_nets as mn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")
# (wmin, wmax) forms of the reference's test_weights and of the two branches of the initial draw
BOUNDS = {"none": {}, "scalar": dict(wmin=-0.5, wmax=2.0), "inf_lo": dict(wmax=1.5), "tensor": dict(wmin=torch.tensor([0.0, -1.0, 0.5, 0.0]),
          wmax=torch.tensor([1.0, 1.0, 3.0, 2.0])), "tensor_inf": dict(wmin=torch.tensor([0.0, -np.inf, 0.5, 0.0]), wmax=1.0)}
W_GIVEN = {"none": None, "plain": torch.tensor([5.0, -5.0, 0.25, 1.0])}


def _build(ns, bounds, w, **kw):
    src, tgt = ns.nodes.Input(shape=[1, 6, 6]), ns.nodes.LIFNodes(shape=[4])
    torch.manual_seed(11)
    extra = dict(BOUNDS[bounds])
    if W_GIVEN[w] is not None:
        extra["w"] = W_GIVEN[w].clone()
    return ns.topology.MeanFieldConnection(src, tgt, **extra, **kw)


# ---- 1. construction parity ------------------------------------------------------------------------------------------

@reference_side([f"{b}_{w}" for b in BOUNDS for w in W_GIVEN])
def _live_construct(ns, case):
    b, w = case.rsplit("_", 1)
    c = _build(ns, b, w, weight_decay=0.25)
    return {"w": c.w.detach().clone(), "reduction": torch.tensor(float(c.reduction)), "weight_decay": torch.tensor(float(c.weight_decay)),
            "rule_decay": torch.tensor(float(c.update_rule.weight_decay))}


@pytest.mark.parametrize("bounds", list(BOUNDS))
@pytest.mark.parametrize("w", list(W_GIVEN))
def test_construction_matches_reference(bounds, w):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        c = _build(B200, bounds, w, weight_decay=0.25)
    ref = load(_live_construct, f"{bounds}_{w}")
    assert torch.equal(c.w.detach(), ref["w"])
    assert float(c.reduction) == float(ref["reduction"]) == 0.25
    assert float(c.weight_decay) == float(ref["weight_decay"]) == 0.0
    assert float(c.update_rule.weight_decay) == float(ref["rule_decay"]) == 1.0


def test_construction_errors():
    ns = B200
    src, tgt = ns.nodes.Input(n=4), ns.nodes.LIFNodes(n=4)
    with pytest.raises(TypeError):
        ns.topology.MeanFieldConnection(src, tgt, reduction=torch.sum)
    with pytest.raises(NotImplementedError, match="norm"):
        ns.topology.MeanFieldConnection(src, tgt, norm=1.0)
    with pytest.raises(NotImplementedError):
        ns.topology.MeanFieldConnection(src, tgt, w_dtype=torch.float16)
    for rule in (ns.learning.PostPre, ns.learning.WeightDependentPostPre, ns.learning.Hebbian):
        with pytest.raises(AssertionError):   # traces first, as in the reference
            ns.topology.MeanFieldConnection(src, tgt, update_rule=rule, wmin=0.0, wmax=1.0)
        with pytest.raises(NotImplementedError):
            ns.topology.MeanFieldConnection(ns.nodes.Input(n=4, traces=True), ns.nodes.LIFNodes(n=4, traces=True), update_rule=rule,
                                            wmin=0.0, wmax=1.0)
    for rule in (ns.learning.MSTDP, ns.learning.MSTDPET):
        with pytest.raises(NotImplementedError):
            ns.topology.MeanFieldConnection(src, tgt, update_rule=rule)
    c = ns.topology.MeanFieldConnection(src, tgt, update_rule=ns.learning.NoOp, w=torch.tensor(0.5))
    c.normalize()
    assert float(c.w) == 0.5


def test_test_weights_loop_of_the_reference():
    """The reference's test_weights for this class (test/network/test_connections.py:185-191): NoOp with no, scalar,
    tensor and +-inf-masked bounds, defined values in place of torch.Tensor(*shape)'s uninitialised memory."""
    ns = B200
    src, tgt = ns.nodes.Input(shape=[1, 28, 28]), ns.nodes.LIFNodes(shape=[1, 26, 26])
    shape = (1, 26)
    wmins = [None, -0.5, torch.full(shape, -0.5), torch.where(torch.arange(26).view(shape) % 2 == 0, -np.inf, -0.5)]
    wmaxs = [None, 0.75, torch.full(shape, 0.75), torch.where(torch.arange(26).view(shape) % 3 == 0, np.inf, 0.75)]
    for wmin, wmax in zip(wmins, wmaxs):
        kw = {k: v for k, v in (("wmin", wmin), ("wmax", wmax)) if v is not None}
        c = ns.topology.MeanFieldConnection(src, tgt, decay=1, update_rule=ns.learning.NoOp, **kw)
        assert c.w.dtype == torch.float32
        if wmin is not None:
            assert bool((c.w >= c.wmin).all()) and bool((c.w <= c.wmax).all())


# ---- 2. the oracle against the live reference ------------------------------------------------------------------------

@reference_side(mn.LIVE_CASES)
def _live_mf(ns, case):
    net, inputs, T, kw = mn.mf_net(ns, case)
    return mn.flat(mn.run_two_windows(net, inputs, T, **kw))


def _check_against(ref, ours, what):
    for k, v in ref.items():
        o = ours[k]
        assert o.shape == v.shape, (what, k)
        if k.endswith("s") or k.endswith("Yv") or k.endswith("/w"):   # spikes, McCullochPitts' raw input, weights
            assert torch.equal(o.float(), v.float()), f"{what}: {k} differs"
        else:
            torch.testing.assert_close(o.float(), v.float(), rtol=1e-5, atol=1e-4, msg=f"{what}: {k}")


@pytest.mark.parametrize("case", mn.LIVE_CASES)
def test_oracle_matches_live_reference(case):
    from meanfield_oracle import MeanFieldOracleBackend

    net, inputs, T, kw = mn.mf_net(B200, case)
    with MeanFieldOracleBackend() as ob:
        ours = mn.flat(mn.run_two_windows(net, inputs, T, **kw))
    assert ob.err == 0
    _check_against(load(_live_mf, case), ours, case)
    assert ours["w1/Yv"].abs().sum() > 0


def test_silent_sample_receives_the_batch_mean():
    """Sample 0 of the Input never spikes, yet its McCullochPitts input is fl(mean * w) of the whole batch's spikes."""
    from meanfield_oracle import MeanFieldOracleBackend

    net, inputs, T, kw = mn.mf_net(B200, "b3_in_n_mf")
    w = net.connections[("X", "Y")].w.detach().clone()
    with MeanFieldOracleBackend():
        ours = mn.flat(mn.run_two_windows(net, inputs, T))
    x = inputs["X"][0].float()
    v0 = ours["w0/Yv"][:, 0]   # [T, C, W] of the silent sample
    for t in range(1, T):
        mean = x[t - 1].mean()
        assert torch.equal(v0[t], (mean * w).expand(2, 4)), t
    assert bool((v0[1:] != 0).any())


# ---- 3. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

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
    from meanfield_oracle import MeanFieldOracleBackend

    outs = []
    for backend in (emu.EmuBackend, MeanFieldOracleBackend):
        net, inputs, T, rkw = build()
        net.force_tier = 1

        def run():
            with backend() as be:
                outs.append(mn.flat(mn.run_two_windows(net, inputs, T, **rkw, **kw)))
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
@pytest.mark.parametrize("case", mn.LIVE_CASES)
def test_emulated_kernel_bit_exact(case, env):
    _emu_vs_oracle(lambda: mn.mf_net(B200, case), ENVS[env])


@pytest.mark.parametrize("case", ["b3_in_n_mf", "b3_lif_n_dense_mf", "b8_dc1_c1_mf", "b3_self_n_mf_dense", "b8_in_full_mf_dense"])
def test_emulated_kernel_one_step_bit_exact(case):
    _emu_vs_oracle(lambda: mn.mf_net(B200, case), one_step=True)


@pytest.mark.parametrize("B,T", [(520, 5), (7, 13)])
def test_emulated_kernel_batch_sizes_bit_exact(B, T):
    _emu_vs_oracle(lambda: mn.mf_net(B200, f"b{B}_lif_full_mf_dense", T=T))


@pytest.mark.parametrize("one_step", [False, True])
def test_emulated_kernel_consecutive_windows_bit_exact(one_step):
    import emu
    from meanfield_oracle import MeanFieldOracleBackend

    outs = []
    for backend in (emu.EmuBackend, MeanFieldOracleBackend):
        net, inputs, T, kw = mn.mf_net(B200, "b3_self_n_dense_mf", T=9)
        net.force_tier = 1
        with backend():
            outs.append(mn.flat(mn.run_two_windows(net, inputs, T, reset=False, one_step=one_step)))
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


def test_stepwise_equals_window():
    """T one-step windows reproduce one T-step window: the spike count of step -1 comes from the layers' s."""
    import emu

    res = []
    for stepwise in (False, True):
        net, inputs, T, kw = mn.mf_net(B200, "b3_lif_c1_dense_mf", T=11)
        net.force_tier = 1
        with emu.EmuBackend():
            x = inputs["X"][0]
            if stepwise:
                for t in range(T):
                    net.run(inputs={"X": x[t:t + 1].clone()}, time=1)
            else:
                net.run(inputs={"X": x.clone()}, time=T)
        res.append(mn.state(net, monitors=False))
    for k in res[0]:
        assert torch.equal(res[0][k], res[1][k]), k


@pytest.mark.parametrize("one_step", [False, True])
def test_scripted_tier_equals_window(one_step):
    """A user-defined population sends the network to the scripted tier, which steps the single operators; a mean-field
    connection there gives what the window gives."""
    import emu
    from meanfield_oracle import MeanFieldOracleBackend

    def build(user):
        ns = B200
        B, T = 3, 10
        g = torch.Generator().manual_seed(5)
        net = ns.Network(dt=1.0, batch_size=B, learning=False)
        X = ns.nodes.Input(n=16)
        if user:
            from test_scripted_tier import MyLIF
            A = MyLIF(n=8, thresh=-62.0)
        else:
            A = ns.nodes.LIFNodes(n=8, thresh=-62.0)
        Y = ns.nodes.McCullochPitts(shape=[2, 4], thresh=0.05)
        for name, layer in (("X", X), ("A", A), ("Y", Y)):
            net.add_layer(layer, name=name)
        net.add_connection(ns.topology.Connection(X, A, w=6.0 * torch.rand(16, 8, generator=g)), source="X", target="A")
        net.add_connection(ns.topology.MeanFieldConnection(A, Y, w=torch.rand(2, 1, generator=g) - 0.3), source="A", target="Y")
        net.add_connection(ns.topology.MeanFieldConnection(X, Y, w=torch.rand(B, 2, 4, generator=g)), source="X", target="Y")
        x = torch.bernoulli(0.3 * torch.ones(T, B, 16), generator=g).bool()
        return net, x, T

    outs = []
    for user, backend in ((True, emu.EmuBackend), (True, MeanFieldOracleBackend), (False, emu.EmuBackend)):
        net, x, T = build(user)
        with backend():
            net.run(inputs={"X": x.clone()}, time=T, one_step=one_step)
        outs.append({k: v for k, v in mn.state(net, monitors=False).items()})
    for o in outs[1:]:
        for k in outs[0]:
            assert torch.equal(outs[0][k], o[k]), k


# ---- 4. the standalone compute ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("form", ["0d", "n", "1w", "c1", "full"])
def test_standalone_compute(form):
    import emu

    B = 5
    g = torch.Generator().manual_seed(3)
    ns = B200
    src, tgt = ns.nodes.Input(n=37), ns.nodes.LIFNodes(shape=[2, 4])
    w = mn.w_of(form, B, g)
    c = ns.topology.MeanFieldConnection(src, tgt, w=w)
    s = torch.bernoulli(0.3 * torch.ones(B, 37), generator=g).bool()
    with emu.EmuBackend():
        out = c.compute(s)
    assert out.shape == w.shape
    assert torch.equal(out, s.float().mean() * w)


# ---- 5. refusals and tier selection ----------------------------------------------------------------------------------

def _small(ns, w, B=2, target_shape=(2, 4)):
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X, Y = ns.nodes.Input(n=6), ns.nodes.LIFNodes(shape=list(target_shape))
    net.add_layer(X, name="X")
    net.add_layer(Y, name="Y")
    net.add_connection(ns.topology.MeanFieldConnection(X, Y, w=w), source="X", target="Y")
    return net


def test_shape_errors_raise_before_anything_runs():
    import emu

    for w in (torch.ones(8), torch.ones(3, 2, 4)):
        net = _small(B200, w)
        with emu.EmuBackend():
            with pytest.raises(RuntimeError):
                net.run(inputs={"X": torch.zeros(3, 2, 6, dtype=torch.bool)}, time=3)


def test_large_batch_refused():
    import emu

    net = _small(B200, torch.tensor(1.0), B=1 << 22)   # B * n_src = 6 * 2^22 >= 2^24
    with emu.EmuBackend():
        with pytest.raises(NotImplementedError, match="2\\*\\*24"):
            net.run(inputs={"X": torch.zeros(1, 1 << 22, 6, dtype=torch.bool)}, time=1)


def test_masks_refused():
    import emu

    net = _small(B200, torch.tensor(1.0))
    with emu.EmuBackend():
        with pytest.raises(NotImplementedError, match="dense Connection only"):
            net.run(inputs={"X": torch.zeros(2, 2, 6, dtype=torch.bool)}, time=2, masks={("X", "Y"): torch.tensor(True)})


def test_tier_selection():
    """Tier 0 selects the generic kernel; a forced fused tier is refused (SNN_ERR_UNSUPPORTED)."""
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    net = _small(B200, torch.tensor(0.5))
    with emu.EmuBackend():
        d, keep = _plan.build_net(net, 2, {}, {}, {}, {}, {})
        for tier, want in ((0, 1), (1, 1), (2, 0), (3, 0)):
            o = _abi.SnnRunOpts()
            o.T, o.B, o.tier = 4, 2, tier
            assert emu.lib().snn_b200_select_tier(d, o) == want
        assert d.conns[0].kind == _abi.SNN_CONN_MEANFIELD


def test_reference_binding_with_the_references_objects():
    """reference_binding runs the reference's own MeanFieldConnection objects; the result equals the reference's."""
    from meanfield_oracle import lib
    from bindsnet_b200 import reference_binding

    ref = cases.namespace("reference")
    outs = []
    for bound in (False, True):
        net, inputs, T, kw = mn.mf_net(ref, "b3_lif_c1_dense_mf")
        if bound:
            assert reference_binding.run_window(net, {"X": inputs["X"][0].clone()}, T, library=lib()) == 0
        else:
            net.run(inputs={"X": inputs["X"][0].clone()}, time=T)
        outs.append(mn.state(net, monitors=False))
    for k in outs[0]:
        if k.endswith("s") or k.endswith("/w"):
            assert torch.equal(outs[0][k].float(), outs[1][k].float()), k
        else:
            torch.testing.assert_close(outs[0][k].float(), outs[1][k].float(), rtol=1e-5, atol=1e-4)
