"""MulticompartmentConnection pipelines with Probability / Mask / Intensity features besides the Weight (reference:
topology.py:437-479, topology_features.py:365-549, :724-769), run on the generic window kernel.  CPU tests: the oracle
against the live reference's stored results, the emulated kernel against the oracle bit for bit, equivalences that need
no oracle, and the host API.  "The oracle" here is tests/feature_oracle.c: the CPU oracle extended by the features.  The
stored reference results are regenerated with ``python tests/golden/gen_live.py test_mcc_features``; the reference's
Probability.compute is patched for the run to draw with snn_synapse_draw."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import cases
import helpers
import mcc_feature_nets as fn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

@reference_side(fn.LIVE_CASES)
def _live_features(ns, case):
    net, inputs, T = fn.live_net(ns, case)
    fn.patch_reference_probability(net, fn.SEED)
    net.run(inputs=inputs, time=T)
    return fn.live_state(net)


@reference_side([0])
def _live_default_values(ns, seed):
    """value=None: the features draw their own values from torch's CPU generator (topology_features.py:434-441,
    :513-524, :758-769) in pipeline order."""
    F, _ = fn.features(ns)
    torch.manual_seed(seed)
    X, Y = ns.nodes.Input(12), ns.nodes.LIFNodes(9)
    pipe = [F.Probability("p"), F.Mask("m"), F.Intensity("i"), F.Weight("w")]
    ns.topology.MulticompartmentConnection(source=X, target=Y, device="cpu", pipeline=pipe)
    return {"p": pipe[0].value.detach().clone(), "m": pipe[1].value.detach().clone(), "i": pipe[2].value.detach().float().clone(),
            "w": pipe[3].value.detach().clone()}


@pytest.mark.parametrize("case", fn.LIVE_CASES)
def test_oracle_matches_live_reference(case):
    from feature_oracle import FeatureOracleBackend

    ref = load(_live_features, case)
    net, inputs, T = fn.live_net(B200, case)
    with FeatureOracleBackend() as ob:
        net.run(inputs=inputs, time=T, one_spike_seed=fn.SEED)
    assert ob.err == 0
    ours = fn.live_state(net)
    assert torch.equal(ours["Ys"], ref["Ys"]), "spike rasters differ"
    assert ours["Ys"].sum() > 0
    for k in ("X/x", "Y/x", "Y/v", "Y/refrac_count", "XY/w", "YY/w"):
        torch.testing.assert_close(ours[k], ref[k], rtol=1e-5, atol=1e-4, msg=k)


def test_default_values_equal_the_references():
    ref = load(_live_default_values, 0)
    ours = _live_default_values(B200, 0)
    for k in ("p", "m", "i", "w"):
        assert torch.equal(ours[k], ref[k].to(ours[k].dtype)), k


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _emu_vs_oracle(build, env=None, windows=1, one_step=False):
    import emu
    from feature_oracle import FeatureOracleBackend

    outs = []
    for backend in (emu.EmuBackend, FeatureOracleBackend):
        net, inputs, T = build()
        net.force_tier = 1
        old = {k: os.environ.get(k) for k in (env or {})}
        os.environ.update(env if backend is emu.EmuBackend and env else {})
        try:
            with backend() as be:
                for w in range(windows):
                    net.run(inputs=inputs, time=T, one_step=one_step, one_spike_seed=fn.SEED + w)
                assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
        outs.append(fn.snapshot(net, T))
    return outs


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["prob_b4", "mask_b1", "int_mask", "reservoir"])
def test_emulated_kernel_bit_exact(case, env):
    a, b = _emu_vs_oracle(lambda: fn.live_net(B200, case), ENVS[env])
    helpers.assert_bit_identical(a, b, f"{case} {env}")
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("case", ["prob_b1", "mask_int"])
def test_emulated_kernel_one_step_and_two_windows_bit_exact(case):
    a, b = _emu_vs_oracle(lambda: fn.live_net(B200, case), ENVS["sms3"], windows=2, one_step=True)
    helpers.assert_bit_identical(a, b, f"{case} one_step, two windows")
    a, b = _emu_vs_oracle(lambda: fn.live_net(B200, case), ENVS["sms7"], windows=2)
    helpers.assert_bit_identical(a, b, f"{case} two windows")


def test_emulated_kernel_wide_source_bit_exact():
    a, b = _emu_vs_oracle(lambda: fn.wide_net(B200), ENVS["sms3"])
    helpers.assert_bit_identical(a, b, "9000-neuron source")
    assert a["M/Ys"].sum() > 0


def test_emulated_kernel_large_batch_bit_exact():
    a, b = _emu_vs_oracle(lambda: fn.big_batch_net(B200), ENVS["sms3"])
    helpers.assert_bit_identical(a, b, "B = 520")
    assert a["M/Ys"].sum() > 0


# ---- 3. equivalences that need no oracle (learning off) -----------------------------------------------------------

def _ff_net(pipeline_of, B=3, T=30, one_step=False, stepwise=False, user=False):
    """Input(50) -> LIFNodes(40) through the pipeline ``pipeline_of(F, g)`` returns, learning off."""
    from test_scripted_tier import MyLIF

    g = torch.Generator().manual_seed(5)
    net = B200.Network(dt=1.0, batch_size=B, learning=False)
    X = B200.nodes.Input(50)
    Y = MyLIF(40, thresh=-60.0, tc_decay=30.0, refrac=2) if user else B200.nodes.LIFNodes(40, thresh=-60.0, tc_decay=30.0, refrac=2)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    F, _ = fn.features(B200)
    net.add_connection(B200.topology.MulticompartmentConnection(source=X, target=Y, pipeline=pipeline_of(F, g)), "X", "Y")
    net.add_monitor(B200.monitors.Monitor(Y, ["s", "refrac_count"] if stepwise else ["s"], time=T), "Ys")
    x = (torch.rand(T, B, 50, generator=torch.Generator().manual_seed(6)) < 0.3).to(torch.uint8)
    return net, {"X": x}, T


def _run_emu(net, inputs, T, one_step=False):
    import emu

    with emu.EmuBackend() as be:
        net.run(inputs=inputs, time=T, one_step=one_step, one_spike_seed=fn.SEED)
    assert be.err == 0
    return {k: v for k, v in fn.snapshot(net, T).items() if not k.startswith("C/")}


def _same(a, b, what):
    helpers.assert_bit_identical(a, b, what)
    assert a["M/Ys"].sum() > 0, what


def _mats(g):
    w = 4.0 * torch.rand(50, 40, generator=g) - 1.0
    m = torch.rand(50, 40, generator=g) < 0.5
    i = 2.0 * torch.rand(50, 40, generator=g) - 1.0
    return w, m, i


def test_weight_mask_equals_masked_weight():
    a = _run_emu(*_ff_net(lambda F, g: [F.Weight("w", _mats(g)[0]), F.Mask("m", _mats(torch.Generator().manual_seed(5))[1])]))
    w, m, _ = _mats(torch.Generator().manual_seed(5))
    b = _run_emu(*_ff_net(lambda F, g: [F.Weight("w", w * m)]))
    _same(a, b, "[Weight(w), Mask(m)] vs [Weight(w * m)]")


def test_weight_intensity_equals_rounded_product():
    w, _, i = _mats(torch.Generator().manual_seed(5))
    a = _run_emu(*_ff_net(lambda F, g: [F.Intensity("i", i), F.Weight("w", w)]))
    b = _run_emu(*_ff_net(lambda F, g: [F.Weight("w", w * i)]))
    _same(a, b, "[Intensity(I), Weight(w)] vs [Weight(fl(w * I))]")


def test_probability_zero_one_equals_mask():
    w, m, _ = _mats(torch.Generator().manual_seed(5))
    a = _run_emu(*_ff_net(lambda F, g: [F.Probability("p", m.float()), F.Weight("w", w)]))
    b = _run_emu(*_ff_net(lambda F, g: [F.Mask("m", m), F.Weight("w", w)]))
    _same(a, b, "Probability in {0, 1} vs Mask")


def _prob_pipe(F, g):
    w, m, i = _mats(g)
    return [F.Probability("p", torch.rand(50, 40, generator=g)), F.Weight("w", w), F.Intensity("i", i)]


@pytest.mark.parametrize("one_step", [False, True])
def test_stepwise_equals_window(one_step):
    """A monitor on refrac_count sends the network through one-step windows (step_offset + t); the draws are the window's."""
    a = _run_emu(*_ff_net(_prob_pipe, stepwise=True), one_step=one_step)
    b = _run_emu(*_ff_net(_prob_pipe), one_step=one_step)
    a.pop("M/Ys"); b.pop("M/Ys")
    helpers.assert_bit_identical(a, b, "stepwise vs window")


@pytest.mark.parametrize("one_step", [False, True])
def test_scripted_tier_equals_window(one_step):
    """A user-defined population: the connection runs through its single-operator compute, drawing with the window's
    (seed, step, connection) — the emulated single operators and the oracle give the same bits, and the built-in LIF's
    window the same spikes."""
    from feature_oracle import FeatureOracleBackend
    import emu

    outs = []
    for user, backend in ((True, emu.EmuBackend), (True, FeatureOracleBackend), (False, emu.EmuBackend)):
        net, inputs, T = _ff_net(_prob_pipe, user=user)
        assert net._scripted_required() == user
        with backend():
            net.run(inputs=inputs, time=T, one_step=one_step, one_spike_seed=fn.SEED)
        outs.append(fn.snapshot(net, T))
    helpers.assert_bit_identical(outs[0], outs[1], "scripted tier: emulated single operators vs oracle")
    assert outs[0]["M/Ys"].sum() > 0
    assert np.array_equal(outs[0]["M/Ys"], outs[2]["M/Ys"])
    for k in outs[2]:
        np.testing.assert_allclose(outs[0][k].astype(np.float64), outs[2][k].astype(np.float64), rtol=1e-5, atol=1e-4, err_msg=k)


def test_window_draws_follow_the_seed():
    """Another seed, other masks: the runs differ; the same seed twice, the same bits."""
    a = _run_emu(*_ff_net(_prob_pipe))
    b = _run_emu(*_ff_net(_prob_pipe))
    helpers.assert_bit_identical(a, b, "same seed")
    net, inputs, T = _ff_net(_prob_pipe)
    import emu
    with emu.EmuBackend():
        net.run(inputs=inputs, time=T, one_spike_seed=fn.SEED + 1)
    assert not np.array_equal(fn.snapshot(net, T)["L/Y/v"], a["L/Y/v"])


# ---- 4. host API -------------------------------------------------------------------------------------------------

def test_refusals():
    F, ML = fn.features(B200)
    T = B200.topology
    X, Y = B200.nodes.Input(6), B200.nodes.LIFNodes(5)
    with pytest.raises(NotImplementedError, match="learning rule on a Probability"):
        F.Probability("p", torch.rand(6, 5), learning_rule=ML.PostPre, nu=(0.1, 0.1))
    with pytest.raises(NotImplementedError, match="norm on a Probability"):
        F.Probability("p", torch.rand(6, 5), norm=1.0)
    for cls, kw in ((F.Probability, {}), (F.Mask, {}), (F.Intensity, {}), (F.Weight, {})):
        with pytest.raises(NotImplementedError, match="sparse"):
            cls("f", sparse=True, **kw)
    for cls in (F.Bias, F.Degradation, F.MeanField):
        with pytest.raises(NotImplementedError, match="dense"):
            cls("f")
    for kind in ("Probability", "Mask", "Intensity"):
        make = {"Probability": lambda: F.Probability("p", torch.rand(6, 5)), "Mask": lambda: F.Mask("m", torch.rand(6, 5) < 0.5),
                "Intensity": lambda: F.Intensity("i", torch.rand(6, 5))}[kind]
        c = T.MulticompartmentConnection(source=X, target=Y, pipeline=[make(), F.Weight("w", torch.rand(6, 5)), make()])
        with pytest.raises(NotImplementedError, match=f"two {kind} features"):
            c.w
    c = T.MulticompartmentConnection(source=X, target=Y, pipeline=[F.Probability("p", torch.rand(6, 5))])
    with pytest.raises(NotImplementedError, match="exactly one Weight"):
        c.w
    # the reference's own failures
    with pytest.raises(AttributeError, match="dtype"):
        F.Probability("p", 0.5)
    with pytest.raises(AttributeError, match="dtype"):
        F.Intensity("i", 0.5)
    with pytest.raises(AssertionError):
        T.MulticompartmentConnection(source=X, target=Y, pipeline=[F.Probability("p", torch.tensor(0.5)), F.Weight("w", torch.rand(6, 5))])
    with pytest.raises(AssertionError, match="out of range"):
        F.Probability("p", torch.rand(6, 5) + 1.0)
    with pytest.raises(AssertionError, match="out of range"):
        F.Intensity("i", 3.0 * torch.ones(6, 5))
    with pytest.raises(AssertionError, match="less than 0"):
        F.Probability("p", torch.rand(6, 5), range=[-1, 1])
    with pytest.raises(AssertionError, match="bool"):
        F.Mask("m", torch.ones(6, 5))


def test_scalar_mask_is_folded():
    """Mask(True) lets every spike through (no mask in the plan); Mask(False) blocks every synapse."""
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    w, _, _ = _mats(torch.Generator().manual_seed(5))
    a = _run_emu(*_ff_net(lambda F, g: [F.Weight("w", w), F.Mask("m", True)]))
    b = _run_emu(*_ff_net(lambda F, g: [F.Weight("w", w)]))
    _same(a, b, "Mask(True)")
    net, inputs, T = _ff_net(lambda F, g: [F.Weight("w", w), F.Mask("m", True)])
    d = _abi.SnnConn()
    _plan.fill_conn(d, net.connections[("X", "Y")], 0, 1, 1.0, 3)
    assert not d.f_mask
    c = _run_emu(*_ff_net(lambda F, g: [F.Weight("w", w), F.Mask("m", False)]))
    assert c["M/Ys"].sum() == 0 and not np.any(c["L/Y/v"] > -65.0)


def test_seed_is_drawn_only_with_a_draw_on_the_path():
    import emu

    def consumed(pipeline_of, one_spike=False):
        net, inputs, T = _ff_net(pipeline_of)
        torch.manual_seed(1)
        before = torch.get_rng_state()
        with emu.EmuBackend():
            net.run(inputs=inputs, time=3)
        return not torch.equal(before, torch.get_rng_state()), net.last_one_spike_seed

    w, m, i = _mats(torch.Generator().manual_seed(5))
    assert consumed(lambda F, g: [F.Weight("w", w), F.Mask("m", m), F.Intensity("i", i)]) == (False, 0)
    took, seed = consumed(_prob_pipe)
    assert took and seed != 0
    torch.manual_seed(1)
    assert seed == int(torch.randint(0, 2**31 - 1, (1,)).item())


def test_fused_tiers_are_never_selected():
    """DiehlAndCook2015 goes to a fused kernel; with a Mask on its input connection it goes to the generic one, and a
    forced fused tier is refused."""
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    F, _ = fn.features(B200)
    net = B200.models.DiehlAndCook2015(n_inpt=64, n_neurons=16, batch_size=4)
    for l in net.layers.values():
        l.set_batch_size(4)

    def tier(force):
        plan, keep = _plan.build_net(net, 4, {}, {}, {}, {}, {})
        opts = _abi.SnnRunOpts()
        opts.T, opts.B, opts.tier = 5, 4, force
        return int(emu.lib().snn_b200_select_tier(C.byref(plan), C.byref(opts)))

    assert tier(0) in (2, 3)
    conn = net.connections[("X", "Ae")]
    conn.append_pipeline(F.Mask("m", torch.rand(64, 16) < 0.5))
    assert tier(0) == 1 and tier(1) == 1 and tier(2) == 0 and tier(3) == 0
    x = (torch.rand(5, 4, 64) < 0.2).to(torch.uint8)
    net.force_tier = 2
    with emu.EmuBackend(), pytest.raises(RuntimeError, match="not implemented"):
        net.run(inputs={"X": x}, time=5)


def test_standalone_compute_draws_a_fresh_seed_per_call():
    import emu
    from feature_oracle import FeatureOracleBackend

    net, _, _ = _ff_net(_prob_pipe)
    c = net.connections[("X", "Y")]
    s = torch.rand(4, 50, generator=torch.Generator().manual_seed(2)) < 0.5
    with emu.EmuBackend():
        torch.manual_seed(3)
        a1, a2 = c.compute(s), c.compute(s)
    with FeatureOracleBackend():
        torch.manual_seed(3)
        b1, b2 = c.compute(s), c.compute(s)
    assert torch.equal(a1.view(torch.int32), b1.view(torch.int32)) and torch.equal(a2.view(torch.int32), b2.view(torch.int32))
    assert not torch.equal(a1, a2)
    assert torch.equal(a1[0], a1[0]) and not torch.equal(a1[0], a1[1])


def test_draw_twins_agree():
    """The Python twin (bindsnet_b200._abi), the vectorised test twin and the C definition (through the oracle's compute
    with w = 1, one spiking row) give the same draws."""
    from bindsnet_b200 import _abi
    import feature_oracle

    ns, nt = 7, 300
    p = torch.rand(ns, nt, generator=torch.Generator().manual_seed(4))
    h = feature_oracle.draw_matrix(99, 5, 3, ns, nt)
    for i in range(ns):
        for j in range(0, nt, 37):
            assert int(h[i, j]) == _abi.synapse_draw(99, 5, 3, i, j)
            assert _abi.synapse_transmits(int(h[i, j]), float(p[i, j])) == bool(feature_oracle.transmit_matrix(p.numpy(), 99, 5, 3)[i, j])
    lib = feature_oracle.lib()
    w = torch.ones(ns, nt)
    d = _abi.SnnConn()
    d.kind, d.w, d.f_prob = _abi.SNN_CONN_MCC, w.data_ptr(), p.data_ptr()
    d.draw_seed, d.draw_step, d.draw_conn = 99, 5, 3
    for i in range(ns):
        s = torch.zeros(1, ns, dtype=torch.uint8)
        s[0, i] = 1
        out = torch.empty(1, nt)
        assert lib.snn_oracle_conn_compute(C.byref(d), ns, nt, 1, s.data_ptr(), out.data_ptr()) == 0
        expect = torch.from_numpy(feature_oracle.transmit_matrix(p.numpy(), 99, 5, 3)[i])
        assert torch.equal(out[0], expect)
    # the stream is apart from the one_spike tie-break's under the same seed
    assert _abi.synapse_draw(1, 0, 0, 0, 0) != _abi.one_spike_hash(1, 0, 0, 0, 0)


def test_transmitted_fraction_follows_p():
    """CPU-sized distribution check of the draw: per p bin within 5 sigma of p."""
    import feature_oracle

    g = np.random.default_rng(0)
    p = g.random((512, 512)).astype(np.float32)
    tr = feature_oracle.transmit_matrix(p, 7, 0, 0)
    for lo in np.arange(0.0, 1.0, 0.1):
        sel = (p >= lo) & (p < lo + 0.1)
        mean_p = p[sel].mean()
        sigma = np.sqrt((p[sel] * (1 - p[sel])).sum()) / sel.sum()
        assert abs(tr[sel].mean() - mean_p) < 5 * sigma + 1e-6, lo


def test_reference_binding_runs_the_references_feature_network():
    """The reference's own feature pipelines, their ABI filled by reference_binding and run by the feature oracle, against
    the reference's own run with its Probability.compute patched to the shared draw."""
    try:
        ref = cases.namespace("reference")
    except ImportError:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb
    import feature_oracle

    for case in ("prob_b4", "mask_int"):
        a, inputs, T = fn.live_net(ref, case)
        b, _, _ = fn.live_net(ref, case)
        fn.patch_reference_probability(a, fn.SEED)
        a.run(inputs={k: v.clone() for k, v in inputs.items()}, time=T)
        assert rb.run_window(b, {k: v.clone() for k, v in inputs.items()}, time=T, seed=fn.SEED, library=feature_oracle.lib()) == 0
        sa, sb = fn.live_state(a), fn.live_state(b)
        for k in ("Y/v", "Y/x", "X/x", "XY/w", "YY/w"):
            torch.testing.assert_close(sb[k], sa[k], rtol=1e-5, atol=1e-4, msg=f"{case} {k}")
