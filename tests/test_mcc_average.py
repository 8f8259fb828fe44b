"""MCC_learning.PostPre with average_update / continues_update on a MulticompartmentConnection's Weight (reference:
MCC_learning.py:210-302), run on the generic window kernel.  CPU tests: the oracle against the live reference's stored
results, the emulated kernel against the oracle bit for bit, the equivalences average_update=1 == no averaging and
standalone update() == a torch restatement, refusals and tier selection.  "The oracle" here is
tests/mcc_average_oracle.c.  The stored reference results are regenerated with
``python tests/golden/gen_live.py test_mcc_average``."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import cases
import helpers
import mcc_average_nets as an
from live_golden import load, reference_side
from mcc_feature_nets import snapshot

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

@reference_side(an.LIVE_CASES)
def _live_average(ns, case):
    net, inputs, T = an.live_net(ns, case)
    return an.run_windows(net, inputs, T, reference=True)


@pytest.mark.parametrize("case", an.LIVE_CASES)
def test_oracle_matches_live_reference(case):
    from mcc_average_oracle import AverageOracleBackend

    ref = load(_live_average, case)
    net, inputs, T = an.live_net(B200, case)
    w0 = an.rule_of(net.connections[("X", "Y")]).feature_value.detach().clone()
    with AverageOracleBackend() as ob:
        ours = an.run_windows(net, inputs, T)
    assert ob.err == 0
    for k in ("0", "2"):
        assert torch.equal(ours[f"{k}/Ys"], ref[f"{k}/Ys"]), f"window {k}: spike rasters differ"
        assert ours[f"{k}/Ys"].sum() > 0
        assert torch.equal(ours[f"{k}/idx"], ref[f"{k}/idx"]), f"window {k}: buffer indices differ"
        for name in ["Y/v", "XY/w", "YY/w", "buf_pre", "buf_post"]:
            torch.testing.assert_close(ours[f"{k}/{name}"], ref[f"{k}/{name}"], rtol=1e-4, atol=1e-4, msg=f"window {k} {name}")
    assert not torch.equal(ours["2/XY/w"], w0), "the Weight did not learn"
    p = an.params(case)
    assert (ours["2/buf_pre"].abs().sum() > 0) == (p["nu"][0] != 0)
    assert (ours["2/buf_post"].abs().sum() > 0) == (p["nu"][1] != 0)


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _emu_vs_oracle(case, env, one_step=False, stepwise=False, B=None, n_in=40, n=30):
    import emu
    from mcc_average_oracle import AverageOracleBackend

    outs = []
    for backend in (emu.EmuBackend, AverageOracleBackend):
        net, inputs, T = an.live_net(B200, case, B=B, n_in=n_in, n=n)
        net.force_tier = 1
        if stepwise:   # a monitor on a state the kernel does not record: one-step windows
            net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["s", "refrac_count"], time=T), "Yr")
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env if backend is emu.EmuBackend else {})
        try:
            with backend() as be:
                an.run_windows(net, inputs, T, one_step=one_step)
                assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
        outs.append(an.full_snapshot(net, T))
    return outs


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["k3", "k7c", "b4_mean", "pw", "wm", "pre_only", "post_only", "decay"])
def test_emulated_kernel_bit_exact(case, env):
    a, b = _emu_vs_oracle(case, ENVS[env])
    helpers.assert_bit_identical(a, b, f"{case} {env}")
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("mode", ["one_step", "stepwise", "stepwise_one_step"])
@pytest.mark.parametrize("case", ["k3", "b4_sum", "t5"])
def test_emulated_kernel_one_step_and_stepwise_bit_exact(case, mode):
    a, b = _emu_vs_oracle(case, ENVS["sms3"], one_step="one_step" in mode, stepwise="stepwise" in mode)
    helpers.assert_bit_identical(a, b, f"{case} {mode}")


def test_emulated_kernel_large_batch_odd_T_bit_exact():
    """B = 520 (more than 16 words of samples, the trace tile no longer staged in shared memory) and T = 5."""
    a, b = _emu_vs_oracle("t5", ENVS["sms3"], B=520, n_in=70, n=40)
    helpers.assert_bit_identical(a, b, "B=520")
    assert a["M/Ys"].sum() > 0


def test_two_windows_without_reset_bit_exact():
    import emu
    from mcc_average_oracle import AverageOracleBackend

    outs = []
    for backend in (emu.EmuBackend, AverageOracleBackend):
        net, inputs, T = an.live_net(B200, "k7")
        with backend() as be:
            for k in range(3):
                net.run(inputs=an.window_inputs(inputs, T, k), time=T, one_spike_seed=5 + k)
            assert be.err == 0
        outs.append(an.full_snapshot(net, T))
    helpers.assert_bit_identical(outs[0], outs[1], "three windows")
    assert list(outs[0]["R/idx"]) == [3 * 8 % 7] * 2


# ---- 3. equivalences (no oracle) -------------------------------------------------------------------------------------

def _plain_twin(case, cont):
    """The case's network with average_update=1 (continues or not) and without averaging."""
    nets = []
    for k in (1, 0):
        p = an.params(case)
        net, inputs, T = an.live_net(B200, case)
        c = net.connections[("X", "Y")]
        r = an.rule_of(c)
        if k == 0:
            r.average_update = 0
        else:
            r.continues_update = cont
            assert r.average_update == p["k"]
            ML = sys.modules[type(r).__module__]
            fresh = ML.PostPre(connection=c, feature_value=r.feature_value, range=[r.min, r.max], nu=(float(r.nu[0]), float(r.nu[1])),
                               reduction=p["reduction"], decay=p["decay"], average_update=1, continues_update=cont)
            [f for f in c.pipeline if type(f).__name__ == "Weight"][0].learning_rule = fresh
        nets.append((net, inputs, T))
    return nets


@pytest.mark.parametrize("cont", [False, True])
@pytest.mark.parametrize("case", ["k3", "b4_mean", "pw"])
def test_average_update_one_equals_no_averaging(case, cont):
    import emu

    outs = []
    for net, inputs, T in _plain_twin(case, cont):
        with emu.EmuBackend() as be:
            for k in range(2):
                net.run(inputs=an.window_inputs(inputs, T, k), time=T, one_spike_seed=9 + k)
        assert be.err == 0
        outs.append(snapshot(net, T))
    helpers.assert_bit_identical(outs[0], outs[1], f"average_update=1 continues={cont} vs plain")


def _torch_update(w, bufs, idx, s_src, x_src, s_tgt, x_tgt, nu, k, cont, dt, reduction, decay, lo, hi):
    """PostPre._connection_update (MCC_learning.py:224-302) with averaging, in torch on the CPU, in the fixed order of
    include/snn_b200.h (ascending slot sums from +0; the skipped zero slots leave them as they are)."""
    B = s_src.shape[0]
    red = (lambda t: t.sum(0)) if reduction != "mean" else (lambda t: t.sum(0) / float(B))
    w = w.clone()
    for side in (0, 1):
        if nu[side] == 0:
            continue
        if side == 0:
            term = red(s_src.float().unsqueeze(2) * (x_tgt * nu[0]).unsqueeze(1))
        else:
            term = red(x_src.unsqueeze(2) * (s_tgt.float() * nu[1]).unsqueeze(1))
        bufs[side][idx[side]] = term
        idx[side] = (idx[side] + 1) % k
        if cont or idx[side] == 0:
            s = torch.zeros_like(w)
            for q in range(k):
                s = s + bufs[side][q]
            d = (s / float(k)) * dt
            w = w - d if side == 0 else w + d
    if decay != 1.0:
        w = w * decay
    return w.clamp(lo, hi)


@pytest.mark.parametrize("cont", [False, True])
@pytest.mark.parametrize("B,reduction", [(1, None), (3, "sum"), (3, "mean")])
def test_standalone_update_equals_torch_restatement(B, reduction, cont):
    """conn.update(learning=True) (the scripted and stepwise paths' call) against the torch restatement, step by step;
    the MCC connection's dt is not 1."""
    import emu

    F, ML = an.features(B200)
    g = torch.Generator().manual_seed(11 + B)
    X, Y = B200.nodes.Input(37, traces=True), B200.nodes.LIFNodes(45, traces=True)
    net = B200.Network(dt=0.5, batch_size=B)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    k, nu = 3, (0.07, 0.05)
    kw = {"reduction": torch.mean if reduction == "mean" else torch.sum} if reduction else {}
    wt = F.Weight("w", 0.9 * torch.rand(37, 45, generator=g), learning_rule=ML.PostPre, nu=nu, range=[0.0, 0.9], decay=1e-2, **kw)
    c = B200.topology.MulticompartmentConnection(source=X, target=Y, pipeline=[wt], average_update=k, continues_update=cont)
    net.add_connection(c, "X", "Y")
    r = wt.learning_rule
    w = c.w.clone()
    bufs, idx = [torch.zeros(k, 37, 45), torch.zeros(k, 37, 45)], [0, 0]
    with emu.EmuBackend() as be:
        for step in range(7):
            X.s = torch.rand(B, 37, generator=g) < 0.3
            Y.s = torch.rand(B, 45, generator=g) < 0.2
            X.x = torch.rand(B, 37, generator=g) * (torch.rand(B, 37, generator=g) < 0.5)
            Y.x = torch.rand(B, 45, generator=g)
            w = _torch_update(w, bufs, idx, X.s, X.x, Y.s, Y.x, nu, k, cont, float(c.dt), reduction, r.decay, 0.0, 0.9)
            c.update(learning=True)
            assert be.err == 0
            assert np.array_equal(c.w.numpy().view(np.uint32), w.numpy().view(np.uint32)), f"step {step}"
            assert [r.average_buffer_index_pre, r.average_buffer_index_post] == idx
            assert torch.equal(r.average_buffer_pre, bufs[0]) and torch.equal(r.average_buffer_post, bufs[1])


# ---- 4. host API, refusals, tier selection -------------------------------------------------------------------------

def test_rule_state_names_and_shapes():
    F, ML = an.features(B200)
    X, Y = B200.nodes.Input(6, traces=True), B200.nodes.LIFNodes(5, traces=True)
    w = F.Weight("w", torch.rand(6, 5), learning_rule=ML.PostPre)
    B200.topology.MulticompartmentConnection(source=X, target=Y, pipeline=[w], average_update=4, continues_update=True)
    r = w.learning_rule
    assert (r.average_update, r.continues_update) == (4, True)
    assert r.average_buffer_pre.shape == r.average_buffer_post.shape == (4, 6, 5)
    assert (r.average_buffer_index_pre, r.average_buffer_index_post) == (0, 0)
    w2 = F.Weight("w", torch.rand(6, 5), learning_rule=ML.PostPre)
    B200.topology.MulticompartmentConnection(source=X, target=Y, pipeline=[w2])
    assert w2.learning_rule.average_update == 0 and not hasattr(w2.learning_rule, "average_buffer_pre")


def test_refusals():
    F, ML = an.features(B200)
    X, Y = B200.nodes.Input(6, traces=True), B200.nodes.LIFNodes(5, traces=True)
    for rule in (ML.MSTDP, ML.MSTDPET):
        with pytest.raises(NotImplementedError):
            B200.topology.MulticompartmentConnection(source=X, target=Y, average_update=3,
                                                     pipeline=[F.Weight("w", torch.rand(6, 5), learning_rule=rule)])
    with pytest.raises(NotImplementedError, match="enforce_polarity"):
        B200.topology.MulticompartmentConnection(source=X, target=Y, average_update=3, pipeline=[
            F.Weight("w", torch.rand(6, 5), learning_rule=ML.PostPre, enforce_polarity=True)])


def test_sharded_runner_refuses_averaging():
    from bindsnet_b200 import distributed

    net, inputs, T = an.live_net(B200, "k3")
    with pytest.raises(NotImplementedError, match="average_update"):
        distributed.ShardedWindowRunner(net)._learned()


def test_tier_selection_and_forced_fused_tiers():
    """A plan with an averaged rule runs on tier 1; a forced fused tier is refused.  The metric's network (no averaging)
    keeps its tier."""
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    net, inputs, T = an.live_net(B200, "k3")
    plan, keep = _plan.build_net(net, 1, {}, {}, {}, {}, {})
    assert plan.conns[0].rule == _abi.SNN_RULE_MCC_POSTPRE | _abi.SNN_RULE_AVG and plan.conns[0].avg_k == 3
    lib = emu.lib()
    opts = _abi.SnnRunOpts()
    opts.T, opts.B = T, 1
    for tier, want in ((0, 1), (1, 1), (2, 0), (3, 0)):
        opts.tier = tier
        assert lib.snn_b200_select_tier(C.byref(plan), C.byref(opts)) == want, tier
    plan.conns[0].avg_k = 0
    assert lib.snn_b200_run_window(C.byref(plan), C.byref(opts), None, 0, None) == _abi.SNN_ERR_BAD_ARG
    plan.conns[0].avg_k = 3
    plan.conns[0].rule = _abi.SNN_RULE_MSTDP | _abi.SNN_RULE_AVG
    assert lib.snn_b200_run_window(C.byref(plan), C.byref(opts), None, 0, None) == _abi.SNN_ERR_UNSUPPORTED


@pytest.mark.parametrize("case", ["k3", "b4_sum", "post_only"])
def test_reference_binding_fills_the_averaging_state(case):
    """The reference's own PostPre (its buffers and indices) described through the ABI by reference_binding and run by the
    oracle library equals the same network built from this package's classes, run by the oracle, over three windows.
    Skipped where the reference is not present."""
    try:
        ref = cases.namespace("reference")
    except Exception as e:  # pragma: no cover
        pytest.skip(f"the reference is missing: {e}")
    from bindsnet_b200 import reference_binding as rb
    import mcc_average_oracle
    from mcc_average_oracle import AverageOracleBackend

    states = []
    for ns in (ref, B200):
        net, inputs, T = an.live_net(ns, case)
        for k in range(3):
            x = an.window_inputs(inputs, T, k)
            if ns is ref:
                assert rb.run_window(net, x, time=T, seed=SEED_W + k, library=mcc_average_oracle.lib()) == 0
            else:
                with AverageOracleBackend() as ob:
                    net.run(inputs=x, time=T, one_spike_seed=SEED_W + k)
                assert ob.err == 0
        st = an.rule_state(net)
        st["w"] = an.rule_of(net.connections[("X", "Y")]).feature_value.detach().clone()
        states.append({k: v.numpy() for k, v in st.items()})
    helpers.assert_bit_identical(states[0], states[1], case)


SEED_W = 21
