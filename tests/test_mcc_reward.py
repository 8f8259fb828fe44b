"""MCC_learning.MSTDP and MSTDPET on a MulticompartmentConnection's Weight (reference: MCC_learning.py:392-738), with and
without Probability / Mask features, run on the generic window kernel.  CPU tests: the oracle against the live
reference's stored results, the emulated kernel against the oracle bit for bit, the equivalence with learning.MSTDP /
MSTDPET on a dense Connection, refusals and tier selection.  "The oracle" here is tests/mcc_reward_oracle.c.  The stored
reference results are regenerated with ``python tests/golden/gen_live.py test_mcc_reward``; the reference's
Probability.compute is patched for the run to draw with snn_synapse_draw."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import cases
import helpers
import mcc_reward_nets as rn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

@reference_side(rn.LIVE_CASES)
def _live_reward(ns, case):
    net, inputs, T = rn.live_net(ns, case)
    return rn.run_two_windows(net, inputs, T, case, reference=True)


@pytest.mark.parametrize("case", rn.LIVE_CASES)
def test_oracle_matches_live_reference(case):
    from mcc_reward_oracle import RewardOracleBackend

    ref = load(_live_reward, case)
    net, inputs, T = rn.live_net(B200, case)
    w0 = rn.rule_of(net.connections[("X", "Y")]).feature_value.detach().clone()
    with RewardOracleBackend() as ob:
        ours = rn.run_two_windows(net, inputs, T, case)
    assert ob.err == 0
    state = ["p_plus", "p_minus", "eligibility"] + (["eligibility_trace"] if case.endswith("et") else [])
    for k in ("0", "1"):
        assert torch.equal(ours[f"{k}/Ys"], ref[f"{k}/Ys"]), f"window {k}: spike rasters differ"
        assert ours[f"{k}/Ys"].sum() > 0
        for name in ["Y/v", "Y/x", "XY/w", "YY/w"] + state:
            torch.testing.assert_close(ours[f"{k}/{name}"], ref[f"{k}/{name}"], rtol=1e-4, atol=1e-5, msg=f"window {k} {name}")
        assert not torch.equal(ours[f"{k}/XY/w"], w0), "the Weight did not learn"
        for name in state:
            assert ours[f"{k}/{name}"].abs().sum() > 0, f"{name} stayed zero"
    assert not torch.equal(ours["0/XY/w"], ours["1/XY/w"])
    assert not torch.equal(ours["0/p_plus"], ours["1/p_plus"])


def test_network_reset_leaves_the_eligibility_trace_alone():
    """Weight.reset_state_variables does nothing (topology_features.py:630-631), so Network.reset_state_variables never
    reaches MSTDPET.reset_state_variables; the rule's own call zeroes the eligibility and its trace."""
    from mcc_reward_oracle import RewardOracleBackend

    net, inputs, T = rn.live_net(B200, "wm_et")
    with RewardOracleBackend():
        net.run(inputs=rn.window_inputs(inputs, T, 0), time=T, **rn.WINDOW_KWARGS[0])
    r = rn.rule_of(net.connections[("X", "Y")])
    before = {k: v.clone() for k, v in rn.rule_state(net).items()}
    net.reset_state_variables()
    for k, v in rn.rule_state(net).items():
        assert torch.equal(v, before[k]), k
    assert r.eligibility_trace.abs().sum() > 0 and r.eligibility.abs().sum() > 0
    r.reset_state_variables()
    assert r.eligibility_trace.abs().sum() == 0 and r.eligibility.abs().sum() == 0
    assert torch.equal(r.p_plus, before["p_plus"])


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _emu_vs_oracle(case, env, one_step=False, stepwise=False):
    import emu
    from mcc_reward_oracle import RewardOracleBackend

    outs = []
    for backend in (emu.EmuBackend, RewardOracleBackend):
        net, inputs, T = rn.live_net(B200, case, T=12)
        net.force_tier = 1
        if stepwise:   # a monitor on a state the kernel does not record: one-step windows
            net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["s", "refrac_count"], time=T), "Yr")
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env if backend is emu.EmuBackend else {})
        try:
            with backend() as be:
                rn.run_two_windows(net, inputs, T, case, one_step=one_step)
                assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
        outs.append(rn.full_snapshot(net, T))
    return outs


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["w_b4", "pw_b4", "wm_et", "decay_range"])
def test_emulated_kernel_bit_exact(case, env):
    a, b = _emu_vs_oracle(case, ENVS[env])
    helpers.assert_bit_identical(a, b, f"{case} {env}")
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("mode", ["one_step", "stepwise", "stepwise_one_step"])
@pytest.mark.parametrize("case", ["w_b1", "pw_b4", "decay_range_et"])
def test_emulated_kernel_one_step_and_stepwise_bit_exact(case, mode):
    a, b = _emu_vs_oracle(case, ENVS["sms3"], one_step="one_step" in mode, stepwise="stepwise" in mode)
    helpers.assert_bit_identical(a, b, f"{case} {mode}")


# ---- 3. equivalence with the dense rules (no oracle) ----------------------------------------------------------------

def _readout_pair(rule, B, T=20, **kw):
    """A small reservoir + readout, once with MCC[Weight] + MCC_learning.<rule>, once with Connection + learning.<rule>."""
    nets = []
    for mcc in (True, False):
        net, x = rn.reservoir_readout(B200, rule, B, T, n_res=120, n_in=60, mcc=mcc, seed=3)
        nets.append(net)
    return nets, x


def _readout_state(net) -> dict:
    c = net.connections[("R", "O")]
    r = c.update_rule if hasattr(c, "update_rule") else rn.rule_of(c)
    out = {"w": c.w.detach().cpu().numpy().copy(), "R/s": net.layers["R"].s.cpu().numpy().copy(),
           "O/s": net.layers["O"].s.cpu().numpy().copy(), "O/v": net.layers["O"].v.cpu().numpy().copy()}
    for name in ("p_plus", "p_minus", "eligibility_trace", "_spre", "_spost"):
        v = getattr(r, name, None)
        if isinstance(v, torch.Tensor):
            out[name] = v.detach().cpu().numpy().reshape(-1).copy()
    return out


@pytest.mark.parametrize("rule,B,one_step", [("MSTDP", 1, False), ("MSTDP", 5, False), ("MSTDP", 5, True), ("MSTDPET", 1, False)])
def test_mcc_rule_equals_dense_rule(rule, B, one_step):
    import emu

    (a, b), x = _readout_pair(rule, B)
    outs = []
    for net in (a, b):
        with emu.EmuBackend() as be:
            for k in range(2):
                net.run(inputs={"X": x}, time=x.shape[0], one_spike_seed=7 + k, one_step=one_step, **rn.WINDOW_KWARGS[k])
        assert be.err == 0
        outs.append(_readout_state(net))
    helpers.assert_bit_identical(outs[0], outs[1], f"MCC {rule} vs dense {rule}")
    w0 = rn.reservoir_readout(B200, rule, B, 1, n_res=120, n_in=60, seed=3)[0].connections[("R", "O")].w
    assert not np.array_equal(outs[0]["w"], w0.numpy()), "the readout did not learn"


def test_learning_off_and_manual_update_leave_the_weight_alone():
    import emu
    from bindsnet_b200.network.topology import MulticompartmentConnection

    for how in ("learning", "manual_update"):
        net, inputs, T = rn.live_net(B200, "w_b4")
        c = net.connections[("X", "Y")]
        if how == "learning":
            net.learning = False
        else:
            c.manual_update = True
        w0 = c.w.clone()
        kwargs = rn.WINDOW_KWARGS[0] if how == "learning" else {}   # manual_update: the rule never runs, no reward needed
        with emu.EmuBackend() as be:
            net.run(inputs=rn.window_inputs(inputs, T, 0), time=T, **kwargs)
        assert be.err == 0 and net.monitors["Ys"].get("s").sum() > 0
        assert torch.equal(c.w, w0), how
        assert isinstance(c, MulticompartmentConnection)


def test_scripted_tier_next_to_a_user_defined_population():
    """Like learning.MSTDP on a Connection: with learning off the network runs on the scripted tier and equals the window;
    with learning on the rule's standalone update is refused, as it is for the dense form."""
    import emu
    from test_scripted_tier import MyLIF

    def build(user, mcc=True):
        F, ML = rn.features(B200)
        g = torch.Generator().manual_seed(9)
        net = B200.Network(dt=1.0, batch_size=2, learning=False)
        X = B200.nodes.Input(30, traces=True)
        Y = (MyLIF if user else B200.nodes.LIFNodes)(20, thresh=-60.0, traces=True)
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        w = torch.rand(30, 20, generator=g)
        if mcc:
            conn = B200.topology.MulticompartmentConnection(
                source=X, target=Y, pipeline=[F.Probability("p", torch.rand(30, 20, generator=g)),
                                              F.Weight("w", w, learning_rule=ML.MSTDP, nu=(1e-2, 1e-2), reduction=torch.sum)])
        else:
            conn = B200.topology.Connection(X, Y, w=w, update_rule=B200.learning.MSTDP, nu=1e-2, wmin=-1.0, wmax=1.0)
        net.add_connection(conn, "X", "Y")
        net.add_monitor(B200.monitors.Monitor(Y, ["s"], time=10), "Ys")
        return net, {"X": (torch.rand(10, 2, 30, generator=g) < 0.3).to(torch.uint8)}

    outs = []
    for user in (True, False):
        net, inputs = build(user)
        assert net._scripted_required() == user
        with emu.EmuBackend():
            net.run(inputs=inputs, time=10, one_spike_seed=3, reward=1.0)
        outs.append(net.monitors["Ys"].get("s").clone())
    assert torch.equal(outs[0], outs[1]) and outs[0].sum() > 0
    for mcc in (True, False):
        net, inputs = build(True, mcc)
        net.learning = True
        with emu.EmuBackend(), pytest.raises(NotImplementedError, match="standalone call is not exposed"):
            net.run(inputs=inputs, time=10, one_spike_seed=3, reward=1.0)


def test_reward_fn_supplies_the_reward():
    """A reward_fn's compute replaces the run's reward (network.py:325-326), for the MCC rule as for the dense one."""
    import emu
    from bindsnet_b200.learning.reward import AbstractReward

    class Const(AbstractReward):
        def compute(self, **kwargs):
            return 0.25

        def update(self, **kwargs):
            pass

    outs = []
    for reward_fn in (Const, None):
        net, inputs, T = rn.live_net(B200, "w_b4")
        net.reward_fn = reward_fn() if reward_fn else None
        with emu.EmuBackend():
            net.run(inputs=rn.window_inputs(inputs, T, 0), time=T, reward=0.25 if reward_fn is None else 9.0)
        outs.append(rn.full_snapshot(net, T))
    helpers.assert_bit_identical(outs[0], outs[1], "reward_fn")


# ---- 4. host API -------------------------------------------------------------------------------------------------

def test_rule_defaults_and_state_shapes():
    F, ML = rn.features(B200)
    X, Y = B200.nodes.Input(6), B200.nodes.LIFNodes(5)
    w = F.Weight("w", torch.rand(6, 5), learning_rule=ML.MSTDP)
    c = B200.topology.MulticompartmentConnection(source=X, target=Y, pipeline=[w])
    r = w.learning_rule
    assert (r.min, r.max) == (-torch.inf, torch.inf)   # the Weight's default range is passed on (topology_features.py:618)
    assert r.nu.tolist() == pytest.approx([0.2, 0.1]) and float(r.tc_plus) == 20.0 and float(r.tc_minus) == 20.0
    assert not hasattr(r, "p_plus")
    r2 = ML.MSTDPET(connection=c, feature_value=w.value)
    assert (r2.min, r2.max) == (-1, 1) and float(r2.tc_e_trace) == 25.0
    assert r2.p_plus.shape == (6,) and r2.p_minus.shape == (5,) and r2.eligibility_trace.shape == (6, 5)
    assert r2.eligibility.shape == (6, 5) and r2.eligibility.abs().sum() == 0


def test_refusals():
    import emu

    F, ML = rn.features(B200)
    X, Y = B200.nodes.Input(6), B200.nodes.LIFNodes(5)

    def conn(rule=ML.MSTDP, **kw):
        return B200.topology.MulticompartmentConnection(
            source=X, target=Y, pipeline=[F.Weight("w", torch.rand(6, 5), learning_rule=rule, nu=(0.1, 0.1))], **kw)

    for rule in (ML.MSTDP, ML.MSTDPET):
        with pytest.raises(NotImplementedError, match="average_update"):
            conn(rule, average_update=3)
        with pytest.raises(NotImplementedError, match="continues_update"):
            conn(rule, continues_update=True)
        c = conn(rule)
        with pytest.raises(NotImplementedError, match="enforce_polarity"):
            rule(connection=c, feature_value=c.w, enforce_polarity=True)
        with pytest.raises(NotImplementedError, match="standalone call"):
            rn.rule_of(c).update(reward=1.0)
        with pytest.raises(NotImplementedError, match="standalone call"):
            c.update(learning=True, reward=1.0)
        c.update(learning=False, reward=1.0)             # topology.py:509-518: the rule is not reached
    with pytest.raises(NotImplementedError, match="enforce_polarity"):
        F.Weight("w", torch.rand(6, 5), learning_rule=ML.MSTDP, enforce_polarity=True)
    with pytest.raises(NotImplementedError, match="sparse"):
        F.Weight("w", torch.rand(6, 5), learning_rule=ML.MSTDP, sparse=True)
    with pytest.raises(NotImplementedError, match="Connection type"):
        ML.MSTDP(connection=B200.topology.Connection(X, Y), feature_value=torch.rand(6, 5))

    def run(rule, B=1, **kwargs):
        net = B200.Network(batch_size=B)
        x, y = B200.nodes.Input(6), B200.nodes.LIFNodes(5)
        net.add_layer(x, "X"); net.add_layer(y, "Y")
        net.add_connection(B200.topology.MulticompartmentConnection(
            source=x, target=y, pipeline=[F.Weight("w", torch.rand(6, 5), learning_rule=rule, nu=(0.1, 0.1),
                                                   reduction=torch.sum)]), "X", "Y")
        with emu.EmuBackend():
            net.run({"X": torch.zeros(3, B, 6, dtype=torch.uint8)}, time=3, **kwargs)

    for rule in (ML.MSTDP, ML.MSTDPET):
        with pytest.raises(KeyError, match="reward"):
            run(rule)
        for key, bad in (("reward", torch.ones(2)), ("a_plus", torch.ones(5)), ("a_minus", torch.ones(3)), ("reward", {"r": 1.0})):
            with pytest.raises(NotImplementedError, match=f"{key}=...\\) must be a scalar"):
                run(rule, **{"reward": 1.0, key: bad})
        run(rule, reward=torch.tensor(0.5), a_plus=torch.tensor([0.3]))
    with pytest.raises(NotImplementedError, match="batch size 1 only"):
        run(ML.MSTDPET, B=2, reward=1.0)
    run(ML.MSTDP, B=2, reward=1.0)


def test_kernel_plan_checks():
    """SNN_RULE_MSTDP / MSTDPET on SNN_CONN_MCC need the pointers they need on SNN_CONN_DENSE; MSTDPET needs B = 1."""
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    for case in ("w_b4", "wm_et"):
        net, inputs, T = rn.live_net(B200, case)
        net._rule_kwargs = dict(reward=1.0)
        B = net.batch_size

        def check(plan, B=B):
            opts = _abi.SnnRunOpts()
            opts.T, opts.B, opts.tier = 4, B, 1
            return int(emu.lib().snn_b200_select_tier(C.byref(plan), C.byref(opts)))

        plan, keep = _plan.build_net(net, B, {}, {}, {}, {}, {})
        assert plan.conns[0].kind == _abi.SNN_CONN_MCC and _abi.SNN_RULE_MSTDP <= plan.conns[0].rule <= _abi.SNN_RULE_MSTDPET
        assert check(plan) == 1
        if case == "wm_et":
            assert check(plan, B=2) == 0
        for field in ("p_plus", "p_minus", "mst_spre", "mst_spost") + (("e_trace",) if case == "wm_et" else ()):
            plan, keep = _plan.build_net(net, B, {}, {}, {}, {}, {})
            setattr(plan.conns[0], field, None)
            assert check(plan) == 0, field


def test_fused_tiers_are_never_selected():
    """DiehlAndCook2015 with MCC_learning.MSTDP on its input Weight runs on the generic kernel; a forced fused tier is
    refused."""
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    F, ML = rn.features(B200)
    net = B200.models.DiehlAndCook2015(n_inpt=64, n_neurons=16, batch_size=4)
    for l in net.layers.values():
        l.set_batch_size(4)
    net._rule_kwargs = dict(reward=1.0)

    def tier(force):
        plan, keep = _plan.build_net(net, 4, {}, {}, {}, {}, {})
        opts = _abi.SnnRunOpts()
        opts.T, opts.B, opts.tier = 5, 4, force
        return int(emu.lib().snn_b200_select_tier(C.byref(plan), C.byref(opts)))

    assert tier(0) in (2, 3)
    conn = net.connections[("X", "Ae")]
    w = conn._weight()
    w.learning_rule = ML.MSTDP(connection=conn, feature_value=w.value, range=[0.0, 1.0], nu=(1e-2, 1e-2), reduction=torch.sum)
    assert tier(0) == 1 and tier(1) == 1 and tier(2) == 0 and tier(3) == 0
    x = (torch.rand(5, 4, 64, generator=torch.Generator().manual_seed(1)) < 0.2).to(torch.uint8)
    net.force_tier = 2
    with emu.EmuBackend(), pytest.raises(RuntimeError, match="not implemented"):
        net.run(inputs={"X": x}, time=5, reward=1.0)
    net.force_tier = 0
    w0 = w.value.clone()
    with emu.EmuBackend() as be:
        net.run(inputs={"X": x}, time=5, reward=1.0)
    assert be.err == 0 and emu.last_tier == 1 and not torch.equal(w.value, w0)
