"""Per-synapse wmin / wmax and learning-rate tensors of a dense Connection (reference: topology.py:74-81, 308-317;
learning.py:58-67, 97-104), run on the generic window kernel.  CPU tests: the oracle against the live reference's stored
results, the emulated kernel against the oracle bit for bit, equivalences (constant tensors = scalars, broadcast =
materialised), refusals and tier selection.  "The oracle" here is tests/synapse_oracle.c.  The stored reference results
are regenerated with ``python tests/golden/gen_live.py test_synapse_tensors``."""
import os
import sys

import numpy as np
import pytest
import torch

import cases
import helpers
import synapse_nets as sn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

@reference_side(sn.LIVE_CASES)
def _live(ns, case):
    net, inputs, T, masks = sn.live_net(ns, case)
    return sn.run_two_windows(net, inputs, T, case, masks=masks, reference=True)


@pytest.mark.parametrize("case", sn.LIVE_CASES)
def test_oracle_matches_live_reference(case):
    from synapse_oracle import SynapseOracleBackend

    ref = load(_live, case)
    net, inputs, T, masks = sn.live_net(B200, case)
    w0 = {k: c.w.detach().clone() for k, c in net.connections.items()}
    with SynapseOracleBackend() as ob:
        ours = sn.run_two_windows(net, inputs, T, case, masks=masks)
    assert ob.err == 0
    learned = ("Y", "Y") if case == "ei" else ("X", "Y")
    for k in ("0", "1"):
        assert torch.equal(ours[f"{k}/Ys"], ref[f"{k}/Ys"]), f"window {k}: spike rasters differ"
        assert ours[f"{k}/Ys"].sum() > 0
        for name in ["Y/v", "Y/x", "XY/w", "YY/w"]:
            torch.testing.assert_close(ours[f"{k}/{name}"], ref[f"{k}/{name}"], rtol=1e-4, atol=1e-5, msg=f"window {k} {name}")
    assert not torch.equal(ours[f"1/{''.join(learned)}/w"], w0[learned]), "the weights did not learn"


def test_bounds_hold_and_clamp_the_user_weights():
    """Case "ei": every recurrent weight ends inside its row's sign bounds, though the user's w started outside them."""
    from synapse_oracle import SynapseOracleBackend

    net, inputs, T, masks = sn.live_net(B200, "ei")
    yy = net.connections[("Y", "Y")]
    assert bool(((yy.w < yy.wmin) | (yy.w > yy.wmax)).any())
    with SynapseOracleBackend():
        sn.run_two_windows(net, inputs, T, "ei")
    assert bool(((yy.w >= yy.wmin) & (yy.w <= yy.wmax)).all())


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _emu_vs_oracle(case, env, T=12, one_step=False, stepwise=False):
    import emu
    from synapse_oracle import SynapseOracleBackend

    outs = []
    for backend in (emu.EmuBackend, SynapseOracleBackend):
        net, inputs, T, masks = sn.live_net(B200, case, T=T)
        net.force_tier = 0
        if stepwise:   # a monitor on a state the kernel does not record: one-step windows
            net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["s", "refrac_count"], time=T), "Yr")
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env if backend is emu.EmuBackend else {})
        try:
            with backend() as be:
                sn.run_two_windows(net, inputs, T, case, masks=masks, one_step=one_step)
                assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
        outs.append(sn.snapshot(net))
    return outs


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["pp_full", "wdep_full", "hebb_full", "mstdp_b4", "mstdpet", "ei"])
def test_emulated_kernel_bit_exact(case, env):
    a, b = _emu_vs_oracle(case, ENVS[env])
    helpers.assert_bit_identical(a, b, f"{case} {env}")
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("mode", ["one_step", "stepwise"])
@pytest.mark.parametrize("case", ["pp_tgt_mean", "wdep_src", "hebb_tgt", "mstdp_b1"])
def test_emulated_kernel_one_step_and_stepwise_bit_exact(case, mode):
    a, b = _emu_vs_oracle(case, ENVS["sms3"], T=7, one_step=mode == "one_step", stepwise=mode == "stepwise")
    helpers.assert_bit_identical(a, b, f"{case} {mode}")


def test_emulated_kernel_large_batch_odd_T():
    """B = 520 (more than 512 samples: several groups of the staging and event slots), odd T, two windows."""
    import emu
    from synapse_oracle import SynapseOracleBackend

    outs = []
    for backend in (emu.EmuBackend, SynapseOracleBackend):
        net, x = sn.ei_network(B200, 96, 520, 7, n_in=64, seed=5)
        with backend() as be:
            for k in range(2):
                net.run(inputs={"X": x}, time=7)
            assert be.err == 0
        outs.append(sn.snapshot(net))
    helpers.assert_bit_identical(outs[0], outs[1], "B = 520, T = 7")


def test_scripted_tier_with_a_user_defined_layer_and_rule():
    """The scripted tier (a user-defined population and a user-defined rule in the network): the built-in rule's
    single-operator update reads the tensors, the user rule's base update clamps with them."""
    import emu
    from synapse_oracle import SynapseOracleBackend
    from test_scripted_tier import MyLIF

    class Shrink(B200.learning.LearningRule):
        def update(self, **kwargs):
            self.connection.w *= 0.9
            self.connection.w += 0.05
            super().update()

    def build():
        g = torch.Generator().manual_seed(11)
        net = B200.Network(dt=1.0, batch_size=2, learning=True)
        X = B200.nodes.Input(20, traces=True)
        Y = B200.nodes.LIFNodes(16, traces=True, thresh=-60.0)
        U = MyLIF(12)
        net.add_layer(X, "X"); net.add_layer(Y, "Y"); net.add_layer(U, "U")
        lo, hi = sn.bounds("full", 20, 16, g, inf=False)
        nu = (1e-2 * torch.rand(20, 16, generator=g), 1e-2 * torch.rand(20, 16, generator=g))
        net.add_connection(B200.topology.Connection(X, Y, w=torch.rand(20, 16, generator=g), wmin=lo, wmax=hi, nu=nu,
                                                    update_rule=B200.learning.WeightDependentPostPre, reduction=torch.sum), "X", "Y")
        lo2, hi2 = sn.bounds("tgt", 16, 12, g)
        net.add_connection(B200.topology.Connection(Y, U, w=torch.rand(16, 12, generator=g) * 3, wmin=lo2, wmax=hi2,
                                                    update_rule=Shrink), "Y", "U")
        x = (torch.rand(10, 2, 20, generator=g) < 0.4).to(torch.uint8)
        return net, x

    outs = []
    for backend in (emu.EmuBackend, SynapseOracleBackend):
        net, x = build()
        with backend() as be:
            net.run(inputs={"X": x}, time=10)
            assert be.err == 0
        outs.append(sn.snapshot(net))
    helpers.assert_bit_identical(outs[0], outs[1], "scripted tier")
    yu = outs[0]["C/YU/w"]
    net, _ = build()
    c = net.connections[("Y", "U")]
    assert np.all(yu >= c.wmin.numpy()) and np.all(yu <= c.wmax.numpy())


# ---- 3. equivalences, bit for bit ------------------------------------------------------------------------------------

def _run_emu(net, x, windows=2, **kw):
    import emu

    with emu.EmuBackend() as be:
        for k in range(windows):
            net.run(inputs={"X": x}, time=x.shape[0], **kw)
        assert be.err == 0
    return sn.snapshot(net)


@pytest.mark.parametrize("B", [1, 4])
def test_constant_tensors_equal_scalars(B):
    a = _run_emu(*sn.ei_network(B200, 64, B, 9, n_in=48, seed=2, scalar_twin=True))
    b = _run_emu(*sn.constant_twin(B200, 64, B, 9, n_in=48, seed=2))
    helpers.assert_bit_identical(a, b, "constant tensors vs scalars")


@pytest.mark.parametrize("B", [1, 3])
def test_broadcast_equals_materialised(B):
    a = _run_emu(*sn.ei_network(B200, 64, B, 9, n_in=48, seed=4))
    b = _run_emu(*sn.ei_network(B200, 64, B, 9, n_in=48, seed=4, full_bounds=True))
    helpers.assert_bit_identical(a, b, "per-row bounds vs their [n, n] copy")


@pytest.mark.parametrize("rule", ["PostPre", "WeightDependentPostPre", "Hebbian"])
def test_standalone_update_matches_torch(rule):
    """connection.update() (the single-operator update) against a torch restatement of the reference's update."""
    import emu

    g = torch.Generator().manual_seed(8)
    B, ns_, nt = 3, 24, 20
    X = B200.nodes.Input(ns_, traces=True)
    Y = B200.nodes.LIFNodes(nt, traces=True)
    net = B200.Network(batch_size=B)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    lo, hi = sn.bounds("full", ns_, nt, g, inf=rule != "WeightDependentPostPre")
    nu = sn.rates("tgt" if rule == "PostPre" else "full", rule, ns_, nt, g)
    c = B200.topology.Connection(X, Y, w=torch.rand(ns_, nt, generator=g), wmin=lo, wmax=hi, nu=nu,
                                 update_rule=getattr(B200.learning, rule), reduction=torch.sum)
    net.add_connection(c, "X", "Y")
    X.s = torch.rand(B, ns_, generator=g) < 0.4
    Y.s = torch.rand(B, nt, generator=g) < 0.4
    X.x = torch.rand(B, ns_, generator=g)
    Y.x = torch.rand(B, nt, generator=g)
    w = c.w.detach().clone()
    ss, sx, ts, tx = X.s.float().unsqueeze(2), X.x.unsqueeze(2), Y.s.float().unsqueeze(1), Y.x.unsqueeze(1)
    n0, n1 = c.update_rule.nu[0], c.update_rule.nu[1]
    if rule == "PostPre":
        w = w - torch.bmm(ss, tx * n0).sum(0)
        w = w + torch.bmm(sx, ts * n1).sum(0)
    elif rule == "WeightDependentPostPre":
        upd = 0 - n0 * torch.bmm(ss, tx).sum(0) * (w - lo)
        upd = upd + n1 * torch.bmm(sx, ts).sum(0) * (hi - w)
        w = w + upd
    else:
        w = w + n0 * torch.bmm(ss, tx).sum(0)
        w = w + n1 * torch.bmm(sx, ts).sum(0)
    w = w.clamp(lo, hi)
    with emu.EmuBackend():
        c.update()
    torch.testing.assert_close(c.w.detach(), w, rtol=1e-5, atol=1e-6)


# ---- 4. refusals and tier selection ----------------------------------------------------------------------------------

def test_postpre_with_a_per_synapse_rate_raises_like_the_reference():
    import emu

    net, inputs, T, _ = sn.live_net(B200, "pp_full")
    c = net.connections[("X", "Y")]
    c.update_rule.nu = torch.stack([torch.full((sn.N_IN, sn.N), 1e-2), torch.full((sn.N_IN, sn.N), 1e-2)])
    c.update_rule._nu_tensors = True
    w0 = c.w.detach().clone()
    with emu.EmuBackend():
        with pytest.raises(RuntimeError, match="batch2"):
            net.run(inputs=sn.window_inputs(inputs, T, 0), time=T)
    assert torch.equal(c.w, w0)


def test_weight_dependent_rule_with_an_infinite_bound_element_is_refused():
    g = torch.Generator().manual_seed(1)
    lo, hi = sn.bounds("full", 12, 10, g)
    X, Y = B200.nodes.Input(12, traces=True), B200.nodes.LIFNodes(10, traces=True)
    c = B200.topology.Connection(X, Y, wmin=lo, wmax=hi, update_rule=B200.learning.WeightDependentPostPre, nu=(1e-2, 1e-2))
    from bindsnet_b200.network import _plan

    with pytest.raises(NotImplementedError, match="NaN"):
        _plan._conn_desc(c, 1)


def test_a_rate_on_another_device_raises():
    net, inputs, T, _ = sn.live_net(B200, "wdep_full")
    c = net.connections[("X", "Y")]
    c.update_rule.nu = c.update_rule.nu.to("meta")
    with pytest.raises(RuntimeError, match="same device"):
        from bindsnet_b200.network import _plan

        _plan._conn_desc(c, 2)


def test_out_of_scope_kinds_keep_their_errors():
    T = B200.topology
    X, Y = B200.nodes.Input(16, shape=(1, 4, 4), traces=True), B200.nodes.LIFNodes(8, shape=(2, 2, 2), traces=True)
    lo = -torch.ones(16, 8)
    with pytest.raises(NotImplementedError, match="learning-rate tensors"):
        T.Conv2dConnection(X, Y, kernel_size=3, stride=1, update_rule=B200.learning.PostPre, nu=(torch.ones(2, 1, 3, 3), torch.ones(2, 1, 3, 3)))
    c = T.Conv2dConnection(X, Y, kernel_size=3, stride=1, wmin=-torch.ones(2, 1, 3, 3), wmax=torch.ones(2, 1, 3, 3))
    with pytest.raises(NotImplementedError, match="wmin/wmax tensors"):
        from bindsnet_b200.network import _plan

        _plan._conn_desc(c, 1)
    X2, Y2 = B200.nodes.Input(16, traces=True), B200.nodes.LIFNodes(8, traces=True)
    s = T.SparseConnection(X2, Y2, wmin=lo, wmax=-lo)
    with pytest.raises(NotImplementedError, match="SparseConnection"):
        _plan._conn_desc(s, 1)
    with pytest.raises(NotImplementedError, match="learning-rate tensors"):
        T.SparseConnection(X2, Y2, nu=(torch.ones(16, 8), torch.ones(16, 8)))


def test_distributed_refuses_tensor_bounds():
    from bindsnet_b200.distributed import ShardedWindowRunner

    net, _, _, _ = sn.live_net(B200, "wdep_full")
    with pytest.raises(NotImplementedError, match="per-synapse"):
        ShardedWindowRunner(net)._learned()


def test_dc2015_with_tensor_bounds_runs_on_tier_1_and_refuses_fused_tiers():
    """A DiehlAndCook2015-shaped graph (Connection + PostPre into DiehlAndCookNodes, recurrent inhibition): the fused
    tiers take it with scalar bounds; with tensor bounds tier 0 selects the generic kernel and a forced fused tier is
    refused before anything runs."""
    import emu
    from bindsnet_b200 import _backend

    def model(tensors):
        g = torch.Generator().manual_seed(21)
        n_in, n = 64, 32
        net = B200.Network(dt=1.0, batch_size=2)
        X = B200.nodes.Input(n_in, traces=True)
        E = B200.nodes.DiehlAndCookNodes(n, traces=True)
        I = B200.nodes.LIFNodes(n, traces=False)
        net.add_layer(X, "X"); net.add_layer(E, "Ae"); net.add_layer(I, "Ai")
        lo, hi = (torch.zeros(n_in, n), torch.ones(n)) if tensors else (0.0, 1.0)
        net.add_connection(B200.topology.Connection(X, E, w=0.3 * torch.rand(n_in, n, generator=g), update_rule=B200.learning.PostPre,
                                                    nu=(1e-4, 1e-2), reduction=torch.sum, wmin=lo, wmax=hi, norm=20.0), "X", "Ae")
        net.add_connection(B200.topology.Connection(E, I, w=22.5 * torch.eye(n)), "Ae", "Ai")
        net.add_connection(B200.topology.Connection(I, E, w=-120.0 * (1 - torch.eye(n))), "Ai", "Ae")
        x = (torch.rand(10, 2, n_in, generator=g) < 0.2).to(torch.uint8)
        return net, x

    with emu.EmuBackend():
        net, x = model(False)
        net.run(inputs={"X": x}, time=10)
        assert emu.last_tier in (2, 3)
        net, x = model(True)
        net.run(inputs={"X": x}, time=10)
        assert emu.last_tier == 1
        for tier in (2, 3):
            net, x = model(True)
            w0 = net.connections[("X", "Ae")].w.detach().clone()
            net.force_tier = tier
            with pytest.raises((_backend.BackendError, RuntimeError), match="not implemented"):   # (the emulation's error)
                net.run(inputs={"X": x}, time=10)
            assert torch.equal(net.connections[("X", "Ae")].w, w0)


def test_reference_network_through_reference_binding():
    """The reference's own network with tensor bounds and rates, bound to the ABI by reference_binding and run on the
    oracle, equals the reference's own run of it."""
    from bindsnet_b200 import reference_binding as rb
    from synapse_oracle import lib as oracle_lib

    try:
        ref = cases.namespace("reference")
    except ImportError:
        pytest.skip("the reference copy is not built")
    outs = []
    for bound in (False, True):
        net, inputs, T, _ = sn.live_net(ref, "wdep_full")
        x = sn.window_inputs(inputs, T, 0)
        if bound:
            rb.run_window(net, x, T, library=oracle_lib())
        else:
            net.run(inputs=x, time=T)
        outs.append({f"{s}{t}": c.w.detach().clone() for (s, t), c in net.connections.items()})
        outs[-1]["Y/v"] = net.layers["Y"].v.detach().clone()
    for k in outs[0]:
        torch.testing.assert_close(outs[1][k], outs[0][k], rtol=1e-4, atol=1e-5, msg=k)
