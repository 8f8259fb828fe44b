"""Weight(norm_frequency='time step') and per-target norm tensors (reference: topology_features.py:250-266, :583-671;
topology.py:383-392), run on the generic window kernel.  CPU tests: the oracle (tests/weight_norm_oracle.c) against the
live reference's stored results, the emulated kernel against the oracle bit for bit (window, one-step, stepwise and
scripted tiers), the standalone normalisation against a torch restatement of the reference's arithmetic, the
equivalences with the per-sample and scalar forms, refusals, tier selection, and the reference's own network through
reference_binding.  The stored reference results are regenerated with ``python tests/golden/gen_live.py test_weight_norm``."""
import os
import sys

import numpy as np
import pytest
import torch

import cases
import helpers
import weight_norm_nets as wn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

def _as_tensors(snap: dict) -> dict:
    return {k: torch.from_numpy(v) for k, v in snap.items()}


@reference_side(wn.LIVE_CASES)
def _live(ns, case):
    net, inputs, T, kw = wn.build(ns, case)
    wn.run_windows(net, inputs, T, kw, reference=True)
    return _as_tensors(wn.full_snapshot(net, T))


@reference_side(["ts_pp1", "tt_noop1"])
def _live_one_step(ns, case):
    net, inputs, T, kw = wn.build(ns, case)
    wn.run_windows(net, inputs, T, kw, reference=True, one_step=True)
    return _as_tensors(wn.full_snapshot(net, T))


def _check_live(ref: dict, ours: dict, what: str) -> None:
    assert ref.keys() == ours.keys(), what
    for k in ref:
        if k.endswith("/s") or k.startswith("M/"):
            assert torch.equal(ours[k], ref[k]), f"{what}: {k} differs"
        else:
            torch.testing.assert_close(ours[k], ref[k], rtol=1e-4, atol=1e-4, msg=f"{what}: {k}")


@pytest.mark.parametrize("case", wn.LIVE_CASES)
def test_oracle_matches_live_reference(case):
    from weight_norm_oracle import WeightNormOracleBackend

    net, inputs, T, kw = wn.build(B200, case)
    w0 = wn.weight_of(net.connections[("X", "Y")]).clone()
    with WeightNormOracleBackend() as ob:
        wn.run_windows(net, inputs, T, kw)
    assert ob.err == 0
    ours = _as_tensors(wn.full_snapshot(net, T))
    _check_live(load(_live, case), ours, case)
    assert ours["M/Ys"].sum() > 0
    assert not torch.equal(ours["W/XY"], w0)


@pytest.mark.parametrize("case", ["ts_pp1", "tt_noop1"])
def test_oracle_matches_live_reference_one_step(case):
    from weight_norm_oracle import WeightNormOracleBackend

    net, inputs, T, kw = wn.build(B200, case)
    with WeightNormOracleBackend() as ob:
        wn.run_windows(net, inputs, T, kw, one_step=True)
    assert ob.err == 0
    _check_live(load(_live_one_step, case), _as_tensors(wn.full_snapshot(net, T)), case)


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

def _emu_vs_oracle(case, env, one_step=False, stepwise=False, reset=True, **kw):
    import emu
    from weight_norm_oracle import WeightNormOracleBackend

    outs = []
    for backend in (emu.EmuBackend, WeightNormOracleBackend):
        net, inputs, T, run_kw = wn.build(B200, case, **kw)
        net.force_tier = 1
        if stepwise:   # a monitor on a state the kernel does not record: one-step windows
            net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["s", "refrac_count"], time=T), "Yr")
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env if backend is emu.EmuBackend else {})
        try:
            with backend() as be:
                wn.run_windows(net, inputs, T, run_kw, one_step=one_step, reset=reset)
                assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend and not stepwise and not kw.get("custom"):
            assert emu.last_tier == 1
        outs.append(wn.full_snapshot(net, T))
    return outs


@pytest.mark.parametrize("case", wn.CASES)
def test_emulated_kernel_bit_exact(case):
    a, b = _emu_vs_oracle(case, ENVS["sms3"])
    helpers.assert_bit_identical(a, b, case)
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("env", ["sms1", "sms7", "shuffle"])
@pytest.mark.parametrize("case", ["tt_pp4", "pw", "neg"])
def test_emulated_kernel_grids_bit_exact(case, env):
    a, b = _emu_vs_oracle(case, ENVS[env])
    helpers.assert_bit_identical(a, b, f"{case} {env}")


@pytest.mark.parametrize("mode", ["one_step", "stepwise"])
@pytest.mark.parametrize("case", ["ts_pp1", "tt_noop1", "off"])
def test_emulated_kernel_one_step_and_stepwise_bit_exact(case, mode):
    a, b = _emu_vs_oracle(case, ENVS["sms3"], one_step=mode == "one_step", stepwise=mode == "stepwise")
    helpers.assert_bit_identical(a, b, f"{case} {mode}")


@pytest.mark.parametrize("case", ["off", "ts_pp1", "tt_pp4", "pw"])
def test_scripted_tier_bit_exact(case):
    """A user-defined target population sends the network to the scripted tier, whose gather calls each connection's
    single-operator compute: a 'time step' Weight is normalised there too, every step."""
    a, b = _emu_vs_oracle(case, ENVS["sms3"], custom=True)
    helpers.assert_bit_identical(a, b, f"{case} scripted")
    if case == "off":   # learning off: every column sums to its norm
        net, _, _, _ = wn.build(B200, case)
        norm = [f for f in net.connections[("X", "Y")].pipeline if type(f).__name__ == "Weight"][0].norm
        np.testing.assert_allclose(a["W/XY"].sum(0), norm.numpy(), rtol=1e-5, atol=1e-5)


def test_emulated_kernel_large_batch_odd_shapes_bit_exact():
    """B = 520, T = 5, n_src = 45 (not a multiple of 16) and n_tgt = 37 (not a multiple of 32), two windows without a
    reset between them."""
    a, b = _emu_vs_oracle("t5", ENVS["sms3"], B=520, n_in=45, n=37, reset=False)
    helpers.assert_bit_identical(a, b, "B=520")
    assert a["M/Ys"].sum() > 0


def test_learning_off_still_normalises_every_step():
    """A 'time step' Weight changes in a window with learning off: every column sums to its norm afterwards."""
    from weight_norm_oracle import WeightNormOracleBackend

    net, inputs, T, kw = wn.build(B200, "off")
    norm = [f for f in net.connections[("X", "Y")].pipeline if type(f).__name__ == "Weight"][0].norm
    w0 = wn.weight_of(net.connections[("X", "Y")]).clone()
    with WeightNormOracleBackend():
        net.run(inputs={"X": inputs["X"][:T]}, time=T)
    w = wn.weight_of(net.connections[("X", "Y")])
    assert not torch.equal(w, w0)
    torch.testing.assert_close(w.sum(0), norm, rtol=1e-5, atol=1e-5)


def _chunk_sum(rows: torch.Tensor) -> torch.Tensor:
    """The rows summed one by one in ascending order from +0."""
    part = torch.zeros(rows.shape[1])
    for r in rows:
        part = part + r
    return part


def _restated(w: torch.Tensor, norm, chunks: int = 16) -> torch.Tensor:
    """The reference's per-step normalize (topology_features.py:264-266) with the column sum in the SNN_NORM_CHUNKS
    order: float / Tensor is reciprocal() * norm, Tensor / Tensor a true division."""
    ns = w.shape[0]
    c = (ns + chunks - 1) // chunks
    tot = torch.zeros(w.shape[1])
    for k in range(chunks):
        part = torch.zeros(w.shape[1])
        for i in range(k * c, min((k + 1) * c, ns)):
            part = part + w[i]
        tot = tot + part
    tot[tot == 0] = 1.0
    f = norm / tot if isinstance(norm, torch.Tensor) else tot.reciprocal() * norm
    return w * f


@pytest.mark.parametrize("form", ["scalar", "tensor"])
def test_standalone_compute_equals_torch_restatement(form):
    """MulticompartmentConnection.compute() of a 'time step' Weight normalises after the product, in the order and
    rounding of the reference's form of the norm."""
    import emu

    F, _ = __import__("mcc_feature_nets").features(B200)
    g = torch.Generator().manual_seed(5)
    X, Y = B200.nodes.Input(50), B200.nodes.LIFNodes(40)
    w = torch.randn(50, 40, generator=g)
    w[:, 7] = 0.0
    norm = 3.0 + torch.rand(40, generator=g) if form == "tensor" else 2.75
    c = B200.topology.MulticompartmentConnection(source=X, target=Y, device="cpu",
                                                 pipeline=[F.Weight(name="w", value=w, norm=norm, norm_frequency="time step",
                                                                    range=[-10.0, 10.0])])
    s = (torch.rand(3, 50, generator=g) < 0.4).to(torch.uint8)
    with emu.EmuBackend():
        out = c.compute(s)
    assert torch.equal(out, s.float() @ w)
    assert torch.equal(c.w, _restated(w, norm))
    if form == "scalar":   # (a Python number over a tensor is already the reciprocal form; the true division differs
                           # on some column, so the equality above pins the reciprocal form)
        ns, chunks = w.shape[0], 16
        cs = (ns + chunks - 1) // chunks
        tot = torch.zeros(w.shape[1])
        for k in range(chunks):
            tot = tot + _chunk_sum(w[k * cs:(k + 1) * cs])
        nz = tot != 0
        assert not torch.equal((w * (torch.full_like(tot, norm) / tot))[:, nz], c.w[:, nz])


def test_time_step_t1_learning_off_equals_sample():
    """A 'time step' Weight with a [n_tgt] norm, learning off, T = 1, equals the same network with a 'sample' Weight:
    one division by the same sums."""
    import emu

    outs = []
    for freq in ("time step", "sample"):
        F, _ = __import__("mcc_feature_nets").features(B200)
        g = torch.Generator().manual_seed(11)
        X, Y = B200.nodes.Input(30, traces=True), B200.nodes.LIFNodes(20, traces=True)
        net = B200.Network(dt=1.0, batch_size=2, learning=False)
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        norm = 2.0 + torch.rand(20, generator=g)
        net.add_connection(B200.topology.MulticompartmentConnection(
            source=X, target=Y, device="cpu",
            pipeline=[F.Weight(name="w", value=torch.rand(30, 20, generator=g), norm=norm, norm_frequency=freq)]), "X", "Y")
        net.force_tier = 1
        with emu.EmuBackend():
            net.run(inputs={"X": (torch.rand(1, 2, 30, generator=g) < 0.5).to(torch.uint8)}, time=1)
        outs.append(wn.weight_of(net.connections[("X", "Y")]).clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("kind", ["sample", "connection"])
def test_constant_norm_tensor_equals_scalar(kind):
    """A [n_tgt] norm holding one value on a 'sample' Weight or a Connection equals the scalar norm, bit for bit."""
    import emu

    outs = []
    for tensor in (True, False):
        net, inputs, T, kw = wn.build(B200, "sample_t" if kind == "sample" else "conn_t")
        c = net.connections[("X", "Y")]
        owner = c if kind == "connection" else [f for f in c.pipeline if type(f).__name__ == "Weight"][0]
        owner.norm = torch.full((30,), 7.5) if tensor else 7.5
        net.force_tier = 1
        with emu.EmuBackend():
            wn.run_windows(net, inputs, T, kw)
        outs.append(wn.full_snapshot(net, T))
    helpers.assert_bit_identical(outs[0], outs[1], kind)


def test_refusals():
    F, ML = __import__("mcc_feature_nets").features(B200)
    X, Y = B200.nodes.Input(10, traces=True), B200.nodes.LIFNodes(6, traces=True)
    with pytest.raises(NotImplementedError):
        F.Weight(name="w", value=torch.rand(10, 6), norm=1.0, norm_frequency="every step")
    # the reference's prime_feature assertion on the norm's first dimension
    with pytest.raises(AssertionError):
        B200.topology.MulticompartmentConnection(source=X, target=Y, device="cpu",
                                                 pipeline=[F.Weight(name="w", value=torch.rand(10, 6), norm=torch.ones(5))])

    def run_mcc(norm, **kw):
        net = B200.Network(dt=1.0, batch_size=1)
        a, b = B200.nodes.Input(10, traces=True), B200.nodes.LIFNodes(6, traces=True)
        net.add_layer(a, "X"); net.add_layer(b, "Y")
        net.add_connection(B200.topology.MulticompartmentConnection(
            source=a, target=b, device="cpu", pipeline=[F.Weight(name="w", value=torch.rand(10, 6), norm=norm, **kw)]), "X", "Y")
        net.run(inputs={"X": torch.zeros(2, 1, 10, dtype=torch.uint8)}, time=2)

    import emu
    with emu.EmuBackend():
        with pytest.raises(NotImplementedError):   # per-element: [n_src, n_tgt] passes the assertion
            run_mcc(torch.ones(6, 6))
        with pytest.raises(NotImplementedError):
            run_mcc(torch.ones(6, dtype=torch.float64))

        def run_conn(norm):
            net = B200.Network(dt=1.0, batch_size=1)
            a, b = B200.nodes.Input(10), B200.nodes.LIFNodes(6)
            net.add_layer(a, "X"); net.add_layer(b, "Y")
            net.add_connection(B200.topology.Connection(source=a, target=b, norm=norm), "X", "Y")
            net.run(inputs={"X": torch.zeros(2, 1, 10, dtype=torch.uint8)}, time=2)

        for bad in (torch.ones(10, 1), torch.ones(10, 6), torch.ones(6, dtype=torch.float16)):
            with pytest.raises(NotImplementedError):
                run_conn(bad)
        for good in (torch.tensor(2.0), torch.ones(1), torch.ones(6), torch.ones(1, 6)):
            run_conn(good)
        with pytest.raises(NotImplementedError):   # a 'time step' Weight with averaged updates
            net = B200.Network(dt=1.0, batch_size=1)
            a, b = B200.nodes.Input(10, traces=True), B200.nodes.LIFNodes(6, traces=True)
            net.add_layer(a, "X"); net.add_layer(b, "Y")
            net.add_connection(B200.topology.MulticompartmentConnection(
                source=a, target=b, device="cpu", average_update=3,
                pipeline=[F.Weight(name="w", value=torch.rand(10, 6), norm=1.0, norm_frequency="time step",
                                   learning_rule=ML.PostPre, nu=(1e-2, 1e-2))]), "X", "Y")
            net.run(inputs={"X": torch.zeros(2, 1, 10, dtype=torch.uint8)}, time=2)


@pytest.mark.parametrize("case", ["ts_pp1", "conn_t"])
def test_sharded_runner_refuses(case):
    from bindsnet_b200 import distributed

    net, _, _, _ = wn.build(B200, case)
    with pytest.raises(NotImplementedError):
        distributed.ShardedWindowRunner(net)._learned()


def test_tier_selection_and_forced_fused_tiers():
    """Tier 0 picks the generic kernel for a DiehlAndCook2015 graph with either feature; a forced fused tier is
    SNN_ERR_UNSUPPORTED; an unflagged plan keeps its tier."""
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    lib = emu.lib()
    for freq in ("time step", "sample"):
        net, x = wn.dc_graph(B200, 4, freq, n_in=64, n=40, T=10)
        d, _keep = _plan.build_net(net, 4, {"X": x}, {}, {}, {}, {})
        o = _abi.SnnRunOpts()
        o.T, o.B, o.normalize = 10, 4, 1
        flagged = bool(d.conns[0].kind & _abi.SNN_CONN_WNORM)
        assert flagged == (freq == "time step")
        for tier, want in ((0, 1), (1, 1), (2, 0), (3, 0)):
            o.tier = tier
            got = lib.snn_b200_select_tier(d, o)
            if flagged:
                assert got == want, (tier, got)
        o.tier = 0
        if not flagged:
            assert lib.snn_b200_select_tier(d, o) in (1, 2, 3)


@pytest.mark.parametrize("case", ["ts_noop1", "ts_pp1", "tt_pp4", "off", "neg", "sample_t", "conn_t"])
def test_reference_binding_matches_reference_run(case):
    """The reference's own network, described through the ABI by reference_binding (which reads norm_frequency and norm
    tensors) and run by the oracle library, equals the reference's Network.run over three windows.  Skipped where the
    reference is not present."""
    try:
        ref = cases.namespace("reference")
    except Exception as e:  # pragma: no cover
        pytest.skip(f"the reference is missing: {e}")
    import weight_norm_oracle
    from bindsnet_b200 import reference_binding as rb

    snaps = []
    for binding in (False, True):
        net, inputs, T, kw = wn.build(ref, case)
        if not binding:
            wn.run_windows(net, inputs, T, kw, reference=True)
        else:
            learning = net.learning
            for k in range(3):
                net.learning = learning and k != 1
                x = {name: v[k * T:(k + 1) * T] for name, v in inputs.items()}
                assert rb.run_window(net, x, time=T, seed=wn.SEED + k, library=weight_norm_oracle.lib()) == 0
                if k == 0:
                    net.reset_state_variables()
        snaps.append({k: v for k, v in _as_tensors(wn.full_snapshot(net, T)).items() if not k.startswith("M/")})
    _check_live(snaps[0], snaps[1], case)   # (reference_binding records no monitors)
