"""Conv3dConnection (reference: topology.py:847-1025) on the generic window kernel.  CPU tests: the oracle
(tests/conv3d_oracle.c, the CPU oracle extended by the 3-D convolution) against the live reference's stored results, the
emulated kernel against the oracle bit for bit, the standalone operators against F.conv3d and a torch restatement,
refusals, tier selection and the multi-GPU combine.  The stored reference results are regenerated with
``python tests/golden/gen_live.py test_conv3d``."""
import ctypes as C
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import cases
import conv3d_nets as cn
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


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

def _stored(flat):
    """What tests/golden/live keeps of the windows' states: everything, except that a weight tensor of more than 4096
    floats (the example's 25 x 16**3 filters, 400 KB of incompressible floats per window) is kept as every 29th weight,
    a prime stride that visits every filter and every tap position.  The emulated-kernel and GPU tests compare the whole
    tensor with the oracle's."""
    out = {}
    for k, v in flat.items():
        if k.endswith("/w") and v.numel() > 4096:
            out[k + "_every_29th"] = v.flatten()[::29].clone()
        else:
            out[k] = v
    return out


@reference_side(CASES)
def _live(ns, case):
    net, inputs, T = cn.build_case(ns, case)
    return _stored(_flat(cn.run_windows(net, inputs, T, cn.windows_of(case))))


def _check_against(ref, ours, what):
    for k, v in ref.items():
        o = ours[k]
        assert o.shape == v.shape, (what, k)
        if k.endswith("s"):
            assert torch.equal(o.float(), v.float()), f"{what}: {k} differs"
        else:
            torch.testing.assert_close(o.float(), v.float(), rtol=1e-5, atol=1e-4, equal_nan=True, msg=f"{what}: {k}")


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_live_reference(case):
    from conv3d_oracle import Conv3dOracleBackend

    net, inputs, T = cn.build_case(B200, case)
    with Conv3dOracleBackend() as ob:
        ours = _flat(cn.run_windows(net, inputs, T, cn.windows_of(case)))
    assert ob.err == 0
    ref = load(_live, case)
    assert ref.keys() == _stored(ours).keys()
    _check_against(ref, _stored(ours), case)
    assert ours["w0/Ys"].sum() > 0
    if cn.LIVE_CASES[case].get("zero_row"):
        assert torch.isnan(ours["w0/XY/w"][1, 0]).all() and not torch.isnan(ours["w0/XY/w"][0]).any()


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _same(a, b):
    return torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num()))


def _emu_vs_oracle(build, env=None, n=2, **kw):
    import emu
    from conv3d_oracle import Conv3dOracleBackend

    outs = []
    for backend in (emu.EmuBackend, Conv3dOracleBackend):
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
@pytest.mark.parametrize("case", ["example_b1_noop", "c2_noop", "c2_zero_rate_postpre"])
def test_emulated_kernel_bit_exact(case, env):
    a = _emu_vs_oracle(lambda: cn.build_case(B200, case, T=8 if case.startswith("example") else 24), ENVS[env])
    assert a["w1/Ys"].sum() > 0


def test_emulated_kernel_zero_row_bit_exact():
    _emu_vs_oracle(lambda: cn.build_case(B200, "c2_zero_row"), ENVS["sms3"], n=1)


def test_emulated_kernel_one_step_bit_exact():
    _emu_vs_oracle(lambda: cn.multi_net(B200, rule="NoOp", weight_decay=1e-2), ENVS["sms3"], one_step=True)


def test_stepwise_equals_oracle():
    """A monitor on the target's voltages and traces makes the window run step by step (one one-step window per step)."""
    def build():
        net, inputs, T = cn.multi_net(B200, rule="PostPre", weight_decay=1e-2, wmin=0.05, wmax=0.45, T=10)
        net.add_monitor(B200.monitors.Monitor(net.layers["Y"], ["x"], time=T), "Yx")
        return net, inputs, T

    _emu_vs_oracle(build, ENVS["sms3"])


@pytest.mark.parametrize("T", [7, 8])
def test_emulated_kernel_large_batch_bit_exact(T):
    """B = 520 and an odd and an even window length."""
    a = _emu_vs_oracle(lambda: cn.multi_net(B200, rule="NoOp", weight_decay=1e-2, B=520, T=T), ENVS["sms3"])
    assert a["w1/Ys"].sum() > 0


def test_two_windows_without_reset():
    _emu_vs_oracle(lambda: cn.multi_net(B200, rule="NoOp", weight_decay=1e-2, T=9), ENVS["sms3"], reset=False)


def test_wide_kernel_and_unstaged_taps():
    """kw = 33 > 32 (two runs of a kernel row), tiles that cross filters, and tiles that cannot stage their taps."""
    net, _, _ = cn.wide_net(B200)
    p = cn.gather_paths(net.connections[("X", "Y")], 3)
    assert p["kw_over_32"] and p["tile_crosses_filter"] and p["st_taps_some_off"] and not p["st_taps_all"] and p["st_bits"]
    a = _emu_vs_oracle(lambda: cn.wide_net(B200), ENVS["sms7"])
    assert a["w1/Ys"].sum() > 0


def test_example_geometry_staged_and_unstaged_bits():
    """The example geometry: a 686-word source sample, so one sample chunk of B = 1 stages its bit rows and one of B = 8
    does not; every tile lies inside one filter whose 16**3 taps (4096 floats) are staged."""
    net, _, _ = cn.example_net(B200)
    conn = net.connections[("X", "Y")]
    p1, p8 = cn.gather_paths(conn, 1), cn.gather_paths(conn, 8)
    assert p1["st_bits"] and not p8["st_bits"] and p1["st_taps_all"] and not p1["tile_crosses_filter"]
    a = _emu_vs_oracle(lambda: cn.example_net(B200, B=8, T=5, learning=False), ENVS["sms3"], n=1)
    assert a["w0/Ys"].sum() > 0


def test_example_one_spike_bit_exact():
    """The example's DiehlAndCookNodes with one_spike (the window's seeded winner draw) and the NoOp decay."""
    a = _emu_vs_oracle(lambda: cn.example_net(B200, T=8, rule="NoOp", weight_decay=1e-3, one_spike=True), ENVS["sms3"],
                       one_spike_seed=7)
    assert a["w1/Ys"].sum() > 0


def test_multi_net_paths():
    net, _, _ = cn.multi_net(B200)
    p = cn.gather_paths(net.connections[("X", "Y")], 4)
    assert p["st_bits"] and p["st_taps_all"] and p["tile_crosses_filter"]


def test_scripted_tier_equals_window():
    import emu
    from conv3d_oracle import Conv3dOracleBackend
    from test_scripted_tier import MyLIF

    def build(user):
        net, inputs, T = cn.multi_net(B200, rule="PostPre", weight_decay=1e-2, wmin=0.05, wmax=0.45, B=3, T=12)
        if user:   # a user-defined population as the last layer: the network runs on the scripted tier
            Z = MyLIF(6, traces=True, thresh=-62.0)
            net.layers["Z"] = Z
            net.add_layer(Z, "Z")
            net.connections[("Y", "Z")].target = Z
            net.monitors["Zs"].obj = Z
        return net, inputs, T

    outs = []
    for user, backend in ((True, emu.EmuBackend), (True, Conv3dOracleBackend), (False, emu.EmuBackend)):
        net, inputs, T = build(user)
        assert net._scripted_required() == user
        with backend():
            net.run(inputs={"X": inputs["X"][0]}, time=T)
        outs.append(cn.state(net))
    for o in outs[1:]:
        for k in outs[0]:
            assert torch.equal(outs[0][k].float(), o[k].float()), k
    assert outs[0]["Ys"].sum() > 0


# ---- 3. the standalone operators -------------------------------------------------------------------------------------

def test_standalone_compute_matches_conv3d_and_oracle():
    import emu
    from conv3d_oracle import Conv3dOracleBackend

    g = torch.Generator().manual_seed(21)
    for build in (cn.multi_net, cn.wide_net):
        net, _, _ = build(B200)
        conn = net.connections[("X", "Y")]
        s = torch.rand(3, *conn.source.shape, generator=g) < 0.4
        with emu.EmuBackend():
            a = conn.compute(s)
        with Conv3dOracleBackend():
            b = conn.compute(s)
        assert torch.equal(a, b)
        ref = F.conv3d(s.float(), conn.w, conn.b, stride=conn.stride, padding=conn.padding)
        torch.testing.assert_close(a, ref, rtol=1e-5, atol=1e-5)


def test_standalone_update_and_normalize_match_torch():
    import emu

    for rule, kw in (("NoOp", dict(weight_decay=0.02)), ("PostPre", dict(weight_decay=0.02, wmin=0.05, wmax=0.3)),
                     ("WeightDependentPostPre", dict(weight_decay=0.0, wmin=0.1, wmax=0.2))):
        net, _, _ = cn.multi_net(B200, rule=rule, B=2, **kw)
        conn = net.connections[("X", "Y")]
        for L in net.layers.values():
            L.set_batch_size(2)
            L.compute_decays(1.0)
        with emu.EmuBackend():
            for _ in range(2):
                ref = conn.w.clone()
                if kw["weight_decay"]:
                    ref = ref * (1.0 - kw["weight_decay"])
                if rule != "NoOp":
                    ref = ref.clamp(kw["wmin"], kw["wmax"])
                conn.update_rule.update()
                assert torch.equal(conn.w, ref), rule
            with torch.no_grad():
                conn.w[2, 1, 0, 0, 0] = 0.0
            ref = conn.w.clone().view(6, -1)
            ref = ref * (conn.norm / ref.sum(1, keepdim=True))
            conn.normalize()
        torch.testing.assert_close(conn.w.view(6, -1), ref, rtol=1e-6, atol=1e-6)


# ---- 4. refusals and errors ------------------------------------------------------------------------------------------

def _small(ns, B=2, rule="NoOp", learning=True, tgt=(2, 2, 2, 2), **kw):
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=[1, 5, 5, 5], traces=True)
    Y = ns.nodes.LIFNodes(shape=list(tgt), traces=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    net.add_connection(ns.topology.Conv3dConnection(X, Y, kernel_size=3, stride=2, update_rule=getattr(ns.learning, rule), **kw), "X", "Y")
    return net, {"X": (torch.rand(4, B, 1, 5, 5, 5, generator=torch.Generator().manual_seed(1)) < 0.3).to(torch.uint8)}


def _unchanged_after(exc, net, inputs, match=None, **run_kw):
    import emu

    before = {k: v.clone() for k, v in cn.state(net).items()}
    with emu.EmuBackend(), pytest.raises(exc, match=match):
        net.run(inputs=inputs, time=4, **run_kw)
    after = cn.state(net)
    for k in before:
        assert _same(before[k], after[k]), k


@pytest.mark.parametrize("rule,nu", [("PostPre", (1e-4, 1e-2)), ("WeightDependentPostPre", (1e-3, 0.0)), ("Hebbian", (1e-3, 1e-3)),
                                     ("MSTDP", (1e-3, 1e-3)), ("MSTDPET", (1e-3, 1e-3))])
def test_rules_with_a_presynaptic_term_raise_like_the_reference(rule, nu):
    """The rule constructs; a learning window raises the reference's RuntimeError before anything runs; learning=False
    runs."""
    kw = dict(nu=list(nu), wmin=0.0, wmax=1.0)
    ref = _reference()
    if ref is not None:
        net, inputs = _small(ref, rule=rule, **kw)
        with pytest.raises(RuntimeError):   # (MSTDPET fails one line earlier, in a view of the unfolded traces)
            net.run(inputs=inputs, time=4, reward=1.0)
    net, inputs = _small(B200, rule=rule, **kw)
    _unchanged_after(RuntimeError, net, inputs, match="same dtype", reward=1.0)
    if rule in ("PostPre", "WeightDependentPostPre", "Hebbian"):
        with pytest.raises(RuntimeError, match="same dtype"):
            net.connections[("X", "Y")].update_rule.update()
    import emu

    net.learning = False
    with emu.EmuBackend():
        net.run(inputs=inputs, time=4)
    assert emu.last_tier == 1


def test_example_network_with_postpre_raises_before_any_step():
    net, inputs, T = cn.example_net(B200, T=4)
    _unchanged_after(RuntimeError, net, {"X": inputs["X"][0]}, match="same dtype")


@pytest.mark.parametrize("rule", ["PostPre", "WeightDependentPostPre"])
def test_post_only_rule_refused_at_construction(rule):
    with pytest.raises(NotImplementedError, match="post-synaptic"):
        _small(B200, rule=rule, nu=[0.0, 1e-2], wmin=0.0, wmax=1.0)


def test_dilation_refused():
    ref = _reference()
    for ns in (ref, B200):
        if ns is None:
            continue
        with pytest.raises(NotImplementedError):
            _small(ns, dilation=2)


def test_wrong_target_shape_raises_assertion_error():
    ref = _reference()
    for ns in (ref, B200):
        if ns is None:
            continue
        with pytest.raises(AssertionError):
            _small(ns, tgt=(2, 2, 2, 3))


def test_non_float32_weights_refused():
    with pytest.raises(NotImplementedError):
        _small(B200, w_dtype=torch.float16)


def test_empty_output_raises_runtime_error():
    def build(ns):
        net = ns.Network(dt=1.0, batch_size=1, learning=False)
        X, Y = ns.nodes.Input(shape=[1, 4, 4, 4]), ns.nodes.LIFNodes(shape=[2, 0, 0, 0])
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        net.add_connection(ns.topology.Conv3dConnection(X, Y, kernel_size=5), "X", "Y")
        return net, {"X": torch.zeros(4, 1, 1, 4, 4, 4, dtype=torch.uint8)}

    ref = _reference()
    if ref is not None:
        with pytest.raises(RuntimeError):
            net, inputs = build(ref)
            net.run(inputs=inputs, time=4)
    net, inputs = build(B200)
    _unchanged_after(RuntimeError, net, inputs)


def test_masks_refused():
    net, inputs = _small(B200, learning=False)
    _unchanged_after(NotImplementedError, net, inputs, match="dense Connection only",
                     masks={("X", "Y"): torch.zeros(2, 1, 3, 3, 3, dtype=torch.bool)})


def test_mixed_with_sparse_or_features_refused():
    import emu

    F_, _ = __import__("mcc_feature_nets").features(B200)
    for extra in ("sparse", "feature"):
        net, inputs = _small(B200, learning=False)
        Z = B200.nodes.LIFNodes(5)
        net.add_layer(Z, "Z")
        if extra == "sparse":
            c = B200.topology.SparseConnection(net.layers["Y"], Z, w=torch.rand(16, 5))
        else:
            c = B200.topology.MulticompartmentConnection(net.layers["Y"], Z, pipeline=[F_.Mask("m", torch.rand(16, 5) < 0.5),
                                                                                       F_.Weight("w", torch.rand(16, 5))])
        net.add_connection(c, "Y", "Z")
        with emu.EmuBackend(), pytest.raises(NotImplementedError, match="Conv3dConnection"):
            net.run(inputs=inputs, time=4)


def test_other_kinds_stay_refused():
    X, Y = B200.nodes.Input(shape=[1, 6, 6]), B200.nodes.LIFNodes(shape=[2, 2, 2])
    for cls in (B200.topology.Conv1dConnection, B200.topology.LocalConnection1D, B200.topology.LocalConnection3D,
                B200.topology.MaxPool1dConnection, B200.topology.MaxPoo3dConnection):
        with pytest.raises(NotImplementedError):
            cls(X, Y, 3)


def test_construction_attributes_match_reference():
    for ns in (_reference(), B200):
        if ns is None:
            continue
        X, Y = ns.nodes.Input(shape=[2, 7, 9, 8]), ns.nodes.LIFNodes(shape=[3, 4, 3, 9])
        for kw, draw in ((dict(wmin=0.2, wmax=0.7), lambda: 0.5 * torch.rand(3, 2, 3, 2, 4) + 0.2),
                         (dict(wmax=0.7), lambda: torch.rand(3, 2, 3, 2, 4).clamp(max=0.7))):
            torch.manual_seed(4)
            c = ns.topology.Conv3dConnection(X, Y, kernel_size=(3, 2, 4), stride=(2, 3, 1), padding=(1, 0, 2), **kw)
            assert (c.kernel_size, c.stride, c.padding, c.dilation, c.in_channels, c.out_channels) == \
                ((3, 2, 4), (2, 3, 1), (1, 0, 2), (1, 1, 1), 2, 3)
            torch.manual_seed(4)
            torch.testing.assert_close(c.w.data, draw(), rtol=0, atol=1e-7)
            assert torch.equal(c.b.data, torch.zeros(3))


# ---- 5. tier selection -----------------------------------------------------------------------------------------------

def test_tier_selection():
    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    net, inputs = _small(B200, rule="PostPre", nu=[0.0, 0.0], wmin=0.0, wmax=1.0)

    def tier(force):
        plan, keep = _plan.build_net(net, 2, {}, {}, {}, {}, {})
        opts = _abi.SnnRunOpts()
        opts.T, opts.B, opts.tier = 4, 2, force
        return int(emu.lib().snn_b200_select_tier(C.byref(plan), C.byref(opts)))

    assert tier(0) == 1 and tier(1) == 1 and tier(2) == 0 and tier(3) == 0
    net.force_tier = 3
    with emu.EmuBackend(), pytest.raises(RuntimeError, match="not implemented"):
        net.run(inputs=inputs, time=4)
    net.force_tier = 0
    with emu.EmuBackend():
        net.run(inputs=inputs, time=4)
    assert emu.last_tier == 1


# ---- 6. the reference's own objects through the ABI -----------------------------------------------------------------

@pytest.mark.parametrize("case", ["example_b1_noop", "c2_zero_rate_postpre"])
def test_reference_binding_runs_the_references_network(case):
    ref = _reference()
    if ref is None:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb
    import conv3d_oracle

    (a, inputs, T), (b, _, _) = cn.build_case(ref, case), cn.build_case(ref, case)
    a.run(inputs={"X": inputs["X"][0].clone()}, time=T)
    assert rb.run_window(b, {"X": inputs["X"][0].clone()}, time=T, library=conv3d_oracle.lib()) == 0
    sa, sb = cn.state(a), cn.state(b)
    for k in (k for k in sa if "/" in k):   # (the binding runs the window; the reference's monitors are not its business)
        if k.endswith("s"):
            assert torch.equal(sa[k], sb[k]), k
        else:
            torch.testing.assert_close(sb[k], sa[k], rtol=1e-4, atol=1e-4, msg=k)
    assert sa["Ys"].sum() > 0


def test_reference_binding_refuses_presynaptic_learning():
    ref = _reference()
    if ref is None:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb
    import conv3d_oracle

    net, inputs = _small(ref, rule="PostPre", nu=[1e-3, 1e-3], wmin=0.0, wmax=1.0)
    with pytest.raises(RuntimeError, match="same dtype"):
        rb.run_window(net, {"X": inputs["X"]}, time=4, library=conv3d_oracle.lib())


# ---- 7. the multi-GPU combine: sum + clamp on the flattened filters, then the connection's own normalize ------------

def _dist_make(B):
    return cn.multi_net(B200, rule="PostPre", weight_decay=1e-2, wmin=0.05, wmax=0.45, B=B, T=12)[0]


def _dist_inputs():
    return cn.multi_net(B200, B=8, T=12)[1]["X"]


def _dist_worker(rank, world, port, out):
    import torch.distributed as dist

    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from bindsnet_b200.distributed import ShardedWindowRunner
    from conv3d_oracle import Conv3dOracleBackend
    from test_distributed import _patch_cpu_combine

    _patch_cpu_combine()
    shard = _dist_inputs()[:, :, rank * 4:(rank + 1) * 4]
    net = _dist_make(4)
    with Conv3dOracleBackend():
        runner = ShardedWindowRunner(net)
        for window in range(2):
            if window:
                net.reset_state_variables()
            runner.run({"X": shard[window]}, time=12)
    torch.save({f"{s}->{t}": c.w.detach().clone() for (s, t), c in net.connections.items()}, os.path.join(out, f"rank{rank}.pt"))
    dist.destroy_process_group()


def test_two_rank_combine_normalizes_conv3d_filters(tmp_path):
    import numpy as np
    import torch.multiprocessing as mp
    from conv3d_oracle import Conv3dOracleBackend

    port = 33500 + (os.getpid() % 1000)
    mp.spawn(_dist_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    assert all(torch.equal(r0[k], r1[k]) for k in r0), "ranks diverged"

    x = _dist_inputs()
    nets = [_dist_make(4), _dist_make(4)]
    keys = list(nets[0].connections)
    w = {k: nets[0].connections[k].w.detach().clone() for k in keys}
    with Conv3dOracleBackend():
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
    torch.testing.assert_close(sums, torch.full_like(sums, 5.0), rtol=1e-5, atol=1e-5)
