"""SparseConnection (reference: topology.py:2009-2017): a Connection whose w is a torch.sparse_coo tensor, run on the
generic window kernel as a CSR gather.  CPU tests: the oracle against the live reference's stored results, the emulated
kernel against the oracle bit for bit, and the host API.  "The oracle" here is tests/sparse_oracle.c: the CPU oracle
extended by the sparse kind, restated over the CSR.  The stored reference results are regenerated with
``python tests/golden/gen_live.py test_sparse_connection``."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import cases
import helpers
import sparse_nets as sn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


# ---- 1. the oracle against the live reference ------------------------------------------------------------------------

@reference_side([False, True])
def _live_sparse(ns, decay):
    return sn.live_state(sn.run_live(ns, decay))


@pytest.mark.parametrize("decay", [False, True])
def test_oracle_matches_live_reference(decay):
    from sparse_oracle import SparseOracleBackend as OracleBackend

    ref = load(_live_sparse, decay)
    net, inputs = sn.live_net(B200, decay)
    with OracleBackend() as ob:
        net.run(inputs=inputs, time=sn.T_LIVE)
    assert ob.err == 0
    ours = sn.live_state(net)
    assert torch.equal(ours["Ys"], ref["Ys"]), "spike rasters differ"
    for k in ("X/x", "Y/x", "Y/v", "Y/refrac_count", "ZY/w"):
        torch.testing.assert_close(ours[k], ref[k], rtol=1e-5, atol=1e-4, msg=k)
    for c in ("XY", "YY"):
        assert torch.equal(ours[f"{c}/idx"], ref[f"{c}/idx"]), f"{c}: stored indices differ"
        torch.testing.assert_close(ours[f"{c}/val"], ref[f"{c}/val"], rtol=1e-5, atol=1e-6)
    assert net.connections[("X", "Y")].w.is_sparse


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

def _emu_vs_oracle(build, T, env=None, windows=1, one_step=False):
    import emu
    from sparse_oracle import SparseOracleBackend as OracleBackend

    outs = []
    for backend in (emu.EmuBackend, OracleBackend):
        net, inputs, *_ = build()
        net.force_tier = 1
        old = {k: os.environ.get(k) for k in (env or {})}
        os.environ.update(env if backend is emu.EmuBackend and env else {})
        try:
            with backend() as be:
                for _ in range(windows):
                    net.run(inputs=inputs, time=T, one_step=one_step)
                assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
        outs.append(sn.snapshot(net, T))
    return outs


ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("decay", [False, True])
def test_emulated_kernel_live_case_bit_exact(decay, env):
    def build():
        net, inputs = sn.live_net(B200, decay)
        helpers.add_spike_monitors(net, sn.T_LIVE)
        return net, inputs
    a, b = _emu_vs_oracle(build, sn.T_LIVE, ENVS[env])
    helpers.assert_bit_identical(a, b, f"live case decay={decay} {env}")


@pytest.mark.parametrize("seed", list(range(12)))
def test_emulated_kernel_random_sparse_networks_bit_exact(seed):
    env = list(ENVS.values())[seed % 4]
    spec = sn.random_net(B200, seed)[2]
    a, b = _emu_vs_oracle(lambda: sn.random_net(B200, seed), spec["T"], env, windows=2, one_step=spec["one_step"])
    helpers.assert_bit_identical(a, b, f"seed {seed} {spec}")


def test_emulated_kernel_large_index_bit_exact():
    """n_src * n_tgt > 2**31: no index of the sparse path may be formed as i * n_tgt in 32 bits."""
    a, b = _emu_vs_oracle(lambda: sn.big_index_net(B200), 4)
    helpers.assert_bit_identical(a, b, "50 000 x 50 000")
    assert a["L/Y/count"].sum() > 0


def test_emulated_sparse_equals_dense_connection():
    """SparseConnection(w=S) and Connection(w=S.to_dense()) give the same bits (absent entries add +0 to a sum that
    started at +0) — with the NoOp decay too."""
    import emu

    for decay in (False, True):
        outs = []
        for dense in (False, True):
            net, inputs = sn.live_net(B200, decay, dense_recurrent=dense, dense_input=dense)
            net.force_tier = 1
            with emu.EmuBackend() as be:
                net.run(inputs=inputs, time=sn.T_LIVE)
            assert be.err == 0
            st = {k: v for k, v in sn.live_state(net).items() if not k.startswith(("XY", "YY"))}
            st["XY"] = net.connections[("X", "Y")].w.detach()
            outs.append(st)
        for k in outs[0]:
            a, b = outs[0][k], outs[1][k]
            if a.is_sparse:   # the stored values equal the dense matrix at the stored positions
                a = a.coalesce()
                assert torch.equal(a.values().view(torch.int32), b[a.indices()[0], a.indices()[1]].view(torch.int32)), k
            else:
                assert torch.equal(a.view(torch.int32) if a.is_floating_point() else a, b.view(torch.int32) if b.is_floating_point() else b), k


# ---- 3. host API -------------------------------------------------------------------------------------------------

def _decayed(v0, factor, steps):
    v = v0.clone()
    for _ in range(steps):
        v = v * torch.tensor(factor, dtype=torch.float32)
    return v


def test_w_stays_sparse_and_shows_the_decay():
    import emu

    net, inputs = sn.live_net(B200, True)
    c = net.connections[("X", "Y")]
    v0 = c.w.detach().coalesce().values().clone()
    with emu.EmuBackend():
        net.run(inputs=inputs, time=5)
    assert c.w.is_sparse and c.w.layout == torch.sparse_coo and isinstance(c.w, torch.nn.Parameter)
    assert torch.equal(c.w.coalesce().values(), _decayed(v0, 0.9, 5))


def test_uncoalesced_and_replaced_w_are_honoured():
    import emu

    def run(w_first, w_second=None):
        net, inputs = sn.live_net(B200, False)
        c = net.connections[("X", "Y")]
        c.w = torch.nn.Parameter(w_first, requires_grad=False)
        with emu.EmuBackend():
            net.run(inputs=inputs, time=20)
            if w_second is not None:
                c.w = torch.nn.Parameter(w_second, requires_grad=False)
                net.run(inputs=inputs, time=20)
        return sn.snapshot(net, 20)

    g = torch.Generator().manual_seed(9)
    dense = sn._pattern(64, 48, 0.2, 8.0, g)
    S = dense.to_sparse()
    # the same matrix, uncoalesced: entries split in two halves and listed in reverse order
    idx, val = S.indices(), S.values()
    half = val / 2
    U = torch.sparse_coo_tensor(torch.cat([idx, idx], 1).flip(1), torch.cat([half, val - half]).flip(0), S.shape)
    assert not U.is_coalesced()
    a, b = run(S.coalesce() * 1.0), run(U)
    # coalescing sums the halves: compare with the matrix they sum to
    S2 = U.coalesce()
    c2 = run(S2)
    helpers.assert_bit_identical(b, c2, "uncoalesced w")
    # a w assigned between runs takes effect (the cached CSR follows the new index tensor)
    other = sn._pattern(64, 48, 0.3, 9.0, torch.Generator().manual_seed(10)).to_sparse()
    r1 = run(S, other)
    net, inputs = sn.live_net(B200, False)
    net.connections[("X", "Y")].w = torch.nn.Parameter(S, requires_grad=False)
    with emu.EmuBackend():
        net.run(inputs=inputs, time=20)
        net.connections[("X", "Y")].w = torch.nn.Parameter(sn._pattern(64, 48, 0.3, 9.0, torch.Generator().manual_seed(10)).to_sparse(),
                                                           requires_grad=False)
        net.run(inputs=inputs, time=20)
    helpers.assert_bit_identical(r1, sn.snapshot(net, 20), "replaced w")
    assert not np.array_equal(r1["L/Y/v"], a["L/Y/v"])   # the second pattern did change the run


def test_refusals():
    from bindsnet_b200 import _backend
    from bindsnet_b200.network.monitors import NetworkMonitor
    import emu

    T, L, N = B200.topology, B200.learning, B200.nodes
    X, Y = N.Input(10, traces=True), N.LIFNodes(7, traces=True)
    for rule in (L.PostPre, L.WeightDependentPostPre, L.Hebbian, L.MSTDP):
        with pytest.raises(NotImplementedError, match="fixed synapse pattern"):
            T.SparseConnection(X, Y, update_rule=rule, nu=0.01, wmin=0.0, wmax=1.0)
    with pytest.raises(NotImplementedError, match="norm"):
        T.SparseConnection(X, Y, norm=1.0)
    net, inputs = sn.live_net(B200, False)
    with emu.EmuBackend():
        with pytest.raises(NotImplementedError, match="Mask"):
            net.run(inputs=inputs, time=3, masks={("X", "Y"): torch.zeros(64, 48, dtype=torch.bool)})
        with pytest.raises(NotImplementedError, match="Mask"):
            net.connections[("X", "Y")].update(mask=torch.zeros(64, 48, dtype=torch.bool))
        c = net.connections[("X", "Y")]
        c.norm = 1.0      # set after construction: the library refuses the normalize
        with pytest.raises(_backend.BackendError, match="not implemented"):
            c.normalize()
        with pytest.raises(RuntimeError, match="not implemented"):   # the library refuses the plan (BackendError on CUDA)
            net.run(inputs=inputs, time=3)
    net, inputs = sn.live_net(B200, False)
    with pytest.raises(NotImplementedError, match="sparse"):
        NetworkMonitor(net, state_vars=["w"])


def test_compute_single_operator_matches_oracle_and_dense():
    import emu
    from sparse_oracle import SparseOracleBackend as OracleBackend

    net, _ = sn.live_net(B200, False)
    c = net.connections[("X", "Y")]
    s = torch.rand(5, 64, generator=torch.Generator().manual_seed(3)) < 0.3
    with emu.EmuBackend():
        a = c.compute(s)
    with OracleBackend():
        b = c.compute(s)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    dense = s.float() @ c.w.to_dense() + c.b
    torch.testing.assert_close(a, dense, rtol=1e-6, atol=1e-5)


def test_scripted_tier_matches_oracle():
    """A user-defined population as the target: the network runs step by step, the sparse connections through their
    single-operator compute / update.  The emulated kernels and the oracle give the same bits, and the window of the
    built-in LIFNodes (on the oracle) the same result."""
    import emu
    from sparse_oracle import SparseOracleBackend as OracleBackend
    from test_scripted_tier import MyLIF

    def build(user):
        g = torch.Generator().manual_seed(77)
        T_, N = B200.topology, B200.nodes
        net = B200.Network(dt=1.0, batch_size=3, learning=True)
        X = N.Input(64)
        Y = MyLIF(48, tc_decay=40.0, refrac=3) if user else N.LIFNodes(48, tc_decay=40.0, refrac=3)
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        kw = dict(update_rule=B200.learning.NoOp, weight_decay=0.1)
        net.add_connection(T_.SparseConnection(X, Y, w=sn._pattern(64, 48, 0.1, 9.0, g).to_sparse(), b=0.2 * torch.rand(48, generator=g), **kw), "X", "Y")
        net.add_connection(T_.SparseConnection(Y, Y, w=sn._pattern(48, 48, 0.15, -4.0, g).to_sparse(), **kw), "Y", "Y")
        x = (torch.rand(30, 3, 64, generator=g) < 0.12).to(torch.uint8)
        return net, {"X": x}

    outs = []
    for user, backend in ((True, emu.EmuBackend), (True, OracleBackend), (False, OracleBackend)):
        net, inputs = build(user)
        assert net._scripted_required() == user
        with backend():
            net.run(inputs=inputs, time=30)
        outs.append(sn.snapshot(net, 30))
    helpers.assert_bit_identical(outs[0], outs[1], "scripted tier: emulated single operators vs oracle")
    assert outs[0]["L/Y/s"].sum() > 0 or (outs[0]["L/Y/v"] != -65.0).any()
    for k in outs[2]:
        np.testing.assert_allclose(outs[0][k].astype(np.float64), outs[2][k].astype(np.float64), rtol=1e-5, atol=1e-4, err_msg=k)


def test_noop_sparse_weights_stay_out_of_the_multi_gpu_combine():
    from bindsnet_b200.distributed import ShardedWindowRunner

    net, _ = sn.live_net(B200, True)
    learned = ShardedWindowRunner._learned(SimpleNamespace(network=net))
    assert [type(c).__name__ for c, _ in learned] == ["Connection"]


def test_reference_binding_runs_the_references_sparse_network():
    """The reference's own SparseConnection network, its ABI filled by reference_binding and run by the oracle library,
    against the reference's own run."""
    try:
        ref = cases.namespace("reference")
    except ImportError:
        pytest.skip("oracle/_ref/bindsnet is missing: build() copies the reference there from its checkout")
    from bindsnet_b200 import reference_binding as rb
    import sparse_oracle

    for decay in (False, True):
        a, inputs = sn.live_net(ref, decay)
        b, _ = sn.live_net(ref, decay)
        a.run(inputs={k: v.clone() for k, v in inputs.items()}, time=sn.T_LIVE)
        assert rb.run_window(b, {k: v.clone() for k, v in inputs.items()}, time=sn.T_LIVE, library=sparse_oracle.lib()) == 0
        sa, sb = sn.live_state(a), sn.live_state(b)
        for k in ("Y/v", "Y/x", "X/x", "ZY/w"):
            torch.testing.assert_close(sb[k], sa[k], rtol=1e-5, atol=1e-4, msg=k)
        for c in ("XY", "YY"):
            assert torch.equal(sb[f"{c}/idx"], sa[f"{c}/idx"])
            torch.testing.assert_close(sb[f"{c}/val"], sa[f"{c}/val"], rtol=1e-5, atol=1e-6)


def test_sparse_oracle_runs_plans_without_a_sparse_connection_as_the_oracle_does():
    """tests/sparse_oracle.c hands every plan without a SparseConnection to the unchanged oracle's own functions."""
    from oracle.oracle import OracleBackend
    from sparse_oracle import SparseOracleBackend

    outs = []
    for backend in (OracleBackend, SparseOracleBackend):
        fx = helpers.Fixture("lif_postpre_batch")
        net, inputs, kw, T = fx.build("cpu")
        helpers.add_spike_monitors(net, T)
        with backend() as be:
            net.run(inputs=inputs, time=T, one_spike_seed=cases.ONE_SPIKE_SEED, **kw)
        assert be.err == 0
        outs.append({**helpers.snapshot(net), **helpers.spike_counts(net, T)})
    helpers.assert_bit_identical(outs[0], outs[1], "lif_postpre_batch through the sparse oracle")
