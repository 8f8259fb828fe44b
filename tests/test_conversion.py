"""ann_to_snn and its two layer kinds, SubtractiveResetIFNodes and PassThroughNodes (reference: bindsnet/conversion), on
the generic window kernel.  CPU tests: the conversion against the live reference's stored networks, the oracle
(tests/conversion_oracle.c) against the live reference's stored runs, the emulated kernel against the oracle bit for
bit, refusals and tier selection.  The stored reference results are regenerated with
``python tests/golden/gen_live.py test_conversion``."""
import hashlib
import os
import sys
import warnings

import pytest
import torch
import torch.nn as nn

import cases
import conversion_nets as cn
from live_golden import load, reference_side

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")
CONVERSIONS = ["fc_nodata", "fc_data", "cnn_nodata", "cnn_data"]
RUNS = ["cnn_b1", "cnn_b4", "subif_refrac", "subif_lbound", "subif_traces", "subif_postpre", "passthrough"]


def _build(ns, case):
    if case.startswith("cnn_b"):
        return cn.cnn_net(ns, int(case[5:]))
    if case.startswith("subif_"):
        return cn.subif_net(ns, case[6:])
    return cn.passthrough_net(ns)


def _describe(net) -> dict:
    """What ann_to_snn built: per layer its type, shape and sum_input; per connection (in order) its key, type, w, b."""
    out = {"layers": torch.tensor([ord(c) for c in "|".join(f"{k}:{type(v).__name__}:{tuple(v.shape)}:{int(v.sum_input)}"
                                                              for k, v in net.layers.items())])}
    keys = []
    for i, ((s, t), c) in enumerate(net.connections.items()):
        keys.append(f"{s}>{t}:{type(c).__name__}")
        for var in ("w", "b"):
            v = getattr(c, var, None)
            if isinstance(v, torch.Tensor):   # (large ones by a digest of their bytes: still a bit-for-bit check)
                v = v.detach().contiguous()
                out[f"c{i}/{var}"] = v.clone() if v.numel() <= 4096 else torch.tensor(list(hashlib.sha256(v.numpy().tobytes()).digest()))
    out["conns"] = torch.tensor([ord(c) for c in "|".join(keys)])
    return out


# ---- 1. the conversion and the oracle against the live reference -----------------------------------------------------

@reference_side(CONVERSIONS)
def _live_convert(ns, case):
    name, data = case.split("_")
    return _describe(cn.convert(ns, name, data == "data"))


@reference_side(RUNS)
def _live_run(ns, case):
    net, inputs, T = _build(ns, case)
    return cn.flat(cn.run_two_windows(net, inputs, T))


@pytest.mark.parametrize("case", CONVERSIONS)
def test_ann_to_snn_matches_live_reference(case):
    name, data = case.split("_")
    ref, ours = load(_live_convert, case), _describe(cn.convert(B200, name, data == "data"))
    assert ours.keys() == ref.keys()
    for k in ref:
        assert torch.equal(ours[k], ref[k]), f"{case}: {k} differs"   # names, types, shapes, keys; w and b bit-equal


def _check_against(ref, ours, what):
    assert ours.keys() == ref.keys(), what
    for k, v in ref.items():
        o = ours[k]
        assert o.shape == v.shape, (what, k)
        if k.endswith("/s") or k.endswith("/fr"):
            assert torch.equal(o.float(), v.float()), f"{what}: {k} differs"
        else:
            torch.testing.assert_close(o.float(), v.float(), rtol=1e-5, atol=1e-4, msg=f"{what}: {k}")


@pytest.mark.parametrize("case", RUNS)
def test_oracle_matches_live_reference(case):
    from conversion_oracle import ConversionOracleBackend

    net, inputs, T = _build(B200, case)
    with ConversionOracleBackend() as ob:
        ours = cn.flat(cn.run_two_windows(net, inputs, T))
    assert ob.err == 0
    ref = load(_live_run, case)
    _check_against(ref, ours, case)
    for k, v in ours.items():   # PassThroughNodes keep float32 spikes, as the reference's do after a step
        if k.endswith("/s") and (k.startswith("w1/M") or k.split("/")[1] in ("3", "6", "P", "Q")):
            assert v.dtype == torch.float32 and v.dtype == ref[k].dtype, k
    assert ours["w1/8/s" if case.startswith("cnn") else "w1/Y/s"].sum() > 0


def test_last_layer_sums_input_and_reference_quirks():
    conv = cn.conversion(B200)
    with pytest.warns(RuntimeWarning, match="Data is None"):
        net = conv.ann_to_snn(cn.model("cnn"), input_shape=(1, 28, 28))
    assert list(net.layers) == ["Input", "1", "3", "4", "6", "8", "10"]
    assert list(net.connections) == [("0", "1"), ("2", "3"), ("3", "4"), ("5", "6"), ("7", "8"), ("9", "10")]
    assert [bool(l.sum_input) for l in net.layers.values()] == [False] * 6 + [True]
    assert all(c.w.is_contiguous() for c in net.connections.values() if hasattr(c, "w"))
    # the ANN itself is left as it was (ann_to_snn converts a copy)
    m = cn.model("cnn")
    before = [p.clone() for p in m.parameters()]
    conv.ann_to_snn(m, input_shape=(1, 28, 28), data=cn.images("cnn", 8))
    assert all(torch.equal(a, b) for a, b in zip(before, m.parameters()))


def test_refusals():
    from conversion_oracle import ConversionOracleBackend

    conv = cn.conversion(B200)
    for module in (cn.conversion(B200).Permute((0, 2, 1)), nn.ConstantPad2d(1, 0.0)):
        with warnings.catch_warnings(), pytest.raises(TypeError):
            warnings.simplefilter("ignore", RuntimeWarning)
            conv.ann_to_snn(nn.Sequential(nn.Conv2d(1, 2, 3), module, nn.Flatten(), nn.Linear(2 * 26 * 26, 3)), (1, 28, 28), data=None)
    # nn.Conv2d without bias: a zero bias of the output height, refused when the plan is built (before anything runs)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        net = conv.ann_to_snn(cn.small_cnn(conv_bias=False), input_shape=(1, 28, 28))
    net.train(False)
    with ConversionOracleBackend() as ob, pytest.raises(RuntimeError, match="expected bias"):
        net.run({"Input": torch.zeros(4, 1, 1, 28, 28, dtype=torch.bool)}, time=4)
    # learning on (ann_to_snn's default): the pooling connection's NoOp update fails, as in the reference
    net, inputs, T = cn.cnn_net(B200, 1, T=4)
    net.train(True)
    with ConversionOracleBackend(), pytest.raises(AttributeError):
        net.run({"Input": inputs["Input"][0]}, time=T)
    # a connection into a PassThroughNodes layer that is not a pooling one, and a rule at a PassThroughNodes end
    for bad in ("dense_into", "postpre_from"):
        n2 = B200.Network(learning=False)
        X, P = B200.nodes.Input(4, traces=True), conv.PassThroughNodes(4, traces=True)
        Y = conv.SubtractiveResetIFNodes(3, traces=True)
        for name, l in (("X", X), ("P", P), ("Y", Y)):
            n2.add_layer(l, name)
        if bad == "dense_into":
            n2.add_connection(B200.topology.Connection(X, P, w=torch.eye(4)), "X", "P")
        else:
            n2.add_connection(B200.topology.Connection(P, Y, w=torch.ones(4, 3), update_rule=B200.learning.PostPre, nu=0.1), "P", "Y")
        with ConversionOracleBackend(), pytest.raises(NotImplementedError):
            n2.run({"X": torch.zeros(3, 1, 4, dtype=torch.bool), "P": torch.zeros(3, 1, 4)}, time=3)


def test_nonbinary_passthrough_input_is_flagged():
    from conversion_oracle import ConversionOracleBackend

    import emu

    for backend in (ConversionOracleBackend, emu.EmuBackend):
        net, inputs, T = cn.passthrough_net(B200)
        x = inputs["P"][0].clone()
        x[3, 0, 0, 0, 0] = 2.0
        with backend() as be:
            net.run({"P": x}, time=T)
        assert be.err & 16, backend


# ---- 2. the emulated kernel against the oracle, bit for bit ----------------------------------------------------------

ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"},
        "shuffle": {"SNN_EMU_SHUFFLE": "3", "SNN_EMU_SMS": "2"}}


def _emu_vs_oracle(build, env=None, **kw):
    import emu
    from conversion_oracle import ConversionOracleBackend

    outs = []
    for backend in (emu.EmuBackend, ConversionOracleBackend):
        net, inputs, T = build()
        net.force_tier = 1
        old = {k: os.environ.get(k) for k in (env or {})}
        os.environ.update(env if backend is emu.EmuBackend and env else {})
        try:
            with backend() as be:
                outs.append(cn.flat(cn.run_two_windows(net, inputs, T, **kw)))
            assert be.err == 0
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        if backend is emu.EmuBackend:
            assert emu.last_tier == 1
    a, b = outs
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), f"{k} differs"
    return a


@pytest.mark.parametrize("env", list(ENVS))
@pytest.mark.parametrize("case", ["cnn_b4", "subif_refrac", "passthrough"])
def test_emulated_kernel_bit_exact(case, env):
    _emu_vs_oracle(lambda: _build(B200, case), ENVS[env])


@pytest.mark.parametrize("case", ["cnn_b1", "subif_lbound", "subif_traces", "subif_postpre"])
def test_emulated_kernel_more_cases_bit_exact(case):
    _emu_vs_oracle(lambda: _build(B200, case), ENVS["sms3"])


@pytest.mark.parametrize("case", ["cnn_b4", "passthrough", "subif_refrac"])
def test_emulated_kernel_one_step_bit_exact(case):
    _emu_vs_oracle(lambda: _build(B200, case), ENVS["sms3"], one_step=True)


def test_emulated_kernel_large_batch_odd_T_bit_exact():
    """B = 520 (> 512) and an odd window length."""
    a = _emu_vs_oracle(lambda: cn.cnn_net(B200, 520, T=7, monitors=False), ENVS["sms3"])
    assert a["w1/4/s"].sum() > 0


def test_stepwise_and_scripted_equal_window():
    """A Monitor on a variable the kernels do not record runs the window step by step; a user-defined layer runs it on
    the scripted tier (each built-in piece on its single-operator kernel).  Both give the window's result."""
    import emu

    conv = cn.conversion(B200)

    class UserIF(conv.SubtractiveResetIFNodes):   # a population of the user's: its own forward, the same arithmetic
        kind = None

        def forward(self, x):
            self.v += (self.refrac_count == 0).float() * x
            self.refrac_count = (self.refrac_count > 0).float() * (self.refrac_count - self.dt)
            self.s = self.v >= self.thresh
            self.refrac_count.masked_fill_(self.s, float(self.refrac))
            self.v[self.s] = self.v[self.s] - self.thresh
            B200.nodes.Nodes.forward(self, x)

    outs = []
    for mode in ("window", "stepwise", "scripted"):
        net, inputs, T = cn.passthrough_net(B200, T=12)
        if mode == "stepwise":
            net.add_monitor(B200.monitors.Monitor(net.layers["C"], ["refrac_count"], time=T), "rc")
        if mode == "scripted":
            old = net.layers["Y"]
            user = UserIF(5, thresh=1.0, reset=0.0, refrac=0, sum_input=True)
            net.layers["Y"] = user
            user.dt = old.dt
            user.set_batch_size(2)
            net.connections[("Q", "Y")].target = user
        with emu.EmuBackend() as be:
            states = cn.run_two_windows(net, inputs, T)
        assert be.err == 0
        outs.append({k: v for k, v in cn.flat(states).items() if "/rc/" not in k})
    for other in outs[1:]:
        assert outs[0].keys() == other.keys()
        for k in outs[0]:
            assert torch.equal(outs[0][k].float(), other[k].float()), k


def test_passthrough_equals_mcculloch_pitts_downstream():
    """On 0 / 1 input a PassThroughNodes layer spikes exactly where McCullochPitts(thresh=1) does: everything downstream
    is identical."""
    import emu

    outs = []
    for twin in (False, True):
        net, inputs, T = cn.cnn_net(B200, 3, monitors=False)
        if twin:
            for name in ("3", "6"):
                old = net.layers[name]
                mcp = B200.nodes.McCullochPitts(shape=old.shape, thresh=1.0)
                net.add_layer(mcp, name)
                for c in net.connections.values():
                    c.source = mcp if c.source is old else c.source
                    c.target = mcp if c.target is old else c.target
            net.reset_state_variables()
        with emu.EmuBackend() as be:
            outs.append(cn.flat(cn.run_two_windows(net, inputs, T)))
        assert be.err == 0
    a, b = outs
    for k in a:
        if k.split("/")[1] not in ("3", "6"):
            assert torch.equal(a[k].float(), b[k].float()), k
    assert a["w1/8/s"].sum() > 0


def _ref_pool_net(ref):
    """Input [2, 6, 6] -> MaxPool2dConnection -> PassThroughNodes [2, 3, 3] -> dense Connection -> SubtractiveResetIFNodes(5)."""
    conv = cn.conversion(ref)
    g = torch.Generator().manual_seed(3)
    net = ref.Network(dt=1.0, batch_size=2, learning=False)
    X, P = ref.nodes.Input(shape=[2, 6, 6]), conv.PassThroughNodes(shape=[2, 3, 3])
    Y = conv.SubtractiveResetIFNodes(5, thresh=1.0, reset=0.0, refrac=0, sum_input=True)
    for name, layer in (("X", X), ("P", P), ("Y", Y)):
        net.add_layer(layer, name)
    net.add_connection(ref.topology.MaxPool2dConnection(X, P, kernel_size=2, stride=2, decay=1), "X", "P")
    net.add_connection(ref.topology.Connection(P, Y, w=0.5 * torch.rand(18, 5, generator=g)), "P", "Y")
    net.reset_state_variables()
    return net, rate_inputs_x(), 16


def rate_inputs_x():
    return cn.rate_inputs((2, 6, 6), 16, 2, seed=4, windows=1, p=0.8)[0]


@pytest.mark.parametrize("which", ["fc", "pool"])
def test_reference_network_through_reference_binding(which):
    """The reference's own networks — ann_to_snn of the fully connected model, and a pooling network with a
    PassThroughNodes layer — bound by reference_binding (their own objects filled into the ABI) and run by the oracle,
    reproduce the reference's own run."""
    from bindsnet_b200 import reference_binding as rb
    from conversion_oracle import lib

    ref = cases.namespace("reference")
    nets = []
    for _ in range(2):
        if which == "fc":
            net = cn.convert(ref, "fc", data=True)
            net.train(False)
            cn.set_batch(net, 2)
            x, T = cn.rate_inputs((784,), 16, 2, seed=9, windows=1, p=0.9)[0], 16
        else:
            net, x, T = _ref_pool_net(ref)
        nets.append(net)
    ours, theirs = nets
    theirs.run({next(iter(theirs.layers)): x.clone()}, time=T)
    if which == "pool":
        assert ours.layers["P"].s.dtype == torch.bool   # before its first run a PassThroughNodes' s is still bool
    assert rb.run_window(ours, {next(iter(ours.layers)): x.clone()}, time=T, library=lib()) == 0
    for name, layer in theirs.layers.items():
        other = ours.layers[name]
        assert torch.equal(layer.s.float(), other.s.float()), name
        for var in ("v", "refrac_count", "summed"):
            if isinstance(getattr(layer, var, None), torch.Tensor) and getattr(layer, var).numel():
                torch.testing.assert_close(getattr(other, var), getattr(layer, var), rtol=1e-5, atol=1e-4)
    if which == "pool":
        assert ours.layers["P"].s.dtype == torch.float32 and ours.layers["P"].s.sum() > 0


# ---- 3. plan checks and tier selection ---------------------------------------------------------------------------------

def test_tier_selection_and_abi_constants():
    import re

    import emu
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "snn_b200.h")).read()
    for name in ("SNN_NODE_SUBIF", "SNN_NODE_PASSTHROUGH"):
        assert int(re.search(rf"#define\s+{name}\s+(\d+)", header).group(1)) == getattr(_abi, name)
    assert (_abi.SNN_NODE_SUBIF, _abi.SNN_NODE_PASSTHROUGH) == (7, 8)
    assert _abi.SNN_MAX_LAYERS == 8 and _abi.SNN_MAX_CONNS == 12
    L = emu.lib()
    for case in ("subif_refrac", "passthrough"):
        net, inputs, T = _build(B200, case)
        nd, keep = _plan.build_net(net, net.batch_size, {}, {}, {}, {}, {})
        for tier, want in ((0, 1), (1, 1), (2, 0), (3, 0)):
            opts = _abi.SnnRunOpts()
            opts.T, opts.B, opts.tier = T, net.batch_size, tier
            assert L.snn_b200_select_tier(nd, opts) == want, (case, tier)
        opts.tier = 2
        ws = torch.zeros(1 << 20, dtype=torch.uint8)
        assert L.snn_b200_run_window(nd, opts, ws.data_ptr(), ws.numel(), None) == _abi.SNN_ERR_UNSUPPORTED
    # LeNet-5 converted is exactly 8 layers and 7 connections; one more layer is refused with the existing error
    net = cn.convert(B200, "lenet5", data=False)
    assert (len(net.layers), len(net.connections)) == (8, 7)
    net.add_layer(cn.conversion(B200).SubtractiveResetIFNodes(3), "extra")
    with pytest.raises(NotImplementedError, match="layers"):
        _plan.build_net(net, 1, {}, {}, {}, {}, {})
