"""The generic kernel's learning paths that only run inside a window — dense MSTDP / MSTDPET (and their
MulticompartmentConnection forms), the rules of a Conv2dConnection and of a LocalConnection2D — and phase 1's
convolutional and local gathers, at the shapes where their paths switch (cases, float64 restatements and path mirrors:
tests/learning_edges.py).  CPU tests: the oracle against a plain float64 restatement of the reference's formulas within a
rounding-error bound, and the kernels' CUDA source under the CPU emulation (tests/emu) against the oracle, bit for bit,
weights and rule state alike."""
import os
import sys

import pytest
import torch

import cases
import learning_edges as le
from test_kernel_edges import _assert_bit_identical, _assert_within_bound, _emu, _with

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


def oracle_for(kind: str, rule: str = ""):
    """The oracle library that holds the case's connection kinds (the CPU oracle, or its extensions by the
    MulticompartmentConnection reward rules and by LocalConnection2D)."""
    if rule.startswith("mcc"):
        from mcc_reward_oracle import RewardOracleBackend

        return RewardOracleBackend
    if kind == "local":
        from local2d_oracle import Local2dOracleBackend

        return Local2dOracleBackend
    from oracle.oracle import OracleBackend

    return OracleBackend


def run_case(case, d, backend, env=None, spans=None):
    st, net = _with(backend, lambda: le.run_window(B200, case, d, spans=spans), env)
    if backend is _emu():
        import emu

        assert emu.last_tier == 1
    return st, net


def check_against_float64(case, d, st, net):
    """Y's raster is Z's one step later; the weights (and the reward rules' traces) within the float64 bound; the
    case bites."""
    xd, yd = float(net.layers["X"].trace_decay), float(net.layers["Y"].trace_decay)
    w64, bound, raster, traces = le.ref_window(case, d, xd, yd)
    assert torch.equal(st["Ys"], raster.reshape(case.T, -1)), f"{case.name}: Y's raster is not Z's, one step later"
    r = _assert_within_bound(st["w"], w64, bound, case.name)
    if traces is not None:
        gam = le.gamma(2 * case.T + 2)
        for k, v64 in zip(("p_plus", "p_minus"), traces):
            _assert_within_bound(st[k].reshape(v64.shape), v64, gam * v64.abs(), f"{case.name} {k}")
    le.check_window_bites(case, d, st)
    return r


# ---- 1. window learning: the oracle against float64 ------------------------------------------------------------------

@pytest.mark.parametrize("case", le.WINDOW_CASES, ids=lambda c: c.name)
def test_window_oracle_within_float64_bound(case):
    d = le.draw_window(case)
    st, net = run_case(case, d, oracle_for(case.kind, case.rule))
    check_against_float64(case, d, st, net)


# ---- 2. window learning: the emulated kernel against the oracle, bit for bit -----------------------------------------

def _emu_vs_oracle(case, env, spans=None):
    d = le.draw_window(case)
    a, _ = run_case(case, d, _emu(), env, spans)
    b, _ = run_case(case, d, oracle_for(case.kind, case.rule), None, spans)
    assert a.keys() == b.keys()
    for k in a:
        _assert_bit_identical(a[k].float(), b[k].float(), f"{case.name} {k}")
    return a


@pytest.mark.parametrize("case", le.WINDOW_CASES, ids=lambda c: c.name)
def test_window_emulated_kernel_bit_exact(case):
    _emu_vs_oracle(case, {"SNN_EMU_SMS": "3"})


def _small(c):
    return c.B * max(c.ns, c.geo.ns if c.geo else 0) <= 20000


SMS_CASES = [c for c in le.WINDOW_CASES if _small(c)][::3]


@pytest.mark.parametrize("sms", ["1", "7"])
@pytest.mark.parametrize("case", SMS_CASES, ids=lambda c: c.name)
def test_window_emulated_kernel_grid_sizes_bit_exact(case, sms):
    """One and seven emulated SMs: the units of the learning phase land on other CTAs."""
    _emu_vs_oracle(case, {"SNN_EMU_SMS": sms})


def _case(prefix):
    return next(c for c in le.WINDOW_CASES if c.name.startswith(prefix))


SHUFFLED = ["conv_mstdp_b4_t3_sum_c3x10x11", "dense_mstdp_b33_t4_mean_31x45", "local_wdep_b3"]


@pytest.mark.parametrize("prefix", SHUFFLED)
def test_window_emulated_kernel_shuffled_schedule_bit_exact(prefix):
    _emu_vs_oracle(_case(prefix), {"SNN_EMU_SHUFFLE": "11", "SNN_EMU_SMS": "2"})


@pytest.mark.parametrize("prefix", ["conv_mstdp_b4_t3_sum_c3x10x11", "dense_mstdp_b3_t4", "dense_mstdpet_b1_t4",
                                    "dense_mcc_mstdp_b5"])
def test_rule_state_across_windows_of_odd_and_even_length(prefix):
    """The rule state is double-buffered (slot (t + T) & 1): windows of 3 and 2 steps must hand it on like one of 5,
    and the emulated kernel must equal the oracle."""
    case = le.replace(_case(prefix), T=5)
    whole = _emu_vs_oracle(case, {"SNN_EMU_SMS": "3"})
    split = _emu_vs_oracle(case, {"SNN_EMU_SMS": "3"}, spans=[3, 2])
    for k in whole:
        _assert_bit_identical(split[k].float(), whole[k].float(), f"{case.name} {k} split vs whole")


# ---- 3. the cases reach both sides of every switch ---------------------------------------------------------------------

def test_cases_reach_both_sides_of_every_switch():
    sides = {}
    for c in le.WINDOW_CASES:
        for k, v in c.paths().items():
            sides.setdefault(("window", c.kind, c.rule if c.kind != "dense" else "dense", k), set()).add(v)
        for k, side in c.claims:
            assert c.paths()[k] == side, (c.name, k)
    for c in le.GATHER_CASES:
        for k, v in c.paths().items():
            sides.setdefault(("gather", c.kind, k), set()).add(v)
        for k, side in c.claims:
            assert c.paths()[k] == side, (c.name, k)
    need = {
        ("window", "conv", "mstdp", "listed"): {True, False},
        ("window", "conv", "mstdp", "staged"): {True, False},
        ("window", "conv", "mstdp", "stage_pm"): {True, False},
        ("window", "conv", "mstdp", "unit_stride"): {True, False},
        ("window", "conv", "mstdp", "multi_channel"): {True, False},
        ("window", "conv", "mstdp", "shuffle_tail"): {True, False},
        ("window", "dense", "dense", "dense_staged"): {True, False},
        ("window", "dense", "dense", "several_tiles"): {True, False},
        ("gather", "conv", "st_bits"): {True, False},
        ("gather", "conv", "st_taps_all"): {True, False},
        ("gather", "conv", "funnel"): {True, False},
        ("gather", "conv", "two_convs"): {True, False},
        ("gather", "local", "kw_over_32"): {True, False},
        ("gather", "local", "st_bits"): {True},
    }
    for k, want in need.items():
        assert want <= sides.get(k, set()), f"{k}: reached {sides.get(k)}, want {want}"
    cpcs = {c.paths()["cpc"] for c in le.WINDOW_CASES if c.kind == "conv" and c.rule == "mstdp"}
    assert 1 in cpcs and max(cpcs) > 1
    margins = {c.paths()["slist_margin"] for c in le.WINDOW_CASES if c.kind == "conv" and c.rule == "mstdp"}
    assert {0, -1} <= margins
    conv_mstdp = [c for c in le.WINDOW_CASES if c.kind == "conv" and c.rule == "mstdp"]
    assert {1, 31, 32, 33, 65} <= {c.B for c in conv_mstdp} and any(c.red == "mean" for c in conv_mstdp)
    assert {256, 257} <= {c.geo.hin for c in conv_mstdp} and {256, 257} <= {c.geo.win for c in conv_mstdp}
    assert any(c.gain_first for c in conv_mstdp) and any(c.geo == le.C4 for c in conv_mstdp)
    assert any(c.geo.s == (2, 2) and c.geo.p == (1, 1) for c in conv_mstdp)
    dense = [c for c in le.WINDOW_CASES if c.kind == "dense"]
    assert {(128, 44), (128, 45), (768, 2), (769, 2)} <= {(c.B, c.nt) for c in dense if c.rule == "mstdp"}
    assert {1, 3, 33} <= {c.B for c in dense} and {31, 33, 784} <= {c.ns for c in dense}
    assert {(1, 6544), (1, 6545)} <= {(c.B, c.nt) for c in dense if c.rule == "mstdpet"}
    assert {"mcc_mstdp", "mcc_mstdpet"} <= {c.rule for c in dense}
    assert {r for c in dense for r in (("neg" if c.reward < 0 else "zero" if c.reward == 0 else "pos"),)} == {"neg", "zero", "pos"}
    for kind, rules in (("conv", le.CONV_RULES), ("local", le.LOCAL_RULES)):
        cs = [c for c in le.WINDOW_CASES if c.kind == kind]
        assert {c.rule for c in cs} == set(rules)
        assert any(c.red == "mean" for c in cs if c.rule != "mstdp")
    stdp_conv = [c for c in le.WINDOW_CASES if c.kind == "conv" and c.rule != "mstdp"]
    assert any(c.nu_off == 0 for c in stdp_conv) and any(c.nu_off == 1 for c in stdp_conv)
    assert any(c.geo.s != (1, 1) and c.geo.p != (0, 0) for c in stdp_conv) and any(c.geo.cin > 1 for c in stdp_conv)
    assert {1, 3} <= {c.geo.cin for c in le.WINDOW_CASES if c.kind == "local"}
    local_kw = {c.geos[0].k[1] for c in le.GATHER_CASES if c.kind == "local"}
    assert {32, 33, 40} <= local_kw
    conv_kw = {c.geos[0].k[1] for c in le.GATHER_CASES if c.kind == "conv" and c.geos[0].d == (1, 1)}
    assert {32, 33} <= conv_kw
    two = [c for c in le.GATHER_CASES if len(c.geos) > 1]
    assert any(a.geos == b.geos[::-1] for a in two for b in two if a is not b)


# ---- 4. phase-1 gathers --------------------------------------------------------------------------------------------

def _gather(case, backend, env=None):
    d = le.draw_gather(case)
    v = _with(backend, lambda: le.run_gather(B200, case, d), env)
    return v, d


@pytest.mark.parametrize("case", le.GATHER_CASES, ids=lambda c: c.name)
def test_gather_oracle_within_float64_bound(case):
    v, d = _gather(case, oracle_for(case.kind))
    v64, bound = le.ref_gather(B200, case, d)
    assert v.shape == v64.shape
    _assert_within_bound(v, v64, bound, case.name)
    assert (v[1:] != v[:1]).any(), f"{case.name}: the gather never changed"


@pytest.mark.parametrize("case", le.GATHER_CASES, ids=lambda c: c.name)
def test_gather_emulated_kernel_bit_exact(case):
    a, _ = _gather(case, _emu(), {"SNN_EMU_SMS": "3"})
    b, _ = _gather(case, oracle_for(case.kind))
    _assert_bit_identical(a, b, case.name)
    for k, side in case.claims:
        assert case.paths()[k] == side
