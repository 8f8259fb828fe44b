"""The generic kernel's Conv1dConnection, Conv3dConnection and LocalConnection3D paths — phase 1's gathers and their
staging, the learning phases, the normalize phase — and their single-operator twins, at the shapes where their paths
switch (cases, float64 restatements and path mirrors: tests/geometry_edges.py).  CPU tests: each kind's oracle against a
plain float64 restatement of the reference's formulas within a rounding-error bound, and the kernels' CUDA source under
the CPU emulation (tests/emu) against the oracle, bit for bit."""
import os
import sys

import pytest
import torch

import cases
import geometry_edges as ge
from test_kernel_edges import _emu, _with

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


def oracle_for(kind: str):
    """The oracle library that holds the kind (the CPU oracle extended by it)."""
    if kind == "conv1d":
        from conv1d_oracle import Conv1dOracleBackend

        return Conv1dOracleBackend
    if kind == "conv3d":
        from conv3d_oracle import Conv3dOracleBackend

        return Conv3dOracleBackend
    from local3d_oracle import Local3dOracleBackend

    return Local3dOracleBackend


def _assert_emulated_tier1(backend):
    if backend is _emu():
        import emu

        assert emu.last_tier == 1


def run_case(case, d, backend, env=None):
    st, net = _with(backend, lambda: ge.run_window(B200, case, d), env)
    _assert_emulated_tier1(backend)
    return st, net


def check_against_float64(case, d, st, net):
    """Y's raster is Z's one step later; the weights within the float64 bound; the case bites."""
    xd, yd = float(net.layers["X"].trace_decay), float(net.layers["Y"].trace_decay)
    w64, bound, raster, seen = ge.ref_window(case, d, xd, yd)
    assert torch.equal(st["Ys"], raster.reshape(case.T, -1)), f"{case.name}: Y's raster is not Z's, one step later"
    r = ge.assert_within_bound(st["w"], w64, bound, case.name)
    ge.check_window_bites(case, d, st, seen)
    return r


# ---- 1. windows: the oracle against float64, the emulated kernel against the oracle ------------------------------------

@pytest.mark.parametrize("case", ge.WINDOW_CASES, ids=lambda c: c.name)
def test_window_oracle_within_float64_bound(case):
    d = ge.draw_window(case)
    st, net = run_case(case, d, oracle_for(case.kind))
    check_against_float64(case, d, st, net)


def _emu_vs_oracle(case, env):
    d = ge.draw_window(case)
    a, _ = run_case(case, d, _emu(), env)
    b, _ = run_case(case, d, oracle_for(case.kind))
    for k in b:
        ge.assert_same(a[k], b[k], f"{case.name} {k}")


@pytest.mark.parametrize("case", ge.WINDOW_CASES, ids=lambda c: c.name)
def test_window_emulated_kernel_bit_exact(case):
    _emu_vs_oracle(case, {"SNN_EMU_SMS": "3"})


def _small(c):
    return c.B * c.geo.ns <= 20000


SMS_CASES = [c for c in ge.WINDOW_CASES if _small(c)][::3]


@pytest.mark.parametrize("sms", ["1", "7"])
@pytest.mark.parametrize("case", SMS_CASES, ids=lambda c: c.name)
def test_window_emulated_kernel_grid_sizes_bit_exact(case, sms):
    """One and seven emulated SMs: the units of the gather and learning phases land on other CTAs."""
    _emu_vs_oracle(case, {"SNN_EMU_SMS": sms})


SHUFFLED = {"conv1d": "conv1d_wdep_b3_", "conv3d": "conv3d_wdep0_b3_", "local3d": "local3d_postpre_b33_"}


@pytest.mark.parametrize("kind", list(SHUFFLED))
def test_window_emulated_kernel_shuffled_schedule_bit_exact(kind):
    case = next(c for c in ge.WINDOW_CASES if c.name.startswith(SHUFFLED[kind]))
    _emu_vs_oracle(case, {"SNN_EMU_SHUFFLE": "7", "SNN_EMU_SMS": "2"})


# ---- 2. phase-1 gathers --------------------------------------------------------------------------------------------

def _gather(case, backend, env=None):
    d = ge.draw_gather(case)
    v = _with(backend, lambda: ge.run_gather(B200, case, d), env)
    _assert_emulated_tier1(backend)
    return v, d


@pytest.mark.parametrize("case", ge.GATHER_CASES, ids=lambda c: c.name)
def test_gather_oracle_within_float64_bound(case):
    v, d = _gather(case, oracle_for(case.kind))
    v64, bound = ge.ref_gather(case, d)
    ge.assert_within_bound(v, v64, bound, case.name)
    assert (v[2:] != v[1:2]).any() or case.T < 3, f"{case.name}: the gather never changed"
    assert (v[1:] != v[:1]).any(), f"{case.name}: the gather never changed"
    ge.check_claims(case)


@pytest.mark.parametrize("case", ge.GATHER_CASES, ids=lambda c: c.name)
def test_gather_emulated_kernel_bit_exact(case):
    a, _ = _gather(case, _emu(), {"SNN_EMU_SMS": "3"})
    b, _ = _gather(case, oracle_for(case.kind))
    ge.assert_same(a, b, case.name)


# ---- 3. single operators -------------------------------------------------------------------------------------------

def check_op_against_float64(case, d, res, w_in):
    g = case.geo
    out64, obound = ge.ref_compute(g, d["s_in"], d["w"], d["b"] if g.kind != "local3d" else None)
    ge.assert_within_bound(res["out"], out64, obound, f"{case.name} compute")
    w64, bound, seen = ge.ref_op_update(case, d)
    ge.assert_within_bound(res["w_upd"], w64, bound, f"{case.name} update")
    n64, nbound = ge.ref_normalize(g, w_in, d["norm"])
    assert not torch.isfinite(n64.reshape(-1, g.K)[1]).any()
    ge.assert_within_bound(res["w_norm"], n64, nbound, f"{case.name} normalize")
    # the case bites: outputs differ across targets, weights moved, mostly inside the bounds, U and V non-zero
    assert res["out"].unique().numel() > 2, f"{case.name}: the compute is constant"
    changed = res["w_upd"].view(torch.int32) != d["w"].view(torch.int32)
    assert changed.any(), f"{case.name}: the update changed no weight"
    v = res["w_upd"][changed]
    assert ((v > d["wmin"]) & (v < d["wmax"])).float().mean() >= 0.5, f"{case.name}: the clamp decided the update"
    if case.pre_on:
        assert seen[0], f"{case.name}: U is zero"
    if case.post_on:
        assert seen[1], f"{case.name}: V is zero"


@pytest.mark.parametrize("case", ge.OP_CASES, ids=lambda c: c.name)
def test_single_operators_oracle_within_float64_bound(case):
    d = ge.draw_op(case)
    res, w_in = _with(oracle_for(case.kind), lambda: ge.run_op(B200, case, d))
    check_op_against_float64(case, d, res, w_in)


@pytest.mark.parametrize("case", ge.OP_CASES, ids=lambda c: c.name)
def test_single_operators_emulated_kernel_bit_exact(case):
    d = ge.draw_op(case)
    a, _ = _with(_emu(), lambda: ge.run_op(B200, case, d))
    b, _ = _with(oracle_for(case.kind), lambda: ge.run_op(B200, case, d))
    for k in b:
        ge.assert_same(a[k], b[k], f"{case.name} {k}")


# ---- 4. the cases reach both sides of every switch ---------------------------------------------------------------------

def test_cases_reach_both_sides_of_every_switch():
    sides = {}

    def add(kind, key, v):
        sides.setdefault((kind, key), set()).add(v)

    for c in ge.WINDOW_CASES:
        ge.check_claims(c)
        p = c.paths()
        for k, v in p.items():
            if k == "st_bits" and c.B > 32:
                continue   # above 32 samples the chunk size is the grid's business
            add(c.kind, k, v if k != "pad" else tuple(v))
        add(c.kind, "B", c.B)
        add(c.kind, "rule", c.rule)
        add(c.kind, ("red", c.rule), c.red)
        add(c.kind, ("nu_off", c.rule), c.nu_off)
        add(c.kind, "norm", c.norm)
        add(c.kind, "zero_filter", c.zero_filter)
    for c in ge.GATHER_CASES:
        ge.check_claims(c)
        for k, v in c.paths().items():
            if k == "st_bits" and c.B > 32:
                continue
            add(c.kind, k, v if k != "pad" else tuple(v))
    both = {True, False}
    for kind in ge.KINDS:
        for key in ("st_bits", "learned_first", "cross_word", "kw_over_32"):
            assert both <= sides.get((kind, key), set()), f"{kind} {key}: reached {sides.get((kind, key))}"
        assert True in sides[(kind, "off0")] and True in sides[(kind, "off31")], kind   # rows starting at bits 0 and 31
        assert {1, 31, 32, 33, 40, 65} <= sides[(kind, "kw")], (kind, sides[(kind, "kw")])
        assert True in sides[(kind, "norm")]
    for kind in ("conv1d", "conv3d"):
        assert both <= sides[(kind, "st_taps_all")], kind
        # the padding cut and a stride longer than the kernel, on every axis (a LocalConnection3D has no padding)
        for a in ("x",) if kind == "conv1d" else ("z", "y", "x"):
            assert True in sides[(kind, f"cut_{a}")] and True in sides[(kind, f"s_gt_k_{a}")], (kind, a)
    strides = {c.geo.s[0] for c in ge.WINDOW_CASES + ge.GATHER_CASES if c.kind == "conv1d" and c.geo.pad[0] >= 1}
    assert {1, 2, 5} <= strides, strides
    # each Conv3d axis padded on its own
    pads = sides[("conv3d", "pad")]
    for a in range(3):
        assert any(p[a] > 0 and sum(p) == p[a] for p in pads), a
    # the Conv3d case with K = 16^3 = 4096 straddles the tap stage: a tile inside one channel stages, one across two not
    k4096 = [c for c in ge.WINDOW_CASES if c.geo == ge.K4096]
    assert k4096 and all(c.paths()["st_taps_some_on"] and c.paths()["st_taps_some_off"] for c in k4096)
    assert {c.paths()["st_bits"] for c in k4096} == both
    # phase3_conv1d
    assert {1, 2, 3, 5, 16, 17, 31, 32, 33, 65} <= sides[("conv1d", "B")]
    assert {7, 32, 33, 70} <= sides[("conv1d", "L")]
    assert both <= sides[("conv1d", "group_tail")] and both <= sides[("conv1d", "lq_loop")]
    assert True in sides[("conv1d", "unaligned")]
    assert {"cin=1", "cin<L", "cin>L"} <= sides[("conv1d", "wrap")]
    for r in ("postpre", "wdep", "hebbian"):
        assert {"sum", "mean"} <= sides[("conv1d", ("red", r))], r
        assert {-1, 0, 1} <= sides[("conv1d", ("nu_off", r))], r
    assert "noop" in sides[("conv1d", "rule")]
    assert both <= sides[("conv1d", "multi_pass")]
    # phase3_conv3d
    assert {"noop", "postpre0", "wdep0"} <= sides[("conv3d", "rule")] and True in sides[("conv3d", "zero_filter")]
    # phase3_local3d
    assert {1, 127, 128, 129, 257} <= sides[("local3d", "Mw")]
    assert {1, 31, 32, 33, 65} <= sides[("local3d", "B")]
    assert both <= sides[("local3d", "seg_tail")] and both <= sides[("local3d", "b_tail")]
    assert {"postpre", "wdep", "hebbian", "noop"} <= sides[("local3d", "rule")]
    assert True in sides[("local3d", "multi_pass")] and True in sides[("local3d", "zero_filter")]
    # the warp-wide skips: every batch of more than one sample holds a sample whose targets never spike
    for c in ge.WINDOW_CASES:
        if c.kind == "local3d" and c.B > 1:
            d = ge.draw_window(c)
            assert not d["z_in"][:, -1].any() and d["z_in"][:, :-1].any()
    # the single operators: every kind, every rule it has
    assert {c.kind for c in ge.OP_CASES} == set(ge.KINDS)
    assert {"noop", "postpre0", "wdep0"} <= {c.rule for c in ge.OP_CASES if c.kind == "conv3d"}
    for kind in ("conv1d", "local3d"):
        assert {"postpre", "wdep", "hebbian", "noop"} <= {c.rule for c in ge.OP_CASES if c.kind == kind}
