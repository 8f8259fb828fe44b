"""The generic kernel's per-synapse tensor (SYN) and per-neuron parameter (PN) instantiations at the shapes where their
paths switch (cases, float64 restatements and path mirrors: tests/param_edges.py).  CPU tests: the oracle
(tests/neuron_param_oracle.c, which includes the synapse-tensor oracle) against a plain float64 restatement of the
reference's formulas within a rounding-error bound, and the kernels' CUDA source under the CPU emulation (tests/emu)
against the oracle, bit for bit, on the whole state."""
import os
import sys

import pytest
import torch

import cases
import geometry_edges as ge
import param_edges as pe
from test_kernel_edges import _emu, _with

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


def _oracle():
    from neuron_param_oracle import NeuronParamOracleBackend

    return NeuronParamOracleBackend


def _tier1(backend):
    if backend is _emu():
        import emu

        assert emu.last_tier == 1


def assert_same_state(a: dict, b: dict, what: str):
    assert set(a) == set(b), (what, sorted(set(a) ^ set(b)))
    for k in b:
        ge.assert_same(a[k], b[k], f"{what} {k}")


# ---- checks shared with the GPU file ---------------------------------------------------------------------------------

def run_syn(case, d, backend, env=None):
    st, net = _with(backend, lambda: pe.run_syn(B200, case, d), env)
    if not case.op:
        _tier1(backend)
    return st, net


def syn_desc(case, d):
    """The plan entry the host builds for the learned connection (the forms it chose)."""
    from bindsnet_b200.network import _plan

    net, _ = pe.build_syn(B200, case, d)
    conn = net.connections[("X", "Y")]
    for l in net.layers.values():
        l.compute_decays(1.0)
        l.set_batch_size(case.B)
    from bindsnet_b200 import _abi

    desc = _abi.SnnConn()
    _plan.fill_conn(desc, conn, 0, 1, 1.0, case.B, rule_kwargs={"reward": case.reward})
    return desc


def check_syn_against_float64(case, d, st, net):
    """Y's raster is Z's one step later; the weights within the float64 bound; the <SYN, PN> population's voltages too;
    the case bites."""
    if case.op:
        w64, bound, raster = pe.ref_syn(case, d)
    else:
        td, pd, ed = pe.rule_decays(net)
        w64, bound, raster = pe.ref_syn(case, d, td, pd, ed)
        ys = st["M/Ys/s"].reshape(case.T, case.B, case.nt).bool()
        assert torch.equal(ys, raster), f"{case.name}: Y's raster is not Z's, one step later"
    w = st["C/XY/w"]
    ge.assert_within_bound(w, w64, bound, case.name)
    check_syn_bites(case, d, w)
    if case.pn:
        check_pn_against_float64(d["pn"]["case"], d["pn"], [st], net.layers["P"])


def check_syn_bites(case, d, w):
    """Weights changed, at least half of the changed ones strictly inside their per-element bounds."""
    changed = w.contiguous().view(torch.int32) != d["w"].contiguous().view(torch.int32)
    assert changed.any(), f"{case.name}: no weight changed"
    lo, hi = pe.bcast(d["wmin"], case.ns, case.nt), pe.bcast(d["wmax"], case.ns, case.nt)
    v = w.double()[changed]
    inside = ((v > lo[changed]) & (v < hi[changed])).double().mean().item()
    assert inside >= 0.5, f"{case.name}: only {inside:.2f} of the changed weights are inside their bounds"


def check_pn_against_float64(case, d, outs, P):
    pe.check_decay_factors(P)
    ref = pe.ref_pn(case, d, outs, P)
    assert ref["margin_ok"], f"{case.name}: a float64 voltage lies within its bound of the threshold ({ref['min_margin']:.3g})"
    assert ref["raster_ok"], f"{case.name}: the float64 raster differs from the oracle's"
    spikes = 0
    for k, o in enumerate(outs):
        v = o["M/Pm/v"].reshape(case.T, case.B, case.n)
        ge.assert_within_bound(v, ref["v"][k], ref["v_err"][k], f"{case.name} window {k} v")
        ge.assert_within_bound(o["L/P/x"], ref["x"][k], ref["x_err"][k], f"{case.name} window {k} x")
        assert torch.equal(o["L/P/refrac_count"].double(), ref["rc"][k]), f"{case.name} window {k}: refractory counts"
        if case.theta:
            ge.assert_within_bound(o["L/P/theta"].reshape(-1), ref["theta"][k], ref["theta_err"][k], f"{case.name} window {k} theta")
        spikes += int(o["M/Pm/s"].sum())
    assert spikes > 0, f"{case.name}: P never spiked"
    if case.theta and case.learning:
        assert (outs[-1]["L/P/theta"] != 0).any(), f"{case.name}: theta never moved"
    if case.lbound:
        assert any((o["M/Pm/v"] == -70.0).any() for o in outs), f"{case.name}: the lower bound never held a voltage"


def run_pn(case, d, backend, env=None):
    outs, net = _with(backend, lambda: pe.run_pn(B200, case, d), env)
    _tier1(backend)
    return outs, net


# ---- 1. per-synapse tensors --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", pe.SYN_CASES, ids=lambda c: c.name)
def test_syn_oracle_within_float64_bound(case):
    d = pe.draw_syn(case)
    st, net = run_syn(case, d, _oracle())
    check_syn_against_float64(case, d, st, net)
    pe.check_claims(case, pe.syn_paths(case, d))


def _syn_emu_vs_oracle(case, env):
    d = pe.draw_syn(case)
    a, _ = run_syn(case, d, _emu(), env)
    b, _ = run_syn(case, d, _oracle())
    assert_same_state(a, b, f"{case.name} {env}")


@pytest.mark.parametrize("case", pe.SYN_CASES, ids=lambda c: c.name)
def test_syn_emulated_kernel_bit_exact(case):
    _syn_emu_vs_oracle(case, {"SNN_EMU_SMS": "3"})


def _small(c):
    return c.B * c.ns <= 4000


SYN_SMS_CASES = [c for c in pe.SYN_CASES if _small(c)][::3]


@pytest.mark.parametrize("sms", ["1", "7"])
@pytest.mark.parametrize("case", SYN_SMS_CASES, ids=lambda c: c.name)
def test_syn_emulated_kernel_grid_sizes_bit_exact(case, sms):
    _syn_emu_vs_oracle(case, {"SNN_EMU_SMS": sms})


SHUFFLED = {"phase3": lambda c: c.rule == "wdep" and not c.op and c.outside,
            "mstdp_dense": lambda c: c.rule == "mstdp" and not c.op and c.outside,
            "syn_and_pn": lambda c: c.pn and c.stdp}


@pytest.mark.parametrize("inst", list(SHUFFLED))
def test_syn_emulated_kernel_shuffled_schedule_bit_exact(inst):
    """One shuffled schedule per instantiation with per-synapse tensors (<SYN> and <SYN, PN>)."""
    case = next(c for c in pe.SYN_CASES if SHUFFLED[inst](c))
    _syn_emu_vs_oracle(case, {"SNN_EMU_SHUFFLE": "7", "SNN_EMU_SMS": "2"})


# ---- 2. per-neuron parameters ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", pe.PN_CASES, ids=lambda c: c.name)
def test_pn_oracle_within_float64_bound(case):
    d = pe.draw_pn(case)
    outs, net = run_pn(case, d, _oracle())
    check_pn_against_float64(case, d, outs, net.layers["P"])
    paths = pe.pn_paths(case, net)
    pe.check_claims(case, paths)
    assert paths["mask_rows"] == tuple(r for r in pe.PN_ROWS if paths[f"row_{r}"]), (case.name, paths["mask_rows"])


def _pn_emu_vs_oracle(case, env):
    d = pe.draw_pn(case)
    a, _ = run_pn(case, d, _emu(), env)
    b, _ = run_pn(case, d, _oracle())
    for k in range(case.windows):
        assert_same_state(a[k], b[k], f"{case.name} {env} window {k}")


@pytest.mark.parametrize("case", pe.PN_CASES, ids=lambda c: c.name)
def test_pn_emulated_kernel_bit_exact(case):
    _pn_emu_vs_oracle(case, {"SNN_EMU_SMS": "3"})


PN_SMS_CASES = [c for c in pe.PN_CASES if c.B <= 32][::3]


@pytest.mark.parametrize("sms", ["1", "7"])
@pytest.mark.parametrize("case", PN_SMS_CASES, ids=lambda c: c.name)
def test_pn_emulated_kernel_grid_sizes_bit_exact(case, sms):
    _pn_emu_vs_oracle(case, {"SNN_EMU_SMS": sms})


def test_pn_emulated_kernel_shuffled_schedule_bit_exact():
    case = next(c for c in pe.PN_CASES if c.kind == "dc" and c.one_step)
    _pn_emu_vs_oracle(case, {"SNN_EMU_SHUFFLE": "7", "SNN_EMU_SMS": "2"})


# ---- 3. the cases reach both sides of every switch ---------------------------------------------------------------------

def test_cases_reach_both_sides_of_every_switch():
    sides = {}

    def add(key, v):
        sides.setdefault(key, set()).add(v)

    for c in pe.SYN_CASES:
        d = pe.draw_syn(c)
        p = pe.syn_paths(c, d, syn_desc(c, d))
        pe.check_claims(c, p)
        kind = "op" if c.op else ("mstdp" if c.rule.startswith("mstdp") else "phase3")
        for k, v in p.items():
            add((kind, k), v)
            if kind != "mstdp":
                add(("stdp", k), v)
            if k.startswith("form_"):
                add((c.rule, k), v)
        add((kind, "rule"), c.rule)
        add((c.rule, "red"), c.red)
        add((c.rule, "inf"), c.inf)
        add((c.rule, "outside"), c.outside)
        add((kind, "max_events"), p["max_events"])
    both = {True, False}
    for kind in ("phase3", "op"):
        for key in ("staged", "eager", "overflow", "nt_tail", "full_decay", "outside", "copied", "collapsed", "pre_on", "post_on",
                    "row_chunks" if kind == "phase3" else "warp_loops"):
            assert both <= sides[(kind, key)], (kind, key, sides[(kind, key)])
        assert {16, 17} <= sides[(kind, "max_events")], (kind, sides[(kind, "max_events")])
    assert both <= sides[("phase3", "row_skip")] and both <= sides[("phase3", "full_clamp0")]
    assert True in sides[("phase3", "group_skip")]
    assert both <= sides[("mstdp", "mstdp_staged")] and both <= sides[("mstdp", "full_decay")]
    # every tensor form each rule allows, for each tensor (PostPre's rates: per target or one element only)
    for rule in ("wdep", "hebbian", "mstdp"):
        for f in ("wmin", "wmax"):
            assert {"FULL", "TGT", "SRC"} <= sides[(rule, f"form_{f}")], (rule, f, sides[(rule, f"form_{f}")])
        for f in ("nu0", "nu1"):
            assert {"FULL", "TGT", "SRC", "ONE"} <= sides[(rule, f"form_{f}")], (rule, f, sides[(rule, f"form_{f}")])
    for f in ("wmin", "wmax"):
        assert {"FULL", "TGT", "SRC"} <= sides[("postpre", f"form_{f}")], (f, sides[("postpre", f"form_{f}")])
    assert "scalar" in sides[("postpre", "form_wmax")]   # a scalar bound beside a tensor one
    # a one-element bound tensor is a scalar to the host (topology.py Connection._fill_desc reads it into wmin / wmax):
    # the kernels never see SNN_SYN_ONE for a bound
    for c in pe.SYN_CASES:
        if "one" in (c.lo, c.hi):
            d = pe.draw_syn(c)
            desc = syn_desc(c, d)
            for f, form in (("wmin", c.lo), ("wmax", c.hi)):
                if form == "one":
                    assert not getattr(desc, f + "_t") and getattr(desc, f) == float(d[f].reshape(())), (c.name, f)
    assert {c.rule for c in pe.SYN_CASES if "one" in (c.lo, c.hi)} >= {"postpre", "wdep"}
    assert {"TGT", "ONE"} == sides[("postpre", "form_nu0")] - {"scalar"}
    for rule in ("postpre", "hebbian", "mstdp", "mstdpet"):
        assert True in sides[(rule, "inf")], rule
    for rule in pe.SYN_RULES:
        assert True in sides[(rule, "outside")], rule
    assert {"sum", "mean"} <= sides[("mstdp", "red")]
    assert any(c.rule == "mstdp" and c.reward < 0 for c in pe.SYN_CASES)
    assert any(c.rule == "mstdpet" and c.reward < 0 for c in pe.SYN_CASES)
    assert any(c.pn and c.stdp for c in pe.SYN_CASES) and any(c.pn and not c.stdp for c in pe.SYN_CASES)
    # per-neuron parameters
    pn = {}
    for c in pe.PN_CASES:
        for k, v in pe.pn_paths(c).items():
            pn.setdefault(k, set()).add(v)
        pe.check_claims(c, pe.pn_paths(c))
    for r in pe.PN_ROWS:
        assert any(c.rows == (r,) for c in pe.PN_CASES), r
        assert True in pn[f"row_{r}"], r
    assert any(set(c.rows) == set(pe.PN_ROWS) for c in pe.PN_CASES)
    for key in ("n_tail", "chunks", "one_step", "one_spike", "theta_learning", "T1", "per_channel"):
        assert both <= pn[key], (key, pn[key])
    assert {1, 2, 3} <= pn["windows"]
    assert True in pn["lbound"]


# ---- 4. the host's per-tensor caches follow in-place changes -----------------------------------------------------------

def _two_windows(case, d, mutate, backend):
    def go():
        net, inputs = pe.build_syn(B200, case, d)
        net.force_tier = 1
        kw = dict(reward=case.reward) if case.rule.startswith("mstdp") else {}
        net.run(inputs=inputs, time=case.T, **kw)
        w1 = net.connections[("X", "Y")].w.detach().clone()
        mutate(net.connections[("X", "Y")])
        net.run(inputs=inputs, time=case.T, **kw)
        return w1, pe.snapshot(net), net
    return _with(backend, go)


MUTATIONS = {
    # has_clamp is cached per bound tensor: all-infinite bounds, then a finite upper bound written in place
    "clamp_turns_on": (pe.SynCase("postpre", 4, 40, 33, lo="full", hi="full", nu="tgt"),
                       lambda d: (d.__setitem__("wmin", torch.full_like(d["wmin"], -float("inf"))),
                                  d.__setitem__("wmax", torch.full_like(d["wmax"], float("inf")))),
                       lambda c: c.wmax.fill_(0.05)),
    # a per-element bound changed in place (a FULL tensor read in place)
    "bound_values": (pe.SynCase("wdep", 4, 40, 33, lo="full", hi="full", nu="full"), None,
                     lambda c: c.wmax.mul_(0.5)),
    # the FULL copy of a transposed bound is cached per version of the tensor
    "transposed_copy": (pe.SynCase("hebbian", 4, 40, 33, lo="tfull", hi="tfull", nu="src"), None,
                        lambda c: c.wmax.sub_(0.6)),
    # the rate gate nu[0].any(), cached per version of the rate tensor: nu[0] zeroed in place
    "rate_gate_off": (pe.SynCase("postpre", 4, 40, 33, lo="tgt", hi="tgt", nu="tgt"), None,
                      lambda c: c.update_rule.nu[0].zero_()),
}


@pytest.mark.parametrize("name", list(MUTATIONS))
def test_host_caches_follow_in_place_changes(name):
    """The reference re-reads its bounds and rates every step; the host caches has_clamp, the rate gates and FULL copies
    per tensor version.  The second window must follow the new values: against the oracle bit for bit (emulated
    kernel), and against float64 run from the first window's weights with the mutated tensors (oracle)."""
    from dataclasses import replace

    case, prep, mutate = MUTATIONS[name]
    d = pe.draw_syn(case)
    if prep is not None:
        prep(d)
    w1, a, _ = _two_windows(case, d, mutate, _emu())
    w1o, b, onet = _two_windows(case, d, mutate, _oracle())
    assert torch.equal(w1, w1o)
    assert_same_state(a, b, name)
    # float64: the second window from w1 with the mutated bounds / rates (the traces restart from the first window's:
    # the float64 replay runs both windows back to back as one of 2T steps with the tensors switched at T)
    c = onet.connections[("X", "Y")]
    d2 = dict(d)
    d2["wmin"] = c.wmin.detach().clone() if isinstance(c.wmin, torch.Tensor) and c.wmin.numel() > 1 else float(c.wmin)
    d2["wmax"] = c.wmax.detach().clone() if isinstance(c.wmax, torch.Tensor) and c.wmax.numel() > 1 else float(c.wmax)
    nu = c.update_rule.nu
    d2["nu"] = (nu[0].clone(), nu[1].clone())
    case2 = replace(case, lo="full" if case.lo == "tfull" else case.lo, hi="full" if case.hi == "tfull" else case.hi)
    w64, bound = pe.ref_syn_two(case, d, case2, d2, float(onet.layers["X"].trace_decay))
    ge.assert_within_bound(b["C/XY/w"], w64, bound, name)
    assert not torch.equal(b["C/XY/w"], w1), f"{name}: the second window changed nothing"
