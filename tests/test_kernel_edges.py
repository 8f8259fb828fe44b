"""The generic kernel's STDP update (phase3) and the single-operator kernels at the batch sizes and shapes where their
fast paths switch (cases and float64 references: tests/kernel_edges.py).  CPU tests: the oracle against a plain float64
restatement of the reference's formulas within a rounding-error bound (this pins the oracle at shapes the golden
fixtures never had), and the kernels' CUDA source under the CPU emulation (tests/emu) against the oracle, bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch

import cases
import kernel_edges as ke

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int32)


def _assert_bit_identical(a: torch.Tensor, b: torch.Tensor, what: str):
    if not torch.equal(_bits(a), _bits(b)):
        diff = (a.double() - b.double()).abs()
        raise AssertionError(f"{what}: {int((_bits(a) != _bits(b)).sum())} entries differ, max |d| {float(diff.nan_to_num(np.inf).max()):.3e}")


def _assert_within_bound(w, w64, bound, what):
    r = ke.ratio(w, w64, bound)
    assert r <= 1.0, f"{what}: |w - w_f64| reaches {r:.3g} x the rounding-error bound"
    return r


def _with(backend, fn, env=None):
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        with backend() as be:
            out = fn()
        assert be.err == 0
        return out
    finally:
        for k, v in old.items():
            os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)


def _oracle():
    from oracle.oracle import OracleBackend

    return OracleBackend


def _emu():
    import emu

    return emu.EmuBackend


# ---- 1. single-operator update (snn_b200_conn_update = phase3 at t = 0) ---------------------------------------------

@pytest.mark.parametrize("case", ke.UPDATE_CASES, ids=lambda c: c.name)
def test_update_oracle_within_float64_bound(case):
    d = ke.draw_update(case)
    w = _with(_oracle(), lambda: ke.run_update(B200, case, d))
    w64, bound = ke.ref_update(case, d)
    _assert_within_bound(w, w64, bound, case.name)
    ke.check_bites(case, d, w)


@pytest.mark.parametrize("case", ke.UPDATE_CASES, ids=lambda c: c.name)
def test_update_emulated_kernel_bit_exact(case):
    d = ke.draw_update(case)
    a = _with(_emu(), lambda: ke.run_update(B200, case, d))
    b = _with(_oracle(), lambda: ke.run_update(B200, case, d))
    _assert_bit_identical(a, b, case.name)
    ke.check_bites(case, d, a)


def test_update_cases_straddle_every_threshold():
    """The case list reaches both sides of every switch of phase3."""
    cs = ke.UPDATE_CASES
    Bs = {c.B for c in cs}
    assert {1, 2, 16, 17, 31, 32, 33, 63, 64, 65, 129, 768, 769, 1024} <= Bs
    assert any(c.unstaged for c in cs) and any(c.pre_on and c.B == ke.XT_STAGED_MAX_B for c in cs)
    assert any(c.overflow for c in cs) and any(c.pattern == "allcols" and c.B == ke.P3_MAXEV for c in cs)
    assert any(c.B == ke.EAGER_B - 1 for c in cs) and any(c.B == ke.EAGER_B for c in cs)
    assert {c.ns for c in cs} >= {1, 31, 32, 33, 257, 784} and {c.nt for c in cs} >= {1, 31, 32, 33, 95}
    for attr, vals in (("rule", ke.RULES), ("pattern", ke.PATTERNS), ("red", ("sum", "mean", "squeeze"))):
        assert {getattr(c, attr) for c in cs} == set(vals), attr
    assert any(c.recurrent for c in cs) and any(c.bounds == "inf" for c in cs) and any(c.decay for c in cs)
    assert any(c.nu_off == 0 for c in cs) and any(c.nu_off == 1 for c in cs)


# ---- 2. window: phase3 at t > 0 (untouched-row skip, row chunks across CTAs) ----------------------------------------

def _run_window(case, d, backend, env=None):
    def go():
        net, inputs = ke.build_window(B200, case, d)
        net.force_tier = 1
        net.run(inputs=inputs, time=case.T)
        return net
    net = _with(backend, go, env)
    if backend is _emu():
        import emu

        assert emu.last_tier == 1
    return ke.window_state(net), float(net.layers["X"].trace_decay)


def _check_window(case, d, st, trace_decay):
    w64, bound, raster = ke.ref_window(case, d, trace_decay)
    assert torch.equal(st["Ys"], raster.reshape(case.T, -1)), f"{case.name}: Y's raster is not Z's, one step later"
    assert st["Ys"].any()
    r = _assert_within_bound(st["w"], w64, bound, case.name)
    changed = _bits(st["w"]) != _bits(d["w"])
    assert changed.any(), f"{case.name}: no weight changed"
    if case.bounds == "finite":
        v = st["w"][changed]
        assert ((v > d["wmin"]) & (v < d["wmax"])).float().mean() >= 0.5, f"{case.name}: the clamp decided the result"
    return r


@pytest.mark.parametrize("case", ke.WINDOW_CASES, ids=lambda c: c.name)
def test_window_oracle_within_float64_bound(case):
    d = ke.draw_window(case)
    st, dec = _run_window(case, d, _oracle())
    _check_window(case, d, st, dec)


WINDOW_ENVS = {"sms1": {"SNN_EMU_SMS": "1"}, "sms3": {"SNN_EMU_SMS": "3"}, "sms7": {"SNN_EMU_SMS": "7"}}


@pytest.mark.parametrize("env", list(WINDOW_ENVS))
@pytest.mark.parametrize("case", ke.WINDOW_CASES, ids=lambda c: c.name)
def test_window_emulated_kernel_bit_exact(case, env):
    d = ke.draw_window(case)
    a, _ = _run_window(case, d, _emu(), WINDOW_ENVS[env])
    b, _ = _run_window(case, d, _oracle())
    for k in a:
        _assert_bit_identical(a[k].float(), b[k].float(), f"{case.name} {env} {k}")


def test_window_emulated_kernel_shuffled_schedule_bit_exact():
    case = ke.WINDOW_CASES[1]
    d = ke.draw_window(case)
    a, _ = _run_window(case, d, _emu(), {"SNN_EMU_SHUFFLE": "5", "SNN_EMU_SMS": "2"})
    b, _ = _run_window(case, d, _oracle())
    for k in a:
        _assert_bit_identical(a[k].float(), b[k].float(), f"{case.name} shuffled {k}")


# ---- 3. single operators at their edges -----------------------------------------------------------------------------

def _compute(backend, n_src, B, bias):
    conn, s = ke.compute_setup(B200, n_src, 95, B, bias)
    return _with(backend, lambda: conn.compute(s)), conn, s


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("n_src", [1, 33, 257])
@pytest.mark.parametrize("B", [1, 513, 1100])
def test_compute_batch_rows_past_the_grid(B, n_src, bias):
    """conn_compute_kernel's grid has at most 64 x 8 batch rows; B = 513 and 1100 need the grid-stride loop."""
    a, conn, s = _compute(_emu(), n_src, B, bias)
    b, _, _ = _compute(_oracle(), n_src, B, bias)
    _assert_bit_identical(a, b, f"compute B={B} n_src={n_src}")
    out64, bound = ke.ref_compute(conn, s)
    _assert_within_bound(b, out64, bound, f"compute B={B} n_src={n_src}")


def _normalize(backend, n_src, mcc):
    conn = ke.normalize_setup(B200, n_src, mcc=mcc)
    w0 = conn.w.detach().clone()
    ke.poison_weights(conn)
    _with(backend, conn.normalize)
    return w0, conn.w.detach().clone()


@pytest.mark.parametrize("mcc", [False, True], ids=["connection_abs", "mcc_feature_plain"])
@pytest.mark.parametrize("n_src", [1, 5, 15, 16, 17, 33])
def test_normalize_row_chunks_and_zero_column(n_src, mcc):
    """normalize_tile sums each column in 16 row chunks: for n_src < 16 some are empty, for n_src = 17 the last one is
    short.  Column 3 is all zero (the tot == 0 -> 1 guard); Connection.normalize sums absolute values of weights of
    both signs."""
    w0, a = _normalize(_emu(), n_src, mcc)
    _, b = _normalize(_oracle(), n_src, mcc)
    _assert_bit_identical(a, b, f"normalize n_src={n_src}")
    ref, bound = ke.ref_normalize(w0, 7.5 if mcc else 11.0, absolute=not mcc)
    _assert_within_bound(a, ref, bound, f"normalize n_src={n_src}")
    assert (a[:, 3] == 0).all() and torch.isfinite(a).all()
    assert (w0 < 0).any() or mcc


def _conv(backend, geo):
    conn, s = ke.conv_setup(B200, geo)
    w0 = conn.w.detach().clone()

    def go():
        out = conn.compute(s)
        conn.normalize()
        return out
    out = _with(backend, go)
    return out, w0, conn.w.detach().clone(), conn, s


@pytest.mark.parametrize("geo", ke.CONV_GEOMETRIES, ids=lambda g: "k{}x{}_s{}x{}_p{}x{}_d{}x{}".format(*g[4], *g[5], *g[6], *g[7]))
def test_conv2d_compute_and_normalize(geo):
    oa, _, wa, conn, s = _conv(_emu(), geo)
    ob, w0, wb, _, _ = _conv(_oracle(), geo)
    _assert_bit_identical(oa, ob, "conv compute")
    _assert_bit_identical(wa, wb, "conv normalize")
    out64, bound = ke.ref_conv_compute(conn, s, w0)
    assert out64.shape == oa.shape
    _assert_within_bound(oa, out64, bound, "conv compute")
    w64, wbound = ke.ref_conv_normalize(w0, 3.0)
    _assert_within_bound(wa, w64, wbound, "conv normalize")
