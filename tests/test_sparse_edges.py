"""The generic kernel's sparse instantiation and the sparse single operators at the shapes where their paths switch
(cases, float64 restatements and path mirrors: tests/sparse_edges.py).  CPU tests: the oracle (tests/sparse_oracle.c)
against a plain float64 restatement of the reference's formulas within a rounding-error bound, the kernels' CUDA source
under the CPU emulation (tests/emu) against the oracle, bit for bit, on the whole state, the pattern checks of
sparse_prepass, and the bias of dense and sparse connections in every form the reference broadcasts."""
import os
import sys

import pytest
import torch

import cases
import geometry_edges as ge
import sparse_edges as se
from test_kernel_edges import _emu, _with

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

B200 = cases.namespace("b200")


def _oracle():
    from sparse_oracle import SparseOracleBackend

    return SparseOracleBackend


def assert_same_state(a: dict, b: dict, what: str):
    assert set(a) == set(b), (what, sorted(set(a) ^ set(b)))
    for k in b:
        if k.endswith("/idx"):
            assert torch.equal(a[k], b[k]), f"{what} {k}"
        else:
            ge.assert_same(a[k], b[k], f"{what} {k}")


# ---- checks shared with the GPU file ---------------------------------------------------------------------------------

def run_case(case, d, backend, env=None):
    outs, net = _with(backend, lambda: se.run(B200, case, d), env)
    if backend is _emu():
        import emu

        assert emu.last_tier == 1
    return outs, net


def check_against_float64(case, d, outs):
    """Every target's raster and voltages (each step), its refractory counts and currents, and the stored values after
    the last decay, within the float64 bound."""
    ref = se.ref_window(case, d, outs)
    steps = case.T * case.windows
    for tgt, r in ref.items():
        what = f"{case.name} {tgt}"
        assert r["raster_ok"], f"{what}: the float64 raster differs from the oracle's"
        assert r["margin_ok"], f"{what}: a float64 voltage lies within its bound of the threshold ({r['min_margin']:.3g})"
        n = r["v"].shape[2]
        v = torch.cat([o[f"M/{tgt}m/v"] for o in outs]).reshape(steps, case.B, n)
        ge.assert_within_bound(v, r["v"], r["v_err"], f"{what} v")
        assert torch.equal(outs[-1][f"L/{tgt}/refrac_count"].double(), r["rc"]), f"{what}: refractory counts"
        if tgt == "Y" and case.kind == "clif":
            ge.assert_within_bound(outs[-1]["L/Y/i"], r["i"], r["i_err"], f"{what} i")
    for key, w in (("XY", d["w"]), ("XY2", d.get("w2")), ("YY", d.get("wr"))):
        if f"C/{key}/val" in outs[-1]:
            v64, bound = se.ref_values(case.wd, w, steps)
            assert torch.equal(outs[-1][f"C/{key}/idx"], w.coalesce().indices()), f"{case.name} {key}: the pattern changed"
            ge.assert_within_bound(outs[-1][f"C/{key}/val"], v64, bound, f"{case.name} {key} values")


# ---- 1. windows -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", se.CASES, ids=lambda c: c.name)
def test_oracle_within_float64_bound(case):
    d = se.draw(case)
    outs, _ = run_case(case, d, _oracle())
    check_against_float64(case, d, outs)
    check_bites(case, d, outs)


def check_bites(case, d, outs):
    """Every target spikes somewhere and stays silent somewhere; the decaying cases change the stored values, the others
    leave them alone."""
    s = torch.cat([o["M/Ym/s"] for o in outs])
    assert 0 < s.sum() < s.numel(), f"{case.name}: Y spiked {int(s.sum())} times"
    if case.two:
        assert torch.cat([o["M/Y2m/s"] for o in outs]).sum() > 0, f"{case.name}: Y2 never spiked"
    # (after the first window: every case with a factor of -1 runs an odd number of steps in it)
    val, v0 = outs[0]["C/XY/val"], d["w"].coalesce().values()
    decays = se.decay_factor(case.wd) != 1.0 and v0.numel() > 0
    assert bool((val.view(torch.int32) != v0.view(torch.int32)).any()) == decays, f"{case.name}: decay {case.wd}"


def _emu_vs_oracle(case, env):
    d = se.draw(case)
    a, _ = run_case(case, d, _emu(), env)
    b, _ = run_case(case, d, _oracle())
    for k in range(case.windows):
        assert_same_state(a[k], b[k], f"{case.name} {env} window {k}")


@pytest.mark.parametrize("case", se.CASES, ids=lambda c: c.name)
def test_emulated_kernel_bit_exact(case):
    _emu_vs_oracle(case, {"SNN_EMU_SMS": "3"})


SMS_CASES = [c for c in se.CASES if c.B * c.nt <= 20_000][::2]


@pytest.mark.parametrize("sms", ["1", "7"])
@pytest.mark.parametrize("case", SMS_CASES, ids=lambda c: c.name)
def test_emulated_kernel_grid_sizes_bit_exact(case, sms):
    """One and seven emulated SMs: the gather units land on other CTAs, the decay's grid-stride loop wraps differently."""
    _emu_vs_oracle(case, {"SNN_EMU_SMS": sms})


def test_emulated_kernel_shuffled_schedule_bit_exact():
    case = next(c for c in se.CASES if c.rows and c.dense)
    _emu_vs_oracle(case, {"SNN_EMU_SHUFFLE": "5", "SNN_EMU_SMS": "2"})


# ---- 2. the single operators ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", se.OP_CASES, ids=lambda c: c.name)
def test_op_emulated_and_oracle_within_float64_bound(case):
    """connection.compute (sparse_compute_kernel) and connection.update (NoOp's decay): the emulated kernels equal the
    oracle bit for bit, both within the float64 bound."""
    d = se.draw_op(case)
    a = _with(_emu(), lambda: se.run_op(B200, case, d))
    b = _with(_oracle(), lambda: se.run_op(B200, case, d))
    for k in b:
        ge.assert_same(a[k], b[k], f"{case.name} {k}")
    check_op_against_float64(case, d, b)
    se.check_claims(case, se.op_paths(case, d))


def check_op_against_float64(case, d, st):
    out, bound, v, vb = se.ref_op(case, d)
    ge.assert_within_bound(st["out"], out, bound, f"{case.name} out")
    ge.assert_within_bound(st["val"], v, vb, f"{case.name} values")


# ---- 3. the cases reach both sides of every switch ---------------------------------------------------------------------

def test_cases_reach_both_sides_of_every_switch():
    sides = {}
    for c in se.CASES:
        d = se.draw(c)
        p = se.paths(c, d)
        se.check_claims(c, p)
        for k, v in p.items():
            if isinstance(v, set):
                sides.setdefault(k, set()).update(v)
            else:
                sides.setdefault(k, set()).add(v)
    both = {True, False}
    assert {1024, 512, 256, 128} <= sides["bw"], sides["bw"]
    assert {"units", "cap", "floor"} <= sides["stop"], sides["stop"]
    for key in ("partial", "two_widths", "words_gt32", "nnz0", "anyf_skip", "step0_slot2", "cur", "prev_one_step", "nb_gt1"):
        assert both <= sides[key], (key, sides[key])
    for key in ("late_row", "col0", "col_edge", "col_edge_wide", "col_last", "empty_row", "empty_col", "all_group"):
        assert True in sides[key], (key, sides[key])
    assert {0, 1, 7} <= sides["b_tail"], sides["b_tail"]
    assert {0, 1, 8, 9, 32, 33} <= sides["counts"], sorted(sides["counts"])
    assert {0, 1, 32, 33} <= sides["entries"] and max(sides["entries"]) > 64, sorted(sides["entries"])
    assert {1, 2} <= sides["windows"]
    assert {1, 31, 32, 33, 1024, 1025} <= {c.ns for c in se.CASES} and max(c.ns for c in se.CASES) > 2048
    assert {0.0, 0.1, 1.0, 2.0} <= {c.wd for c in se.CASES}
    assert {"lif", "iff", "clif"} <= {c.kind for c in se.CASES}
    assert {"zeros", "inf"} <= {c.values for c in se.CASES}
    assert {"sync", "before", "after", "rec"} <= {c.order for c in se.CASES}
    op = {}
    for c in se.OP_CASES:
        for k, v in se.op_paths(c, se.draw_op(c)).items():
            op.setdefault(k, set()).add(v)
    for key in ("nt_tail", "grid_y_wraps", "update_blocks_capped"):
        assert both <= op[key], (key, op[key])
    assert {1, 8, 513} <= {c.B for c in se.OP_CASES}
    assert {0.0, 0.1, 1.0, 2.0} <= {c.wd for c in se.OP_CASES}


# ---- 4. sparse_prepass refuses a malformed pattern ---------------------------------------------------------------------

BAD_PATTERNS = ("rowptr_not_monotone", "column_out_of_range", "columns_out_of_order")


@pytest.mark.parametrize("bad", BAD_PATTERNS)
def test_emulated_prepass_refuses_a_malformed_pattern(bad, monkeypatch):
    """A hand-filled CSR (the host never builds one like it): the pre-pass raises SNN_ERR_BAD_ARG and enters the bad row
    as empty, so the window runs with the other rows only.  Emulation only: on the GPU this input is a malformed plan."""
    from bindsnet_b200 import _abi
    from bindsnet_b200.network import _plan

    ns, nt, B, T = 6, 40, 2, 3
    rows = [[1, 5], [0, 39], [2, 3, 30], [4], [7, 9], [10]]
    rowptr = [0]
    col = []
    for r in rows:
        col += r
        rowptr.append(len(col))
    bad_row = ns - 1 if bad == "rowptr_not_monotone" else 2   # (the last row: no other row shares the bad pointer)
    rowptr_t, col_t = torch.tensor(rowptr, dtype=torch.int32), torch.tensor(col, dtype=torch.int32)
    if bad == "rowptr_not_monotone":
        rowptr_t[bad_row + 1] = rowptr_t[bad_row] - 1
    elif bad == "column_out_of_range":
        col_t[rowptr[bad_row] + 2] = nt
    else:
        col_t[rowptr[bad_row]], col_t[rowptr[bad_row] + 1] = 3, 2
    vals = torch.arange(1, len(col) + 1, dtype=torch.float32)
    good = [k for k in range(ns) if k != bad_row]
    fill = _plan.fill_sparse

    def fill_bad(d, conn):
        fill(d, conn)
        d.sp_rowptr, d.sp_col, d.nnz = rowptr_t.data_ptr(), col_t.data_ptr(), len(col)
        d.w = vals.data_ptr()

    def build():
        net = B200.Network(dt=1.0, batch_size=B)
        X, Y = B200.nodes.Input(ns), B200.nodes.IFNodes(nt, thresh=1e6)
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        w = torch.sparse_coo_tensor(torch.tensor([[i for i in range(ns) for _ in rows[i]], col]), vals, (ns, nt)).coalesce()
        net.add_connection(B200.topology.SparseConnection(X, Y, w=w), "X", "Y")
        net.force_tier = 1
        return net

    x = torch.ones(T, B, ns, dtype=torch.uint8)
    import emu

    monkeypatch.setattr(_plan, "fill_sparse", fill_bad)
    net = build()
    with emu.EmuBackend() as be:
        net.run(inputs={"X": x}, time=T)
    assert be.err & _abi.SNN_ERR_BAD_ARG, f"{bad}: no SNN_ERR_BAD_ARG ({be.err})"
    # the other rows' entries, each gathered T - 1 times (the first step reads s(-1) = 0)
    want = torch.zeros(nt, dtype=torch.float64)
    for i in good:
        for p in range(rowptr[i], rowptr[i + 1]):
            want[col[p]] += float(vals[p])
    v = net.layers["Y"].v.double()
    assert torch.equal(v, (-65.0 + (T - 1) * want).expand(B, nt)), f"{bad}: the bad row was gathered"


# ---- 5. the bias of dense and sparse connections -----------------------------------------------------------------------

N_B = 48


def _bias_net(sparse: bool, b, B=2, g_seed=0):
    g = torch.Generator().manual_seed(g_seed)
    w = (torch.rand(64, N_B, generator=g) < 0.2) * (torch.rand(64, N_B, generator=g) - 0.3)
    net = B200.Network(dt=1.0, batch_size=B)
    X, Y = B200.nodes.Input(64), B200.nodes.IFNodes(N_B, thresh=1e9)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    C = B200.topology.SparseConnection if sparse else B200.topology.Connection
    net.add_connection(C(X, Y, w=w.to_sparse() if sparse else w, b=b), "X", "Y")
    net.force_tier = 1
    x = (torch.rand(5, B, 64, generator=g) < 0.3).to(torch.uint8)
    return net, x


def _biases():
    g = torch.Generator().manual_seed(4)
    base = torch.rand(N_B, 3, generator=g)
    return {
        "strided": (base[:, 1], base[:, 1].contiguous()),
        "0d": (torch.tensor(0.375), torch.full((N_B,), 0.375)),
        "one": (torch.tensor([-0.25]), torch.full((N_B,), -0.25)),
        "row": (base[:, 2].contiguous().view(1, N_B), base[:, 2].contiguous()),
        "expanded": (torch.tensor(0.5).expand(N_B), torch.full((N_B,), 0.5)),
    }


BACKENDS = {"emu": _emu, "oracle": _oracle}


@pytest.mark.parametrize("backend", list(BACKENDS))
@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
@pytest.mark.parametrize("form", list(_biases()))
def test_bias_forms_equal_the_explicit_bias(form, sparse, backend):
    """A bias that broadcasts to the target (topology.py:342-345 adds it to the [B, n] product) gives the bits of the
    explicit [n] bias, in the window and in connection.compute."""
    b, full = _biases()[form]
    outs = []
    for bias in (b, full):
        net, x = _bias_net(sparse, bias)
        conn = net.connections[("X", "Y")]
        with BACKENDS[backend]()() as be:
            net.run(inputs={"X": x}, time=5)
            out = conn.compute(x[0].bool())
        assert be.err == 0
        outs.append((net.layers["Y"].v.clone(), out.clone()))
    for a, e in zip(*outs):
        assert torch.equal(a.view(torch.int32), e.view(torch.int32)), form
    # and the float64 reference of compute
    w = net.connections[("X", "Y")].w
    w = w.to_dense() if w.is_sparse else w
    ref = x[0].double() @ w.double() + full.double()
    torch.testing.assert_close(outs[0][1].double(), ref, rtol=1e-6, atol=1e-5)


def test_contiguous_bias_is_read_in_place():
    """A contiguous [n] bias is passed as is: an in-place edit between runs takes effect (no stale copy), as does one of
    a strided bias (its copy follows the bias' version)."""
    import emu

    for strided in (False, True):
        base = torch.rand(N_B, 2, generator=torch.Generator().manual_seed(5))
        outs = []
        for edit in (False, True):
            net, x = _bias_net(True, base[:, 0] if strided else base[:, 0].contiguous())
            conn = net.connections[("X", "Y")]
            with emu.EmuBackend():
                net.run(inputs={"X": x}, time=5)
                if edit:
                    with torch.no_grad():
                        conn.b.mul_(-2.0)
                else:
                    with torch.no_grad():
                        conn.b = torch.nn.Parameter(conn.b.detach() * -2.0, requires_grad=False)
                net.run(inputs={"X": x}, time=5)
            outs.append(net.layers["Y"].v.clone())
        assert torch.equal(outs[0], outs[1]), f"strided={strided}: an in-place bias edit did not take effect"


BAD_BIASES = {
    "short": (lambda: torch.zeros(N_B - 1), RuntimeError),
    "long": (lambda: torch.zeros(N_B + 1), RuntimeError),
    "column": (lambda: torch.zeros(N_B, 1), RuntimeError),
    "per_sample": (lambda: torch.zeros(2, N_B), NotImplementedError),
    "per_sample_column": (lambda: torch.zeros(2, 1), NotImplementedError),
    "float64": (lambda: torch.zeros(N_B, dtype=torch.float64), TypeError),
}


@pytest.mark.parametrize("backend", list(BACKENDS))
@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
@pytest.mark.parametrize("bad", list(BAD_BIASES))
def test_bad_bias_is_refused_before_anything_runs(bad, sparse, backend):
    make, exc = BAD_BIASES[bad]
    net, x = _bias_net(sparse, torch.zeros(N_B))
    conn = net.connections[("X", "Y")]
    conn.b = torch.nn.Parameter(make(), requires_grad=False)   # (float64: assigned after the constructor's cast)
    v0 = net.layers["Y"].v.clone()
    with BACKENDS[backend]()():
        with pytest.raises(exc):
            net.run(inputs={"X": x}, time=5)
        with pytest.raises(exc):
            conn.compute(x[0].bool())
    assert torch.equal(net.layers["Y"].v, v0), f"{bad}: the window ran"
