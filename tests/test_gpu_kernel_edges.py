"""The generic kernel's STDP update (phase3) and the single-operator kernels on the H100 at the batch sizes and shapes
where their fast paths switch (cases and float64 references: tests/kernel_edges.py).  Every result is bit-identical to
the CPU oracle and within the rounding-error bound of a plain float64 restatement of the reference's formulas."""
from dataclasses import replace

import pytest
import torch

import cases
import kernel_edges as ke
from test_kernel_edges import _assert_bit_identical, _assert_within_bound, _check_window, _oracle, _with

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


@pytest.mark.parametrize("case", ke.UPDATE_CASES, ids=lambda c: c.name)
def test_gpu_update_bit_exact_and_within_float64_bound(case):
    d = ke.draw_update(case)
    a = ke.run_update(B200, case, d, device="cuda")
    torch.cuda.synchronize()
    b = _with(_oracle(), lambda: ke.run_update(B200, case, d))
    _assert_bit_identical(a, b, case.name)
    w64, bound = ke.ref_update(case, d)
    _assert_within_bound(a, w64, bound, case.name)
    ke.check_bites(case, d, a)


GPU_WINDOW_CASES = [replace(c, ns=784) for c in ke.WINDOW_CASES]


@pytest.mark.parametrize("case", GPU_WINDOW_CASES, ids=lambda c: c.name)
def test_gpu_window_bit_exact_and_within_float64_bound(case):
    from bindsnet_b200 import _backend

    d = ke.draw_window(case)
    net, inputs = ke.build_window(B200, case, d)
    net.force_tier = 1
    net.to("cuda")
    net.run(inputs={k: v.cuda() for k, v in inputs.items()}, time=case.T)
    net.check_errors()
    assert _backend.last_tier == 1
    a = ke.window_state(net)

    def on_oracle():
        n, i = ke.build_window(B200, case, d)
        n.force_tier = 1
        n.run(inputs=i, time=case.T)
        return ke.window_state(n), float(n.layers["X"].trace_decay)
    b, dec = _with(_oracle(), on_oracle)
    for k in a:
        _assert_bit_identical(a[k].float(), b[k].float(), f"{case.name} {k}")
    _check_window(case, d, a, dec)


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("n_src", [1, 33, 257])
@pytest.mark.parametrize("B", [1, 513, 1100])
def test_gpu_compute_batch_rows_past_the_grid(B, n_src, bias):
    conn, s = ke.compute_setup(B200, n_src, 95, B, bias)
    b = _with(_oracle(), lambda: conn.compute(s))
    out64, bound = ke.ref_compute(conn, s)
    conn.to("cuda")
    a = conn.compute(s.cuda()).cpu()
    _assert_bit_identical(a, b, f"compute B={B} n_src={n_src}")
    _assert_within_bound(a, out64, bound, f"compute B={B} n_src={n_src}")


@pytest.mark.parametrize("mcc", [False, True], ids=["connection_abs", "mcc_feature_plain"])
@pytest.mark.parametrize("n_src", [1, 5, 15, 16, 17, 33])
def test_gpu_normalize_row_chunks_and_zero_column(n_src, mcc):
    outs = []
    for dev in ("cuda", "cpu"):
        conn = ke.normalize_setup(B200, n_src, mcc=mcc)
        w0 = conn.w.detach().clone()
        conn.to(dev)
        ke.poison_weights(conn)   # on the device: a read past n_src rows meets NaN
        if dev == "cpu":
            _with(_oracle(), conn.normalize)
        else:
            conn.normalize()
        outs.append(conn.w.detach().cpu().clone())
    _assert_bit_identical(outs[0], outs[1], f"normalize n_src={n_src}")
    ref, bound = ke.ref_normalize(w0, 7.5 if mcc else 11.0, absolute=not mcc)
    _assert_within_bound(outs[0], ref, bound, f"normalize n_src={n_src}")
    assert (outs[0][:, 3] == 0).all() and torch.isfinite(outs[0]).all()


@pytest.mark.parametrize("geo", ke.CONV_GEOMETRIES, ids=lambda g: "k{}x{}_s{}x{}_p{}x{}_d{}x{}".format(*g[4], *g[5], *g[6], *g[7]))
def test_gpu_conv2d_compute_and_normalize(geo):
    res = []
    for dev in ("cuda", "cpu"):
        conn, s = ke.conv_setup(B200, geo)
        w0 = conn.w.detach().clone()
        conn.to(dev)

        def go():
            out = conn.compute(s.to(dev))
            conn.normalize()
            return out.cpu(), conn.w.detach().cpu().clone()
        res.append(go() if dev == "cuda" else _with(_oracle(), go))
    _assert_bit_identical(res[0][0], res[1][0], "conv compute")
    _assert_bit_identical(res[0][1], res[1][1], "conv normalize")
    out64, bound = ke.ref_conv_compute(conn, s, w0)
    _assert_within_bound(res[0][0], out64, bound, "conv compute")
    w64, wbound = ke.ref_conv_normalize(w0, 3.0)
    _assert_within_bound(res[0][1], w64, wbound, "conv normalize")
