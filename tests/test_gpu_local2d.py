"""LocalConnection2D on the H100: the CUDA library's window kernel and single operators bit for bit against the oracle
(tests/local2d_oracle.c), on the cases tests/test_local2d.py checks under emulation, plus the full loc2d_mnist network at
B = 1, T = 250 and a batched variant (Input [1, 28, 28]) at B = 128, T = 250."""
import pytest
import torch

import cases
import local2d_nets as ln

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _flat(states):
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


def _same(a, b):
    return torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num()))


def _gpu_vs_oracle(build, n=2, **kw):
    from bindsnet_b200 import _backend
    from local2d_oracle import Local2dOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = build()
        if gpu:
            net.to("cuda")
            inputs = {k: v.cuda() for k, v in inputs.items()}
            outs.append(_flat(ln.run_windows(net, inputs, T, n, **kw)))
            net.check_errors()
            assert _backend.lib().snn_b200_abi_version() == 13
        else:
            with Local2dOracleBackend() as ob:
                outs.append(_flat(ln.run_windows(net, inputs, T, n, **kw)))
            assert ob.err == 0
    a, b = outs
    assert a.keys() == b.keys()
    for k in a:
        assert _same(a[k], b[k]), f"{k} differs from the oracle"
    return a


@pytest.mark.parametrize("case", list(ln.LIVE_CASES))
def test_window_bit_exact(case):
    a = _gpu_vs_oracle(lambda: ln.build_case(B200, case), n=ln.windows_of(case))
    assert a["w0/Ys"].sum() > 0


@pytest.mark.parametrize("rule", ["PostPre", "WeightDependentPostPre"])
def test_one_step_and_large_batch_bit_exact(rule):
    _gpu_vs_oracle(lambda: ln.multi_net(B200, rule=rule), one_step=True)
    a = _gpu_vs_oracle(lambda: ln.multi_net(B200, rule=rule, B=520, T=9))
    assert a["w1/Ys"].sum() > 0


def test_example_network_t250_bit_exact():
    """The full loc2d_mnist network (Input [1, 20, 20]) at B = 1, T = 250."""
    a = _gpu_vs_oracle(lambda: ln.example_net(B200, T=250, rate=0.05), n=1)
    assert a["w0/Ys"].sum() > 0


def test_batched_variant_b128_t250_bit_exact():
    """Input [1, 28, 28], kernel 12, stride 4, 50 filters (1250 target neurons) at B = 128, T = 250."""
    a = _gpu_vs_oracle(lambda: ln.example_net(B200, B=128, T=250, H=28, W=28, rate=0.05), n=1)
    assert a["w0/Ys"].sum() > 0


def test_standalone_operators_bit_exact():
    from local2d_oracle import Local2dOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = ln.multi_net(B200, rule="WeightDependentPostPre", B=3)
        conn = net.connections[("X", "Y")]
        X, Y = net.layers["X"], net.layers["Y"]
        s = torch.rand(3, 2, 11, 10, generator=torch.Generator().manual_seed(3)) < 0.4
        X.s, X.x = s.clone(), torch.rand(3, 2, 11, 10, generator=torch.Generator().manual_seed(4))
        Y.s = torch.rand(3, 3, 5, 3, generator=torch.Generator().manual_seed(5)) < 0.3
        Y.x = torch.rand(3, 3, 5, 3, generator=torch.Generator().manual_seed(6))
        if gpu:
            net.to("cuda")
            out = conn.compute(s.cuda())
            conn.update_rule.update()
            conn.normalize()
        else:
            with Local2dOracleBackend():
                out = conn.compute(s)
                conn.update_rule.update()
                conn.normalize()
        outs.append((out.cpu(), conn.w.detach().cpu().clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
