"""Conv1dConnection on the H100: the CUDA library's window kernel and single operators bit for bit against the oracle
(tests/conv1d_oracle.c), on the cases tests/test_conv1d.py checks under emulation, plus the conv1d_MNIST network at
B = 1 and B = 128 over T = 250 and the long-sequence network (Input [4, 4096], B = 32)."""
import pytest
import torch

import cases
import conv1d_nets as cn

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _flat(states):
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


def _same(a, b):
    return torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num()))


def _gpu_vs_oracle(build, n=2, **kw):
    from bindsnet_b200 import _backend
    from conv1d_oracle import Conv1dOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = build()
        if gpu:
            net.to("cuda")
            inputs = {k: v.cuda() for k, v in inputs.items()}
            outs.append(_flat(cn.run_windows(net, inputs, T, n, **kw)))
            net.check_errors()
            assert _backend.lib().snn_b200_abi_version() == 13
        else:
            with Conv1dOracleBackend() as ob:
                outs.append(_flat(cn.run_windows(net, inputs, T, n, **kw)))
            assert ob.err == 0
    a, b = outs
    assert a.keys() == b.keys()
    for k in a:
        assert _same(a[k], b[k]), f"{k} differs from the oracle"
    return a


@pytest.mark.parametrize("case", list(cn.LIVE_CASES))
def test_window_bit_exact(case):
    a = _gpu_vs_oracle(lambda: cn.build_case(B200, case), n=cn.windows_of(case))
    assert a["w0/Ys"].sum() > 0


@pytest.mark.parametrize("rule", ["PostPre", "WeightDependentPostPre", "Hebbian"])
def test_one_step_large_batch_and_no_reset_bit_exact(rule):
    _gpu_vs_oracle(lambda: cn.multi_net(B200, rule=rule), one_step=True)
    _gpu_vs_oracle(lambda: cn.multi_net(B200, rule=rule, T=9), reset=False)
    a = _gpu_vs_oracle(lambda: cn.multi_net(B200, rule=rule, B=520, T=9))
    assert a["w0/Ys"].sum() + a["w1/Ys"].sum() > 0


@pytest.mark.parametrize("B", [1, 128])
def test_example_network_t250_bit_exact(B):
    """The conv1d_MNIST network (Input [1, 784], kernel 56, stride 28, 25 filters, PostPre) with learning on."""
    net, _, _ = cn.example_net(B200, B=B)
    a = _gpu_vs_oracle(lambda: cn.example_net(B200, B=B, T=250), n=1)
    assert a["w0/Ys"].sum() > 0 and not torch.equal(a["w0/XY/w"], net.connections[("X", "Y")].w)


def test_long_sequence_bit_exact():
    """Input [4, 4096] -> Conv1dConnection (kernel 9, stride 1, padding 4, 32 filters, PostPre) -> LIFNodes [32, 4096]
    at B = 32, T = 20 (the oracle's share of the test time grows with T)."""
    a = _gpu_vs_oracle(lambda: cn.long_net(B200, T=20, rate=0.05), n=1)
    assert a["w0/Ys"].sum() > 0


def test_standalone_operators_bit_exact():
    from conv1d_oracle import Conv1dOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = cn.multi_net(B200, rule="WeightDependentPostPre", B=3, bias=True)
        conn = net.connections[("X", "Y")]
        X, Y = net.layers["X"], net.layers["Y"]
        s = torch.rand(3, 2, 20, generator=torch.Generator().manual_seed(3)) < 0.4
        X.s, X.x = s.clone(), torch.rand(3, 2, 20, generator=torch.Generator().manual_seed(4))
        Y.s = torch.rand(3, 3, 10, generator=torch.Generator().manual_seed(5)) < 0.3
        Y.x = torch.rand(3, 3, 10, generator=torch.Generator().manual_seed(6))
        if gpu:
            net.to("cuda")
            out = conn.compute(s.cuda())
            conn.update_rule.update()
            conn.normalize()
        else:
            with Conv1dOracleBackend():
                out = conn.compute(s)
                conn.update_rule.update()
                conn.normalize()
        outs.append((out.cpu(), conn.w.detach().cpu().clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
