"""LocalConnection3D on the H100: the CUDA library's window kernel and single operators bit for bit against the oracle
(tests/local3d_oracle.c), on the cases tests/test_local3d.py checks under emulation, plus the full loc3d_mnist network at
B = 1, T = 250 and at B = 32, T = 40 (reduction=torch.sum)."""
import pytest
import torch

import cases
import local3d_nets as ln

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _flat(states):
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


def _same(a, b):
    return torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num()))


def _gpu_vs_oracle(build, n=2, **kw):
    from bindsnet_b200 import _backend
    from local3d_oracle import Local3dOracleBackend

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
            with Local3dOracleBackend() as ob:
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
def test_one_step_and_batch_sizes_bit_exact(rule):
    _gpu_vs_oracle(lambda: ln.multi_net(B200, rule=rule), one_step=True)
    _gpu_vs_oracle(lambda: ln.multi_net(B200, rule=rule, T=9), reset=False)
    for B in (3, 33, 520):
        a = _gpu_vs_oracle(lambda: ln.multi_net(B200, rule=rule, B=B, T=9))
        assert a["w1/Ys"].sum() > 0


@pytest.mark.parametrize("B", [3, 33])
def test_staged_unstaged_and_wide_rows_bit_exact(B):
    """A [1, 20, 20, 20] source: staged bit rows at B = 3, unstaged at B = 33; and kernel rows of 36 bits."""
    _gpu_vs_oracle(lambda: ln.multi_net(B200, rule="Hebbian", B=B, T=7, shape=(1, 20, 20, 20), kernel=(2, 3, 4), stride=(3, 3, 3),
                                        filters=2))
    _gpu_vs_oracle(lambda: ln.multi_net(B200, rule="PostPre", B=B, T=7, shape=(1, 3, 2, 45), kernel=(2, 1, 36), stride=(1, 1, 4),
                                        filters=2))


def test_example_network_t250_bit_exact():
    """The full loc3d_mnist network (Input [1, 20, 20, 20], 2.76 M weights) at B = 1, T = 250."""
    a = _gpu_vs_oracle(lambda: ln.example_net(B200, T=250), n=1)
    assert a["w0/Ys"].sum() > 0


def test_example_network_b32_t40_bit_exact():
    """The loc3d_mnist network at B = 32, T = 40, reduction=torch.sum."""
    a = _gpu_vs_oracle(lambda: ln.example_net(B200, B=32, T=40, reduction=torch.sum), n=1)
    assert a["w0/Ys"].sum() > 0


def test_standalone_operators_bit_exact():
    from local3d_oracle import Local3dOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = ln.multi_net(B200, rule="WeightDependentPostPre", B=3)
        conn = net.connections[("X", "Y")]
        X, Y = net.layers["X"], net.layers["Y"]
        s = torch.rand(3, 2, 7, 5, 11, generator=torch.Generator().manual_seed(3)) < 0.4
        X.s, X.x = s.clone(), torch.rand(3, 2, 7, 5, 11, generator=torch.Generator().manual_seed(4))
        Y.s = torch.rand(3, 3, 3, 4, 3, generator=torch.Generator().manual_seed(5)) < 0.3
        Y.x = torch.rand(3, 3, 3, 4, 3, generator=torch.Generator().manual_seed(6))
        if gpu:
            net.to("cuda")
            out = conn.compute(s.cuda())
            conn.update_rule.update()
            conn.normalize()
        else:
            with Local3dOracleBackend():
                out = conn.compute(s)
                conn.update_rule.update()
                conn.normalize()
        outs.append((out.cpu(), conn.w.detach().cpu().clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
