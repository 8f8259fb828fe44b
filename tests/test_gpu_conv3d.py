"""Conv3dConnection on the H100: the CUDA library's window kernel and single operators bit for bit against the oracle
(tests/conv3d_oracle.c), on the cases tests/test_conv3d.py checks under emulation, plus conv3d_MNIST's network at B = 1,
T = 250 and at B = 128, T = 40."""
import pytest
import torch

import cases
import conv3d_nets as cn

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _flat(states):
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


def _same(a, b):
    return torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num()))


def _gpu_vs_oracle(build, n=2, **kw):
    from bindsnet_b200 import _abi, _backend
    from conv3d_oracle import Conv3dOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = build()
        if gpu:
            net.to("cuda")
            inputs = {k: v.cuda() for k, v in inputs.items()}
            outs.append(_flat(cn.run_windows(net, inputs, T, n, **kw)))
            net.check_errors()
            assert _backend.lib().snn_b200_abi_version() == _abi.SNN_ABI_VERSION
        else:
            with Conv3dOracleBackend() as ob:
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


def test_one_step_large_batch_and_no_reset_bit_exact():
    _gpu_vs_oracle(lambda: cn.multi_net(B200, rule="NoOp", weight_decay=1e-2), one_step=True)
    a = _gpu_vs_oracle(lambda: cn.multi_net(B200, rule="PostPre", weight_decay=1e-2, wmin=0.05, wmax=0.45, B=520, T=9))
    assert a["w1/Ys"].sum() > 0
    _gpu_vs_oracle(lambda: cn.multi_net(B200, rule="NoOp", weight_decay=1e-2, T=9), reset=False)


def test_wide_kernel_and_unstaged_taps_bit_exact():
    a = _gpu_vs_oracle(lambda: cn.wide_net(B200))
    assert a["w1/Ys"].sum() > 0


def test_example_unstaged_bits_bit_exact():
    a = _gpu_vs_oracle(lambda: cn.example_net(B200, B=8, T=10, learning=False), n=1)
    assert a["w0/Ys"].sum() > 0


def test_example_network_b1_t250_bit_exact():
    """conv3d_MNIST's network (one_spike as in the example) with learning off at B = 1, T = 250."""
    a = _gpu_vs_oracle(lambda: cn.example_net(B200, T=250, learning=False, one_spike=True), n=1, one_spike_seed=7)
    assert a["w0/Ys"].sum() > 0


def test_example_network_b128_t40_bit_exact():
    """The same network with learning.NoOp's decay at B = 128, T = 40."""
    a = _gpu_vs_oracle(lambda: cn.example_net(B200, B=128, T=40, rule="NoOp", weight_decay=1e-3, one_spike=True), n=1,
                       one_spike_seed=7)
    assert a["w0/Ys"].sum() > 0


def test_standalone_operators_bit_exact():
    from conv3d_oracle import Conv3dOracleBackend

    outs = []
    for gpu in (True, False):
        net, _, _ = cn.multi_net(B200, rule="PostPre", weight_decay=1e-2, wmin=0.05, wmax=0.45, B=3)
        conn = net.connections[("X", "Y")]
        for L in net.layers.values():
            L.set_batch_size(3)
            L.compute_decays(1.0)
        s = torch.rand(3, 2, 7, 9, 8, generator=torch.Generator().manual_seed(3)) < 0.4
        if gpu:
            net.to("cuda")
            out = conn.compute(s.cuda())
            conn.update_rule.update()
            conn.normalize()
        else:
            with Conv3dOracleBackend():
                out = conn.compute(s)
                conn.update_rule.update()
                conn.normalize()
        outs.append((out.cpu(), conn.w.detach().cpu().clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
