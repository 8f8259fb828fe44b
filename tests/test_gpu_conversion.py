"""ann_to_snn networks on the H100: the CUDA library's window kernel bit for bit against the oracle
(tests/conversion_oracle.c), on the cases tests/test_conversion.py checks under emulation, plus the full LeNet-5
conversion at B = 128, T = 250."""
import pytest
import torch

import cases
import conversion_nets as cn
from test_conversion import _build

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _gpu_vs_oracle(build, **kw):
    from conversion_oracle import ConversionOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = build()
        if gpu:
            net.to("cuda")
            net.reset_state_variables()   # (the pooling rates buffers are reallocated on the layers' device)
            inputs = {k: v.cuda() for k, v in inputs.items()}
            outs.append(cn.flat(cn.run_two_windows(net, inputs, T, **kw)))
            net.check_errors()
        else:
            net.reset_state_variables()
            with ConversionOracleBackend() as ob:
                outs.append(cn.flat(cn.run_two_windows(net, inputs, T, **kw)))
            assert ob.err == 0
    a, b = outs
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), f"{k} differs from the oracle"
    return a


@pytest.mark.parametrize("case", ["cnn_b1", "cnn_b4", "subif_refrac", "subif_lbound", "subif_traces", "subif_postpre", "passthrough"])
def test_window_bit_exact(case):
    _gpu_vs_oracle(lambda: _build(B200, case))


@pytest.mark.parametrize("case", ["cnn_b4", "passthrough"])
def test_one_step_bit_exact(case):
    _gpu_vs_oracle(lambda: _build(B200, case), one_step=True)


def test_large_batch_odd_T_bit_exact():
    a = _gpu_vs_oracle(lambda: cn.cnn_net(B200, 520, T=7, monitors=False))
    assert a["w1/4/s"].sum() > 0


def test_nonbinary_passthrough_input_is_flagged():
    from bindsnet_b200 import _backend

    net, inputs, T = cn.passthrough_net(B200)
    net.to("cuda")
    x = inputs["P"][0].clone()
    x[3, 0, 0, 0, 0] = 0.5
    net.run({"P": x.cuda()}, time=T)
    with pytest.raises(_backend.BackendError, match="outside"):
        net.check_errors()


def test_lenet5_b128_t250_bit_exact():
    """The full LeNet-5 conversion (data_based_normalization on seeded images) at B = 128 over a 250-step window."""

    def build():
        net = cn.convert(B200, "lenet5", data=True)
        net.train(False)
        cn.set_batch(net, 128)
        return net, {"Input": cn.rate_inputs((1, 28, 28), 250, 128, seed=12, p=0.3)}, 250

    a = _gpu_vs_oracle(build)
    assert a["w1/10/s"].sum() > 0 and a["w1/12/summed"].abs().sum() > 0
