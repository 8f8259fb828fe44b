"""SparseConnection on the H100: the CUDA library's sparse gather bit for bit against the oracle, and against a dense
Connection holding the same values.  The oracle is tests/sparse_oracle.c (the CPU oracle extended by the sparse kind)."""
import pytest
import torch

import cases
import helpers
import sparse_nets as sn

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _gpu_vs_oracle(build, T, windows=1, one_step=False):
    from sparse_oracle import SparseOracleBackend as OracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, *_ = build()
        net.force_tier = 1
        if gpu:
            net.to("cuda")
            inputs = {k: v.cuda() for k, v in inputs.items()}
            for _ in range(windows):
                net.run(inputs=inputs, time=T, one_step=one_step)
            net.check_errors()
        else:
            with OracleBackend() as ob:
                for _ in range(windows):
                    net.run(inputs=inputs, time=T, one_step=one_step)
            assert ob.err == 0
        outs.append(sn.snapshot(net, T))
    return outs


@pytest.mark.parametrize("decay", [False, True])
def test_gpu_live_case_bit_exact(decay):
    def build():
        net, inputs = sn.live_net(B200, decay)
        helpers.add_spike_monitors(net, sn.T_LIVE)
        return net, inputs
    a, b = _gpu_vs_oracle(build, sn.T_LIVE)
    helpers.assert_bit_identical(a, b, f"live case decay={decay}")


@pytest.mark.parametrize("seed", list(range(12)))
def test_gpu_random_sparse_networks_bit_exact(seed):
    spec = sn.random_net(B200, seed)[2]
    a, b = _gpu_vs_oracle(lambda: sn.random_net(B200, seed), spec["T"], windows=2, one_step=spec["one_step"])
    helpers.assert_bit_identical(a, b, f"seed {seed} {spec}")


def test_gpu_large_index_bit_exact():
    a, b = _gpu_vs_oracle(lambda: sn.big_index_net(B200), 4)
    helpers.assert_bit_identical(a, b, "50 000 x 50 000")
    assert a["L/Y/count"].sum() > 0


def test_gpu_reservoir_bit_exact():
    """N = 20 000, p = 2 %, B = 32, T = 100."""
    def build():
        net, inputs = sn.reservoir(B200, 20_000, 0.02, 32, 100)
        helpers.add_spike_monitors(net, 100)
        return net, inputs
    a, b = _gpu_vs_oracle(build, 100)
    helpers.assert_bit_identical(a, b, "reservoir 20 000 / 2 %")
    assert a["L/Y/count"].sum() > 0


@pytest.mark.parametrize("decay", [False, True])
def test_gpu_sparse_equals_dense_connection(decay):
    outs = []
    for dense in (False, True):
        net, inputs = sn.live_net(B200, decay, dense_recurrent=dense, dense_input=dense)
        net.force_tier = 1
        net.to("cuda")
        net.run(inputs={k: v.cuda() for k, v in inputs.items()}, time=sn.T_LIVE)
        net.check_errors()
        st = {k: v.cpu() for k, v in sn.live_state(net).items() if not k.startswith(("XY", "YY"))}
        st["XY"] = net.connections[("X", "Y")].w.detach().cpu()
        st["YY"] = net.connections[("Y", "Y")].w.detach().cpu()
        outs.append(st)
    for k in outs[0]:
        a, b = outs[0][k], outs[1][k]
        if a.is_sparse:
            a = a.coalesce()
            assert torch.equal(a.values().view(torch.int32), b[a.indices()[0], a.indices()[1]].view(torch.int32)), k
        else:
            assert torch.equal(a.view(torch.int32) if a.is_floating_point() else a, b.view(torch.int32) if b.is_floating_point() else b), k
