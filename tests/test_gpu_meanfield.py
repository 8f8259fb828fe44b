"""MeanFieldConnection on the H100: the CUDA library against the oracle (tests/meanfield_oracle.c), bit for bit, on the
networks of tests/meanfield_nets.py, and a large case."""
import pytest
import torch

import cases
import meanfield_nets as mn

pytestmark = pytest.mark.gpu
B200 = cases.namespace("b200")


def _gpu_vs_oracle(build, **kw):
    from meanfield_oracle import MeanFieldOracleBackend

    outs = []
    for dev in ("cuda", "cpu"):
        net, inputs, T, rkw = build()
        if dev == "cuda":
            net.to("cuda")
            net.force_tier = 1
            inputs = {k: v.cuda() for k, v in inputs.items()}
            rkw = {k: {n: m.cuda() for n, m in v.items()} for k, v in rkw.items()}
            outs.append(mn.flat(mn.run_two_windows(net, inputs, T, **rkw, **kw)))
            net.check_errors()
        else:
            with MeanFieldOracleBackend():
                outs.append(mn.flat(mn.run_two_windows(net, inputs, T, **rkw, **kw)))
    a, b = outs
    for k in b:
        assert torch.equal(a[k], b[k]), f"{k} differs"


@pytest.mark.parametrize("case", mn.LIVE_CASES)
def test_window_bit_exact(case):
    _gpu_vs_oracle(lambda: mn.mf_net(B200, case))


@pytest.mark.parametrize("case", ["b3_in_n_mf", "b8_dc1_c1_mf", "b3_self_n_mf_dense", "b8_in_full_mf_dense"])
def test_one_step_bit_exact(case):
    _gpu_vs_oracle(lambda: mn.mf_net(B200, case), one_step=True)


@pytest.mark.parametrize("B,T", [(520, 5), (7, 13)])
def test_batch_sizes_bit_exact(B, T):
    _gpu_vs_oracle(lambda: mn.mf_net(B200, f"b{B}_lif_full_mf_dense", T=T))


@pytest.mark.parametrize("form", ["0d", "n", "1w", "c1", "full"])
def test_standalone_compute(form):
    B = 5
    g = torch.Generator().manual_seed(3)
    w = mn.w_of(form, B, g)
    c = B200.topology.MeanFieldConnection(B200.nodes.Input(n=37), B200.nodes.LIFNodes(shape=[2, 4]), w=w).to("cuda")
    s = torch.bernoulli(0.3 * torch.ones(B, 37), generator=g).bool()
    out = c.compute(s.cuda())
    assert torch.equal(out.cpu(), s.float().mean() * w)


def test_large_case_bit_exact():
    """Input(784) -> LIF(1600) with PostPre and a LIF -> LIF mean-field connection with negative per-target w, B = 128,
    T = 250: the GPU window against the oracle."""
    from meanfield_oracle import MeanFieldOracleBackend

    res = []
    for dev in ("cuda", "cpu"):
        net, inputs, T = mn.big_net(B200, B=128, T=250)
        if dev == "cuda":
            net.to("cuda")
            net.run(inputs={"X": inputs["X"].cuda()}, time=T)
            net.check_errors()
        else:
            with MeanFieldOracleBackend():
                net.run(inputs=inputs, time=T)
        res.append(mn.state(net, monitors=False))
    for k in res[1]:
        assert torch.equal(res[0][k].cpu(), res[1][k]), k
    assert res[1]["A/s"].sum() > 0 and res[1]["Z/s"].sum() >= 0
