"""MulticompartmentConnection features (Probability / Mask / Intensity) on the H100: the CUDA library's feature gather bit
for bit against the oracle (tests/feature_oracle.c), the equivalences that need no oracle, and the distribution of the
synapse draw at n_src = n_tgt = 4096."""
import numpy as np
import pytest
import torch

import cases
import helpers
import mcc_feature_nets as fn
from test_mcc_features import _ff_net, _mats, _prob_pipe

pytestmark = pytest.mark.gpu

B200 = cases.namespace("b200")


def _gpu_vs_oracle(build, windows=1, one_step=False):
    from feature_oracle import FeatureOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = build()
        net.force_tier = 1
        if gpu:
            net.to("cuda")
            inputs = {k: v.cuda() for k, v in inputs.items()}
            for w in range(windows):
                net.run(inputs=inputs, time=T, one_step=one_step, one_spike_seed=fn.SEED + w)
            net.check_errors()
        else:
            with FeatureOracleBackend() as ob:
                for w in range(windows):
                    net.run(inputs=inputs, time=T, one_step=one_step, one_spike_seed=fn.SEED + w)
            assert ob.err == 0
        outs.append(fn.snapshot(net, T))
    return outs


@pytest.mark.parametrize("case", fn.LIVE_CASES)
def test_gpu_live_cases_bit_exact(case):
    a, b = _gpu_vs_oracle(lambda: fn.live_net(B200, case))
    helpers.assert_bit_identical(a, b, case)
    assert a["M/Ys"].sum() > 0


@pytest.mark.parametrize("case", ["prob_b4", "mask_int"])
def test_gpu_one_step_two_windows_bit_exact(case):
    a, b = _gpu_vs_oracle(lambda: fn.live_net(B200, case), windows=2, one_step=True)
    helpers.assert_bit_identical(a, b, f"{case} one_step")
    a, b = _gpu_vs_oracle(lambda: fn.live_net(B200, case), windows=2)
    helpers.assert_bit_identical(a, b, f"{case} two windows")


def test_gpu_wide_source_and_large_batch_bit_exact():
    for build, what in ((fn.wide_net, "9000-neuron source"), (fn.big_batch_net, "B = 520")):
        a, b = _gpu_vs_oracle(lambda: build(B200))
        helpers.assert_bit_identical(a, b, what)
        assert a["M/Ys"].sum() > 0


def _run_gpu(net, inputs, T, one_step=False):
    net.to("cuda")
    net.run(inputs={k: v.cuda() for k, v in inputs.items()}, time=T, one_step=one_step, one_spike_seed=fn.SEED)
    net.check_errors()
    return {k: v for k, v in fn.snapshot(net, T).items() if not k.startswith("C/")}


def test_gpu_equivalences():
    w, m, i = _mats(torch.Generator().manual_seed(5))
    pairs = [
        ([lambda F, g: [F.Weight("w", w), F.Mask("m", m)]], lambda F, g: [F.Weight("w", w * m)], "Mask"),
        ([lambda F, g: [F.Intensity("i", i), F.Weight("w", w)]], lambda F, g: [F.Weight("w", w * i)], "Intensity"),
        ([lambda F, g: [F.Probability("p", m.float()), F.Weight("w", w)]], lambda F, g: [F.Mask("m", m), F.Weight("w", w)], "Probability 0/1"),
    ]
    for (a_of,), b_of, what in pairs:
        a, b = _run_gpu(*_ff_net(a_of)), _run_gpu(*_ff_net(b_of))
        helpers.assert_bit_identical(a, b, what)
        assert a["M/Ys"].sum() > 0
    for one_step in (False, True):
        a = _run_gpu(*_ff_net(_prob_pipe, stepwise=True), one_step=one_step)
        b = _run_gpu(*_ff_net(_prob_pipe), one_step=one_step)
        a.pop("M/Ys"); b.pop("M/Ys")
        helpers.assert_bit_identical(a, b, f"stepwise vs window one_step={one_step}")


def test_gpu_scripted_tier_matches_oracle():
    from feature_oracle import FeatureOracleBackend

    outs = []
    for gpu in (True, False):
        net, inputs, T = _ff_net(_prob_pipe, user=True)
        if gpu:
            outs.append(_run_gpu(net, inputs, T))
        else:
            with FeatureOracleBackend():
                net.run(inputs=inputs, time=T, one_spike_seed=fn.SEED)
            outs.append({k: v for k, v in fn.snapshot(net, T).items() if not k.startswith("C/")})
    helpers.assert_bit_identical(outs[0], outs[1], "scripted tier on the GPU vs oracle")


N = 4096


def _draw_conn(p, w=None):
    F, _ = fn.features(B200)
    X, Y = B200.nodes.Input(N), B200.nodes.LIFNodes(N)
    w = torch.ones(N, N) if w is None else w
    c = B200.topology.MulticompartmentConnection(source=X, target=Y, device="cuda", pipeline=[F.Probability("p", p), F.Weight("w", w)])
    return c


def test_gpu_draw_distribution():
    """p constant along each column, uniform over the columns: the transmitted count of a column is Binomial(4096, p_j);
    per p bin within 5 sigma.  Samples of one step see one mask; consecutive steps and windows are uncorrelated."""
    from bindsnet_b200.network import _plan

    g = torch.Generator().manual_seed(0)
    pcol = torch.rand(N, generator=g)
    c = _draw_conn(pcol.expand(N, N).contiguous(), w=torch.rand(N, N, generator=g))
    ones = torch.ones(4, N, dtype=torch.bool, device="cuda")
    out = _plan.compute_single_connection(c, ones, draw=(11, 0, 0))
    assert torch.equal(out[0].view(torch.int32).expand(4, N), out.view(torch.int32)), "samples of one step saw different masks"

    c1 = _draw_conn(pcol.expand(N, N).contiguous())
    cnt = _plan.compute_single_connection(c1, ones[:1], draw=(11, 0, 0))[0].double().cpu()
    for lo in np.arange(0.0, 1.0, 0.1):
        sel = (pcol >= lo) & (pcol < lo + 0.1)
        pj = pcol[sel].double()
        expect, var = (N * pj).sum(), (N * pj * (1 - pj)).sum()
        assert abs(float(cnt[sel].sum() - expect)) < 5 * float(var.sqrt()), lo

    # per-synapse masks of 16 rows: sample b spikes row 256 * b only, w = 1
    half = _draw_conn(torch.full((N, N), 0.5))
    s = torch.zeros(16, N, dtype=torch.bool, device="cuda")
    s[torch.arange(16), torch.arange(16) * 256] = True
    masks = {key: _plan.compute_single_connection(half, s, draw=key).flatten().double() - 0.5
             for key in ((11, 0, 0), (11, 1, 0), (12, 0, 0), (11, 0, 1))}
    base = masks[(11, 0, 0)]
    assert abs(float(base.mean())) < 5 * 0.5 / (16 * N) ** 0.5
    for key in ((11, 1, 0), (12, 0, 0), (11, 0, 1)):   # next step, next window's seed, next connection
        r = float((base * masks[key]).mean() / 0.25)
        assert abs(r) < 5 / (16 * N) ** 0.5, (key, r)
