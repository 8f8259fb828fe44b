"""Networks whose Weight is normalised every time step (``Weight(norm_frequency='time step')``) or by a per-target norm
tensor, shared by tests/test_weight_norm.py (CPU: oracle, emulated kernel), tests/test_gpu_weight_norm.py (the CUDA
library) and bench_weight_norm.py.  ``ns`` is a ``cases.namespace``."""
from __future__ import annotations

import numpy as np
import torch

from mcc_feature_nets import SEED, features, patch_reference_probability

# ts / tt: 'time step' Weight with a scalar / [n_tgt] tensor norm; noop / pp / mstdp / mstdpet the rule; 1 / 4 the batch
# size.  pw: [Probability, Weight]; wm: [Weight, Mask]; off: every window with learning off; manual: manual_update; neg:
# negative weights, a zero column and a clamping range; sample_t: a 'sample' Weight with a tensor norm; conn_t: a dense
# Connection with a [n_tgt] norm; t5: odd T.  custom=True makes the target a user-defined population (scripted tier)
CASES = ["ts_noop1", "tt_noop1", "ts_pp1", "tt_pp4", "ts_pp4", "ts_mstdp4", "tt_mstdpet1", "pw", "wm", "off", "manual", "neg",
         "sample_t", "conn_t", "t5"]
# compared with the live reference (stored by ``python tests/golden/gen_live.py test_weight_norm``)
LIVE_CASES = ["ts_noop1", "tt_noop1", "ts_pp1", "tt_pp4", "ts_mstdp4", "tt_mstdpet1", "pw", "wm", "off", "manual", "neg",
              "sample_t", "conn_t", "t5"]


def params(case: str) -> dict:
    p = dict(norm="s", freq="time step", rule="pp", B=1, pipe="W", T=8, rng=[-1.0, 4.0], learning=True, manual=False,
             neg=False, conn=False)
    if case[:2] in ("ts", "tt"):
        p["norm"] = case[1]
        p["rule"] = case[3:-1]
        p["B"] = int(case[-1])
    p.update({"pw": dict(pipe="PW", B=4, norm="t"), "wm": dict(pipe="WM"), "off": dict(learning=False, norm="t"),
              "manual": dict(manual=True), "neg": dict(neg=True, norm="t", rng=[-0.6, 0.8], B=4),
              "sample_t": dict(freq="sample", norm="t", B=4), "conn_t": dict(conn=True, norm="t", B=4),
              "t5": dict(T=5, norm="t")}.get(case, {}))
    return p


def norm_value(p: dict, n: int, g: torch.Generator):
    return 6.0 + 4.0 * torch.rand(n, generator=g) if p["norm"] == "t" else 7.5


def build(ns, case: str, B: int = None, n_in: int = 40, n: int = 30, T: int = None, custom: bool = False):
    """Input(n_in) -> [MCC pipeline with the normalised Weight, or a dense Connection] -> LIFNodes(n), plus a static
    recurrent MCC Weight on the LIF layer.  Returns (net, inputs for three windows, T, run kwargs)."""
    F, ML = features(ns)
    p = params(case)
    B = B or p["B"]
    T = T or p["T"]
    g = torch.Generator().manual_seed(sum(map(ord, case)) + B + n_in)
    X = ns.nodes.Input(n_in, traces=True)
    if custom:
        from test_scripted_tier import MyLIF

        Y = MyLIF(n, traces=True, thresh=-58.0, tc_decay=30.0, refrac=3)
    else:
        Y = ns.nodes.LIFNodes(n, traces=True, thresh=-58.0, tc_decay=30.0, refrac=3)
    net = ns.Network(dt=1.0, batch_size=B, learning=p["learning"])
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    w1 = 0.25 * torch.rand(n_in, n, generator=g)
    if p["neg"]:
        w1 = w1 - 0.08
        w1[:, 3] = 0.0   # a zero column
    norm = norm_value(p, n, g)
    if p["conn"]:
        xy = ns.topology.Connection(source=X, target=Y, w=w1, update_rule=ns.learning.PostPre, nu=(4e-3, 3e-3), norm=norm,
                                    wmin=-1.0, wmax=1.0)
    else:
        rule = {"noop": None, "pp": ML.PostPre, "mstdp": ML.MSTDP, "mstdpet": ML.MSTDPET}[p["rule"]]
        kw = dict(learning_rule=rule, nu=(4e-3, 3e-3), range=p["rng"]) if rule is not None else dict(range=p["rng"])
        make = {"P": lambda: F.Probability(name="p", value=0.3 + 0.7 * torch.rand(n_in, n, generator=g)),
                "M": lambda: F.Mask(name="m", value=torch.rand(n_in, n, generator=g) < 0.6),
                "W": lambda: F.Weight(name="w", value=w1, norm=norm, norm_frequency=p["freq"], **kw)}
        xy = ns.topology.MulticompartmentConnection(source=X, target=Y, device="cpu", pipeline=[make[k]() for k in p["pipe"]],
                                                    manual_update=p["manual"])
    yy = ns.topology.MulticompartmentConnection(source=Y, target=Y, device="cpu",
                                                pipeline=[F.Weight(name="r", value=-1.5 * torch.rand(n, n, generator=g),
                                                                   range=[-2.0, 0.0])])
    net.add_connection(xy, "X", "Y")
    net.add_connection(yy, "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(3 * T, B, n_in, generator=g) < 0.3).to(torch.uint8)
    kwargs = {"reward": 0.5} if p["rule"] in ("mstdp", "mstdpet") else {}
    return net, {"X": x}, T, kwargs


def weight_of(conn) -> torch.Tensor:
    if hasattr(conn, "pipeline"):
        return [f for f in conn.pipeline if type(f).__name__ == "Weight"][0].value
    return conn.w


def run_windows(net, inputs, T, kwargs, one_step=False, reset=True, reference=False) -> None:
    """Window 0 with the case's learning flag, reset_state_variables, window 1 with learning off, window 2 as window 0;
    the draws of window k use seed SEED + k (the reference's Probability patched to match)."""
    learning = net.learning
    for k in range(3):
        net.learning = learning and k != 1
        x = {name: v[k * T:(k + 1) * T] for name, v in inputs.items()}
        if reference:
            if all(hasattr(c, "pipeline") for c in net.connections.values()):
                patch_reference_probability(net, SEED + k)
            net.run(inputs=x, time=T, one_step=one_step, **kwargs)
        else:
            net.run(inputs=x, time=T, one_spike_seed=SEED + k, one_step=one_step, **kwargs)
        if k == 0 and reset:
            net.reset_state_variables()
    net.learning = learning


def full_snapshot(net, T) -> dict:
    """Spikes, layer state, every weight and the monitored raster, as numpy arrays (for bit-for-bit comparisons)."""
    out = {}
    for lname, layer in net.layers.items():
        Bz = layer.s.shape[0]
        out[f"L/{lname}/s"] = layer.s.reshape(Bz, -1).to(torch.uint8).cpu().numpy()
        for var in ("v", "refrac_count", "x", "theta"):
            val = getattr(layer, var, None)
            if isinstance(val, torch.Tensor) and val.numel() > 0:
                out[f"L/{lname}/{var}"] = val.detach().reshape(-1).float().cpu().numpy()
    if "Ys" in net.monitors:
        out["M/Ys"] = net.monitors["Ys"].get("s").to(torch.uint8).cpu().numpy()
    for (s, t), c in net.connections.items():
        out[f"W/{s}{t}"] = weight_of(c).detach().cpu().numpy()
    return out


def dc_graph(ns, B: int, freq: str, n_in: int = 784, n: int = 1600, T: int = 250, seed: int = 0):
    """The DiehlAndCook2015 shape: Input(n_in) -> DiehlAndCookNodes(n) with the input Weight normalised to 78.4 (per
    sample or every step) and learning by MCC PostPre, and lateral inhibition through a second population of n.
    Returns (net, Poisson-like input [T, B, n_in])."""
    F, ML = features(ns)
    g = torch.Generator().manual_seed(seed)
    X = ns.nodes.Input(n_in, traces=True, tc_trace=20.0)
    Ae = ns.nodes.DiehlAndCookNodes(n, traces=True, rest=-65.0, reset=-60.0, thresh=-52.0, refrac=5, tc_decay=100.0,
                                    tc_trace=20.0, theta_plus=0.05, tc_theta_decay=1e7)
    Ai = ns.nodes.LIFNodes(n, traces=False, rest=-60.0, reset=-45.0, thresh=-40.0, tc_decay=10.0, refrac=2, tc_trace=20.0)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    net.add_layer(X, "X"); net.add_layer(Ae, "Ae"); net.add_layer(Ai, "Ai")
    w = 0.3 * torch.rand(n_in, n, generator=g)
    xw = ns.topology.MulticompartmentConnection(
        source=X, target=Ae, device="cpu",
        pipeline=[F.Weight(name="w", value=w, norm=78.4, norm_frequency=freq, learning_rule=ML.PostPre, nu=(1e-4, 1e-2),
                           range=[0.0, 1.0])])
    ei = ns.topology.MulticompartmentConnection(source=Ae, target=Ai, device="cpu",
                                                pipeline=[F.Weight(name="ei", value=22.5 * torch.eye(n), range=[0.0, 22.5])])
    ie = ns.topology.MulticompartmentConnection(source=Ai, target=Ae, device="cpu",
                                                pipeline=[F.Weight(name="ie", value=-120.0 * (torch.ones(n, n) - torch.eye(n)),
                                                                   range=[-120.0, 0.0])])
    net.add_connection(xw, "X", "Ae"); net.add_connection(ei, "Ae", "Ai"); net.add_connection(ie, "Ai", "Ae")
    x = (torch.rand(T, B, n_in, generator=g) < 0.02 + 0.06 * torch.rand(1, B, n_in, generator=g)).to(torch.uint8)
    return net, x
