"""Networks whose MulticompartmentConnection Weight learns with MCC_learning.MSTDP / MSTDPET, shared by
tests/test_mcc_reward.py (CPU: oracle, emulated kernel, stored live-reference results) and tests/test_gpu_mcc_reward.py
(the CUDA library).  ``ns`` is a ``cases.namespace``: the same builder makes the reference's network and ours."""
from __future__ import annotations

import torch

from mcc_feature_nets import SEED, features, patch_reference_probability, snapshot

LIVE_CASES = ["w_b1", "w_b4", "pw_b4", "wm_et", "decay_range", "decay_range_et"]
# the run kwargs of the two windows: reward changes, a_plus / a_minus as scalars, then as dicts keyed by connection
# (a connection without an entry falls back to the rule's default, network.py:440-461)
WINDOW_KWARGS = [dict(reward=1.0, a_plus=0.8, a_minus=-0.6),
                 dict(reward=-0.5, a_plus={("X", "Y"): 0.5}, a_minus={("Y", "Y"): -2.0})]


def rule_of(conn):
    return [f for f in conn.pipeline if type(f).__name__ == "Weight"][0].learning_rule


def live_net(ns, case: str, T: int = 30):
    """Input(40) -> MCC[pipeline, rule] -> LIFNodes(30) plus a static recurrent MCC[Weight] on the LIF layer.
      w_b1 / w_b4       [Weight] + MSTDP, B = 1 / 4
      pw_b4             [Probability, Weight] + MSTDP, B = 4
      wm_et             [Weight, Mask] + MSTDPET, B = 1
      decay_range(_et)  [Weight] + MSTDP (B = 2) / MSTDPET (B = 1) with decay and range [-0.5, 3]
    Returns (net, inputs, T)."""
    F, ML = features(ns)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    et = case.endswith("et")
    B = 1 if et or case == "w_b1" else (2 if case == "decay_range" else 4)
    n_in, n = 40, 30
    X = ns.nodes.Input(n_in, traces=True)
    Y = ns.nodes.LIFNodes(n, traces=True, thresh=-58.0, tc_decay=30.0, refrac=3)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    rng = [-0.5, 3.0] if case.startswith("decay") else [-1.0, 4.0]
    w1 = 2.5 * torch.rand(n_in, n, generator=g)
    kw = dict(learning_rule=ML.MSTDPET if et else ML.MSTDP, nu=(2e-2, 1e-2), range=rng,
              decay=2e-3 if case.startswith("decay") else 0.0)
    if et:
        kw["nu"] = (0.5, 0.5)
    pipe = {"w_b1": "W", "w_b4": "W", "pw_b4": "PW", "wm_et": "WM", "decay_range": "W", "decay_range_et": "W"}[case]
    make = {"P": lambda: F.Probability(name="p", value=0.3 + 0.7 * torch.rand(n_in, n, generator=g)),
            "M": lambda: F.Mask(name="m", value=torch.rand(n_in, n, generator=g) < 0.6),
            "W": lambda: F.Weight(name="w", value=w1, **kw)}
    xy = ns.topology.MulticompartmentConnection(source=X, target=Y, device="cpu", pipeline=[make[k]() for k in pipe],
                                                tc_plus=15.0, tc_minus=25.0, tc_e_trace=10.0)
    yy = ns.topology.MulticompartmentConnection(source=Y, target=Y, device="cpu",
                                                pipeline=[F.Weight(name="r", value=-1.5 * torch.rand(n, n, generator=g),
                                                                   range=[-2.0, 0.0])])
    net.add_connection(xy, "X", "Y")
    net.add_connection(yy, "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2 * T, B, n_in, generator=g) < 0.25).to(torch.uint8)
    return net, {"X": x}, T


def window_inputs(inputs, T, k):
    return {name: v[k * T:(k + 1) * T] for name, v in inputs.items()}


def rule_state(net) -> dict:
    r = rule_of(net.connections[("X", "Y")])
    out = {"p_plus": r.p_plus.detach().clone().cpu(), "p_minus": r.p_minus.detach().clone().cpu(),
           "eligibility": r.eligibility.detach().clone().cpu()}
    if hasattr(r, "eligibility_trace"):
        out["eligibility_trace"] = r.eligibility_trace.detach().clone().cpu()
    return out


def live_state(net) -> dict:
    out = {"Ys": net.monitors["Ys"].get("s").to(torch.uint8).cpu(),
           "Y/v": net.layers["Y"].v.detach().clone().cpu(), "Y/x": net.layers["Y"].x.detach().clone().cpu()}
    for (s, t), c in net.connections.items():
        out[f"{s}{t}/w"] = [f for f in c.pipeline if type(f).__name__ == "Weight"][0].value.detach().clone().cpu()
    out.update(rule_state(net))
    return out


def run_two_windows(net, inputs, T, case, reference=False, one_step=False) -> dict:
    """Two windows with the run kwargs of WINDOW_KWARGS; the MSTDPET case resets the network in between.  The draws of
    window k use seed SEED + k (the reference's Probability patched to match).  Returns the live state after each."""
    out = {}
    for k in range(2):
        if reference:
            patch_reference_probability(net, SEED + k)
            net.run(inputs=window_inputs(inputs, T, k), time=T, **WINDOW_KWARGS[k])
        else:
            net.run(inputs=window_inputs(inputs, T, k), time=T, one_spike_seed=SEED + k, one_step=one_step, **WINDOW_KWARGS[k])
        out.update({f"{k}/{name}": v for name, v in live_state(net).items()})
        if k == 0 and case == "wm_et":
            net.reset_state_variables()
    return out


def full_snapshot(net, T) -> dict:
    """fn.snapshot plus the rule state, as numpy arrays (for bit-for-bit comparisons)."""
    out = snapshot(net, T)
    for (s, t), c in net.connections.items():
        r = rule_of(c)
        for name in ("p_plus", "p_minus", "eligibility_trace", "_spre", "_spost"):
            v = getattr(r, name, None)
            if isinstance(v, torch.Tensor):
                out[f"R/{s}{t}/{name}"] = v.detach().cpu().numpy()
    return out


def reservoir_readout(ns, rule: str, B: int, T: int, n_res: int = 4000, n_in: int = 784, mcc: bool = True, seed: int = 0,
                      device: str = "cpu"):
    """The MCC_reservoir topology (n_in -> n_res LIF, recurrent [Probability, Weight]) with a 10-neuron LIF readout whose
    input learns with MSTDP / MSTDPET: ``mcc`` selects MCC[Weight] + MCC_learning.<rule> or Connection + learning.<rule>
    with the same weights, rates, bounds and decay.  Returns (net, input spikes [T, B, n_in])."""
    F, ML = features(ns)
    g = torch.Generator().manual_seed(seed)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    X = ns.nodes.Input(n_in)
    R = ns.nodes.LIFNodes(n_res, thresh=-52.0, traces=True)
    O = ns.nodes.LIFNodes(10, thresh=-55.0, traces=True)
    net.add_layer(X, "X"); net.add_layer(R, "R"); net.add_layer(O, "O")
    w_in = torch.sign(torch.randint(-1, 2, (n_in, n_res), generator=g)).float() * 2.0
    p_in = torch.rand(n_in, n_res, generator=g)
    w_rec = torch.sign(torch.randint(-1, 2, (n_res, n_res), generator=g)).float()
    p_rec = 0.1 * torch.rand(n_res, n_res, generator=g)
    w_out = 0.5 * torch.rand(n_res, 10, generator=g)
    net.add_connection(ns.topology.MulticompartmentConnection(
        source=X, target=R, device=device, pipeline=[F.Probability("p_in", p_in), F.Weight("w_in", w_in, range=[-2.0, 2.0])]), "X", "R")
    net.add_connection(ns.topology.MulticompartmentConnection(
        source=R, target=R, device=device, pipeline=[F.Probability("p_rec", p_rec), F.Weight("w_rec", w_rec, range=[-1.0, 1.0])]), "R", "R")
    nu = (1e-3, 1e-3)
    if mcc:
        readout = ns.topology.MulticompartmentConnection(
            source=R, target=O, device=device,
            pipeline=[F.Weight("w_out", w_out, range=[-1.0, 1.0], learning_rule=getattr(ML, rule), nu=nu,
                               reduction=torch.sum, decay=1e-4)])
    else:
        L = __import__(("bindsnet" if ns.kind == "reference" else "bindsnet_b200") + ".learning", fromlist=[rule])
        readout = ns.topology.Connection(R, O, w=w_out, update_rule=getattr(L, rule), nu=nu, reduction=torch.sum,
                                         weight_decay=1e-4, wmin=-1.0, wmax=1.0)
    net.add_connection(readout, "R", "O")
    x = (torch.rand(T, B, n_in, generator=g) < 0.05).to(torch.uint8)
    return net, x
