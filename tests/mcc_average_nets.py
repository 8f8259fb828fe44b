"""Networks whose MulticompartmentConnection Weight learns with MCC_learning.PostPre(average_update=k), shared by
tests/test_mcc_average.py (CPU: oracle, emulated kernel, stored live-reference results) and tests/test_gpu_mcc_average.py
(the CUDA library).  ``ns`` is a ``cases.namespace``: the same builder makes the reference's network and ours."""
from __future__ import annotations

import numpy as np
import torch

from mcc_feature_nets import SEED, features, patch_reference_probability, snapshot

# k1 / k3 / k7 (+ "c": continues_update), B = 1 [Weight] (squeeze); b4_sum / b4_mean: B = 4, reduction sum / torch.mean;
# pre_only / post_only: nu = (nu, 0) / (0, nu); decay: decay and range [-0.5, 3]; pw: [Probability, Weight] at B = 4;
# wm: [Weight, Mask] at B = 1; t5: k = 3 over windows of 5 steps
LIVE_CASES = ["k1", "k1c", "k3", "k3c", "k7", "k7c", "b4_sum", "b4_mean", "pre_only", "post_only", "decay", "pw", "wm", "t5"]


def params(case: str) -> dict:
    p = dict(k=3, cont=False, B=1, reduction=None, nu=(4e-2, 3e-2), decay=0.0, rng=[-1.0, 4.0], pipe="W", T=8)
    if case[0] == "k":
        p["k"], p["cont"] = int(case[1]), case.endswith("c")
    p.update({"b4_sum": dict(B=4, cont=True), "b4_mean": dict(B=4, reduction=torch.mean),
              "pre_only": dict(nu=(4e-2, 0.0), cont=True), "post_only": dict(nu=(0.0, 3e-2)),
              "decay": dict(decay=2e-3, rng=[-0.5, 3.0], cont=True), "pw": dict(pipe="PW", B=4, k=7),
              "wm": dict(pipe="WM", cont=True), "t5": dict(T=5)}.get(case, {}))
    return p


def rule_of(conn):
    return [f for f in conn.pipeline if type(f).__name__ == "Weight"][0].learning_rule


def live_net(ns, case: str, B: int = None, n_in: int = 40, n: int = 30):
    """Input(n_in) -> MCC[pipeline, PostPre(average_update=k)] -> LIFNodes(n), plus a static recurrent MCC[Weight] on the
    LIF layer.  Returns (net, inputs for three windows, T)."""
    F, ML = features(ns)
    p = params(case)
    B = B or p["B"]
    g = torch.Generator().manual_seed(sum(map(ord, case)) + B)
    T = p["T"]
    X = ns.nodes.Input(n_in, traces=True)
    Y = ns.nodes.LIFNodes(n, traces=True, thresh=-58.0, tc_decay=30.0, refrac=3)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    kw = dict(learning_rule=ML.PostPre, nu=p["nu"], range=p["rng"], decay=p["decay"])
    if p["reduction"] is not None and ns.kind != "reference":
        kw["reduction"] = p["reduction"]
    w1 = 2.5 * torch.rand(n_in, n, generator=g)
    make = {"P": lambda: F.Probability(name="p", value=0.3 + 0.7 * torch.rand(n_in, n, generator=g)),
            "M": lambda: F.Mask(name="m", value=torch.rand(n_in, n, generator=g) < 0.6),
            "W": lambda: F.Weight(name="w", value=w1, **kw)}
    xy = ns.topology.MulticompartmentConnection(source=X, target=Y, device="cpu", pipeline=[make[k]() for k in p["pipe"]],
                                                average_update=p["k"], continues_update=p["cont"])
    yy = ns.topology.MulticompartmentConnection(source=Y, target=Y, device="cpu",
                                                pipeline=[F.Weight(name="r", value=-1.5 * torch.rand(n, n, generator=g),
                                                                   range=[-2.0, 0.0])])
    if p["reduction"] is not None and ns.kind == "reference":   # (the reference's Weight rejects every reduction=: isinstance
        rule_of(xy).reduction = p["reduction"]                    # (reduction, callable), topology_features.py:117)
    net.add_connection(xy, "X", "Y")
    net.add_connection(yy, "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(3 * T, B, n_in, generator=g) < 0.25).to(torch.uint8)
    return net, {"X": x}, T


def window_inputs(inputs, T, k):
    return {name: v[k * T:(k + 1) * T] for name, v in inputs.items()}


def rule_state(net) -> dict:
    r = rule_of(net.connections[("X", "Y")])
    return {"buf_pre": r.average_buffer_pre.detach().clone().cpu(), "buf_post": r.average_buffer_post.detach().clone().cpu(),
            "idx": torch.tensor([r.average_buffer_index_pre, r.average_buffer_index_post])}


def live_state(net) -> dict:
    out = {"Ys": net.monitors["Ys"].get("s").to(torch.uint8).cpu(), "Y/v": net.layers["Y"].v.detach().clone().cpu()}
    for (s, t), c in net.connections.items():
        out[f"{s}{t}/w"] = [f for f in c.pipeline if type(f).__name__ == "Weight"][0].value.detach().clone().cpu()
    out.update(rule_state(net))
    return out


def run_windows(net, inputs, T, reference=False, one_step=False) -> dict:
    """Window 0 learning, reset_state_variables, window 1 with learning off, window 2 learning; the draws of window k use
    seed SEED + k (the reference's Probability patched to match).  Returns the live state after windows 0 and 2."""
    out = {}
    for k in range(3):
        net.learning = k != 1
        if reference:
            patch_reference_probability(net, SEED + k)
            net.run(inputs=window_inputs(inputs, T, k), time=T)
        else:
            net.run(inputs=window_inputs(inputs, T, k), time=T, one_spike_seed=SEED + k, one_step=one_step)
        if k != 1:
            out.update({f"{k}/{name}": v for name, v in live_state(net).items()})
        if k == 0:
            net.reset_state_variables()
    return out


def full_snapshot(net, T) -> dict:
    """fn.snapshot plus the averaging state, as numpy arrays (for bit-for-bit comparisons)."""
    out = snapshot(net, T)
    r = rule_of(net.connections[("X", "Y")])
    for name in ("average_buffer_pre", "average_buffer_post", "_avg_rows", "_avg_cols"):
        out[f"R/{name}"] = getattr(r, name).detach().cpu().numpy()
    out["R/idx"] = np.array([r.average_buffer_index_pre, r.average_buffer_index_post])
    return out
