"""Networks with MulticompartmentConnection feature pipelines (Probability / Mask / Intensity besides the Weight), shared by
tests/test_mcc_features.py (CPU: oracle, emulated kernel, stored live-reference results) and tests/test_gpu_mcc_features.py
(the CUDA library).  ``ns`` is a ``cases.namespace``: the same builder makes the reference's network and ours."""
from __future__ import annotations

import importlib

import torch

SEED = 20261015          # the window's draw seed (Network.run(one_spike_seed=...))
LIVE_CASES = ["prob_b1", "prob_b4", "mask_b1", "mask_b4", "int_mask", "mask_int", "reservoir"]


def features(ns):
    pkg = "bindsnet" if ns.kind == "reference" else "bindsnet_b200"
    return importlib.import_module(pkg + ".network.topology_features"), importlib.import_module(pkg + ".learning.MCC_learning")


def _mcc(ns, src, tgt, kinds, g, w, learn=False, p=None, m=None, i=None, tag=""):
    F, ML = features(ns)
    n = (src.n, tgt.n)
    make = {
        "P": lambda: F.Probability(name=tag + "p", value=p if p is not None else torch.rand(*n, generator=g)),
        "M": lambda: F.Mask(name=tag + "m", value=m if m is not None else torch.rand(*n, generator=g) < 0.6),
        "I": lambda: F.Intensity(name=tag + "i", value=i if i is not None else 2.0 * torch.rand(*n, generator=g) - 1.0),
        "W": lambda: F.Weight(name=tag + "w", value=w, range=[-20.0, 20.0],
                              **(dict(learning_rule=ML.PostPre, nu=(1e-3, 2e-3)) if learn else {})),
    }
    return ns.topology.MulticompartmentConnection(source=src, target=tgt, device="cpu", pipeline=[make[k]() for k in kinds])


def live_net(ns, case: str):
    """Input(40) -> MCC -> LIFNodes(30) and a recurrent MCC on the LIF layer.
      prob_b1 / prob_b4   [Probability, Weight] both ways, MCC_learning.PostPre on the input Weight, B = 1 / 4
      mask_b1 / mask_b4   [Weight, Mask] on the input (PostPre), [Probability, Weight] recurrent
      int_mask / mask_int [Intensity, Weight, Mask] / [Mask, Intensity, Weight] (same values, two orders), static
      reservoir           MCC_reservoir.py scaled down: Input(100) -> LIFNodes(80, scalar thresh), sign weights, B = 1
    Returns (net, inputs, T)."""
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    B = {"prob_b1": 1, "mask_b1": 1, "reservoir": 1}.get(case, 4)
    T = 40
    if case == "reservoir":
        n_in, n = 100, 80
        X = ns.nodes.Input(n_in, traces=True)
        Y = ns.nodes.LIFNodes(n, thresh=-52.0, traces=True)
    else:
        n_in, n = 40, 30
        X = ns.nodes.Input(n_in, traces=True)
        Y = ns.nodes.LIFNodes(n, traces=True, thresh=-58.0, tc_decay=30.0, refrac=3)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    if case == "reservoir":
        w1 = torch.sign(torch.randint(-1, 2, (n_in, n), generator=g)).float() * 2.0
        w2 = torch.sign(torch.randint(-1, 2, (n, n), generator=g)).float()
        xy = _mcc(ns, X, Y, "PW", g, w1, tag="in_")
        yy = _mcc(ns, Y, Y, "PW", g, w2, tag="rec_")
        rate = 0.2
    else:
        w1 = 4.0 * torch.rand(n_in, n, generator=g)
        w2 = -2.0 * torch.rand(n, n, generator=g)
        if case.startswith("prob"):
            xy = _mcc(ns, X, Y, "PW", g, w1, learn=True, tag="in_")
        elif case.startswith("mask"):
            xy = _mcc(ns, X, Y, "WM", g, w1, learn=True, tag="in_")
        else:
            m = torch.rand(n_in, n, generator=g) < 0.7
            i = 2.0 * torch.rand(n_in, n, generator=g) - 1.0
            xy = _mcc(ns, X, Y, "IWM" if case == "int_mask" else "MIW", g, 3.0 * w1, m=m, i=i, tag="in_")
        yy = _mcc(ns, Y, Y, "PW", g, w2, tag="rec_")
        rate = 0.25
    net.add_connection(xy, "X", "Y")
    net.add_connection(yy, "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(T, B, n_in, generator=g) < rate).to(torch.uint8)
    return net, {"X": x}, T


def weights(net) -> dict:
    out = {}
    for (s, t), c in net.connections.items():
        w = [f for f in c.pipeline if type(f).__name__ == "Weight"][0].value
        out[f"{s}{t}/w"] = w.detach().clone().cpu()
    return out


def live_state(net) -> dict:
    out = {"Ys": net.monitors["Ys"].get("s").to(torch.uint8).cpu()}
    for l in ("X", "Y"):
        out[f"{l}/x"] = net.layers[l].x.detach().clone().cpu()
    out["Y/v"] = net.layers["Y"].v.detach().clone().cpu()
    out["Y/refrac_count"] = net.layers["Y"].refrac_count.detach().clone().cpu()
    out.update(weights(net))
    return out


def patch_reference_probability(net, seed: int):
    """Make the reference's Probability features draw with snn_synapse_draw instead of torch.bernoulli: each feature
    counts its own compute() calls (one per step) and knows its connection's position in the network."""
    import numpy as np

    import feature_oracle

    for c, conn in enumerate(net.connections.values()):
        for f in conn.pipeline:
            if type(f).__name__ == "Probability":
                f._draw = [c, 0]

                def compute(conn_spikes, f=f):   # topology_features.py:425-429 with the shared draw
                    c_, t_ = f._draw
                    f._draw[1] += 1
                    mask = feature_oracle.transmit_matrix(f.value.detach().cpu().numpy(), seed, t_, c_)
                    return conn_spikes * torch.from_numpy(np.ascontiguousarray(mask)).to(conn_spikes.device)

                f.compute = compute


def snapshot(net, T) -> dict:
    out = {}
    for lname, layer in net.layers.items():
        Bz = layer.s.shape[0]
        out[f"L/{lname}/s"] = layer.s.reshape(Bz, -1).to(torch.uint8).cpu().numpy()
        for var in ("v", "refrac_count", "x"):
            val = getattr(layer, var, None)
            if isinstance(val, torch.Tensor) and val.numel() > 0:
                out[f"L/{lname}/{var}"] = val.detach().reshape(Bz, -1).float().cpu().numpy()
    for k, v in weights(net).items():
        out["C/" + k] = v.numpy()
    if "Ys" in net.monitors:
        out["M/Ys"] = net.monitors["Ys"].get("s").to(torch.uint8).cpu().numpy()
    return out


def wide_net(ns):
    """A source wider than 8192 neurons (more than one group of gather blocks): Input(9000) -> LIFNodes(40) through
    [Probability, Weight, Mask, Intensity], B = 2."""
    g = torch.Generator().manual_seed(31)
    n_in, n, B, T = 9000, 40, 2, 5
    X, Y = ns.nodes.Input(n_in), ns.nodes.LIFNodes(n, thresh=-60.0)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    net.add_connection(_mcc(ns, X, Y, "PWMI", g, 0.5 * torch.rand(n_in, n, generator=g)), "X", "Y")
    x = (torch.rand(T, B, n_in, generator=g) < 0.01).to(torch.uint8)
    x[:, :, 8500:] = (torch.rand(T, B, 500, generator=g) < 0.2).to(torch.uint8)   # spikes past neuron 8192
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    return net, {"X": x}, T


def big_batch_net(ns):
    """B = 520 (> 512: the compute kernels' batch loop), [Probability, Weight] feed-forward and recurrent."""
    g = torch.Generator().manual_seed(32)
    n_in, n, B, T = 40, 33, 520, 4
    X, Y = ns.nodes.Input(n_in, traces=True), ns.nodes.LIFNodes(n, traces=True, thresh=-60.0)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    net.add_connection(_mcc(ns, X, Y, "PW", g, 3.0 * torch.rand(n_in, n, generator=g), learn=True), "X", "Y")
    net.add_connection(_mcc(ns, Y, Y, "WP", g, -torch.rand(n, n, generator=g)), "Y", "Y")
    x = (torch.rand(T, B, n_in, generator=g) < 0.3).to(torch.uint8)
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    return net, {"X": x}, T
