"""Networks with a MaxPool2dConnection, shared by tests/test_maxpool.py (CPU: oracle, emulated kernel, stored
live-reference results) and tests/test_gpu_maxpool.py (the CUDA library).  ``ns`` is a ``cases.namespace``: the same
builder makes the reference's network and ours.  Learning is off: the reference's MaxPool2dConnection fails in the
first update of a learning window (its learning.NoOp.update reads connection.w), so the Conv2dConnection's PostPre rule
is attached but does not run."""
from __future__ import annotations

import torch

# name -> (kernel_size, stride, padding, dilation)
GEOMS = {
    "k2s2": (2, 2, 0, 1),        # the usual 2 x 2 pooling
    "k3s1": (3, 1, 0, 1),        # stride < kernel: overlapping windows
    "k3s2p1": (3, 2, 1, 1),      # padding, odd sizes
    "k2s1d2": (2, 1, 0, 2),      # dilation
    "k3s2p1d2": (3, 2, 1, 2),    # padding and dilation
    "k23s12p10": ((2, 3), (1, 2), (1, 0), 1),   # rectangular
}
# (B, decay, geometry)
LIVE_CASES = ["b1_d0.25_k2s2", "b4_d0.25_k3s1", "b1_d0_k3s2p1", "b4_d1_k2s1d2", "b4_d0_k3s2p1d2", "b1_d1_k23s12p10", "b4_d0.25_k23s12p10"]


def parse(case: str):
    b, d, g = case.split("_", 2)
    return int(b[1:]), float(d[1:]), g


def _pair(x):
    return tuple(x) if isinstance(x, tuple) else (x, x)


def pooled_shape(C, H, W, geom):
    k, s, p, d = (_pair(v) for v in GEOMS[geom])
    return C, (H + 2 * p[0] - d[0] * (k[0] - 1) - 1) // s[0] + 1, (W + 2 * p[1] - d[1] * (k[1] - 1) - 1) // s[1] + 1


def conv_pool_net(ns, case: str, H: int = 9, W: int = 11, T: int = 30, C: int = 4):
    """Input [2, H, W] -> Conv2dConnection (3 x 3, padding 1) + PostPre -> LIFNodes [C, H, W] -> MaxPool2dConnection ->
    LIFNodes [C, Hout, Wout] (one pooled spike makes it fire) -> dense Connection -> LIFNodes(10).  Returns
    (net, inputs, T)."""
    B, decay, geom = parse(case)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    k, s, p, d = GEOMS[geom]
    out = pooled_shape(C, H, W, geom)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(shape=[2, H, W], traces=True)
    C1 = ns.nodes.LIFNodes(shape=[C, H, W], traces=True, thresh=-60.0, tc_decay=20.0, refrac=2)
    P = ns.nodes.LIFNodes(shape=list(out), thresh=-64.5, rest=-65.0, reset=-65.0, refrac=1)
    Y = ns.nodes.LIFNodes(10, thresh=-62.0, refrac=2)
    for name, layer in (("X", X), ("C1", C1), ("P", P), ("Y", Y)):
        net.add_layer(layer, name)
    conv = ns.topology.Conv2dConnection(X, C1, kernel_size=3, stride=1, padding=1, update_rule=ns.learning.PostPre, nu=(1e-3, 2e-3),
                                        w=3.5 * torch.rand(C, 2, 3, 3, generator=g), wmin=0.0, wmax=4.0)
    pool = ns.topology.MaxPool2dConnection(C1, P, kernel_size=k, stride=s, padding=p, dilation=d, decay=decay)
    dense = ns.topology.Connection(P, Y, w=0.04 * torch.rand(P.n, 10, generator=g))
    net.add_connection(conv, "X", "C1")
    net.add_connection(pool, "C1", "P")
    net.add_connection(dense, "P", "Y")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 2, H, W, generator=g) < 0.2).to(torch.uint8)
    return net, {"X": x}, T


def tie_net(ns, B: int = 4, T: int = 24, decay: float = 0.0):
    """Input [3, 8, 8] -> MaxPool2dConnection (2 x 2, stride 2) -> LIFNodes [3, 4, 4]: all-zero rates at t = 0, and the
    four inputs of every window spike equally often in a permuted order, so that the rates tie in most windows and the
    first element of the window decides."""
    g = torch.Generator().manual_seed(77)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(shape=[3, 8, 8])
    P = ns.nodes.LIFNodes(shape=[3, 4, 4], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=0)
    net.add_layer(X, "X"); net.add_layer(P, "P")
    net.add_connection(ns.topology.MaxPool2dConnection(X, P, kernel_size=2, stride=2, decay=decay), "X", "P")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    base = (torch.rand(T, B, 3, 4, 4, generator=g) < 0.3)
    x = torch.zeros(T, B, 3, 8, 8, dtype=torch.bool)
    for q, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        perm = torch.randperm(T, generator=g) if q else torch.arange(T)
        x[:, :, :, dy::2, dx::2] = base[perm]
    x[0] = False
    return net, {"X": x.to(torch.uint8)}, T


def run_two_windows(net, inputs, T, reset: bool = True, **kw):
    """Two windows, with reset_state_variables() between them unless ``reset`` is False (the second window's rates then
    start from the first window's and fold in its last spikes); the state after each."""
    states = []
    for w in range(2):
        # a copy per window: the reference's Input aliases its input as s, and reset_state_variables() zeroes s in place
        net.run(inputs={k: (v[w] if v.dim() == 6 else v).clone() for k, v in inputs.items()}, time=T, **kw)
        states.append(state(net))
        if w == 0 and reset:
            net.reset_state_variables()
    return states


def state(net) -> dict:
    out = {}
    for name in ("Ps", "Ys", "Ss"):
        if name in net.monitors:
            out[name] = net.monitors[name].get("s").to(torch.uint8).cpu().clone()
    for lname, layer in net.layers.items():
        out[f"{lname}/s"] = layer.s.to(torch.uint8).cpu().clone()
        for var in ("v", "refrac_count", "x"):
            v = getattr(layer, var, None)
            if isinstance(v, torch.Tensor) and v.numel():
                out[f"{lname}/{var}"] = v.detach().cpu().clone()
    for (s, t), c in net.connections.items():
        if hasattr(c, "firing_rates"):
            out[f"{s}{t}/fr"] = c.firing_rates.detach().cpu().clone()
        else:
            out[f"{s}{t}/w"] = c.w.detach().cpu().clone()
    return out


def c4_pool_net(ns, B: int = 128, T: int = 40):
    """BASELINE config 4's convolution followed by pooling: Input [1, 32, 32] -> Conv2dConnection (5 x 5) -> LIFNodes
    [16, 28, 28] -> MaxPool2dConnection (2 x 2, decay 1, as ann_to_snn builds it) -> LIFNodes [16, 14, 14] -> dense
    Connection -> LIFNodes(10); Bernoulli(0.1) input."""
    g = torch.Generator().manual_seed(404)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(shape=[1, 32, 32])
    C1 = ns.nodes.LIFNodes(shape=[16, 28, 28], thresh=-60.0, refrac=2)
    P = ns.nodes.LIFNodes(shape=[16, 14, 14], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=1)
    Y = ns.nodes.LIFNodes(10, thresh=-62.0, refrac=2)
    for name, layer in (("X", X), ("C1", C1), ("P", P), ("Y", Y)):
        net.add_layer(layer, name)
    net.add_connection(ns.topology.Conv2dConnection(X, C1, kernel_size=5, w=0.9 * torch.rand(16, 1, 5, 5, generator=g)), "X", "C1")
    net.add_connection(ns.topology.MaxPool2dConnection(C1, P, kernel_size=2, stride=2, decay=1.0), "C1", "P")
    net.add_connection(ns.topology.Connection(P, Y, w=0.002 * torch.rand(P.n, 10, generator=g)), "P", "Y")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 1, 32, 32, generator=g) < 0.1).to(torch.uint8)
    return net, {"X": x}, T


def variant_net(ns, B: int = 3, T: int = 14, one_spike: bool = False, target_first: bool = False, decay: float = 0.25):
    """Input [2, 6, 8] -> dense Connection -> source [2, 6, 8] -> MaxPool2dConnection (3 x 3, stride 2, padding 1) ->
    LIFNodes [2, 3, 4].
      one_spike      the source is DiehlAndCookNodes(one_spike=True): its spikes are final only after the per-sample arg-max
      target_first   the pooled layer is added before its source, so in one-step mode it reads the source's previous spikes
    Returns (net, inputs, T)."""
    g = torch.Generator().manual_seed(91 + 2 * one_spike + target_first)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(shape=[2, 6, 8])
    if one_spike:
        S = ns.nodes.DiehlAndCookNodes(shape=[2, 6, 8], one_spike=True, thresh=-58.0, refrac=1)
    else:
        S = ns.nodes.LIFNodes(shape=[2, 6, 8], thresh=-58.0, refrac=1)
    P = ns.nodes.LIFNodes(shape=[2, 3, 4], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=0)
    for name, layer in ((("X", X), ("P", P), ("S", S)) if target_first else (("X", X), ("S", S), ("P", P))):
        net.add_layer(layer, name)
    net.add_connection(ns.topology.Connection(X, S, w=(1.5 if one_spike else 0.3) * torch.rand(96, 96, generator=g)), "X", "S")
    net.add_connection(ns.topology.MaxPool2dConnection(S, P, kernel_size=3, stride=2, padding=1, decay=decay), "S", "P")
    net.add_monitor(ns.monitors.Monitor(S, ["s"], time=T), "Ss")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    x = (torch.rand(2, T, B, 2, 6, 8, generator=g) < 0.3).to(torch.uint8)
    return net, {"X": x}, T
