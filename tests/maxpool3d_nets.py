"""Networks with a MaxPoo3dConnection, shared by tests/test_maxpool3d.py (CPU: oracle, emulated kernel, stored
live-reference results) and tests/test_gpu_maxpool3d.py (the CUDA library).  ``ns`` is a ``cases.namespace``: the same
builder makes the reference's network and ours.  Learning is off: the reference's MaxPoo3dConnection fails in the first
update of a learning window (its learning.NoOp.update reads connection.w)."""
from __future__ import annotations

import torch

from maxpool_nets import state  # noqa: F401  (the same state snapshot)

# name -> (kernel_size, stride, padding, dilation, source volume (D, H, W)); every value a (D, H, W) triple or an int
GEOMS = {
    "k2s2": (2, 2, 0, 1, (4, 6, 6)),                          # the usual 2 x 2 x 2 pooling
    "k3s1": (3, 1, 0, 1, (4, 5, 6)),                          # stride < kernel: overlapping windows
    "k3s2p1": (3, 2, 1, 1, (5, 6, 7)),                        # padding on every axis, odd sizes
    "p100": ((3, 2, 2), 2, (1, 0, 0), 1, (5, 6, 6)),          # padding on the depth axis only
    "p010": ((2, 3, 2), 2, (0, 1, 0), 1, (4, 5, 6)),          # ... the height axis only
    "p001": ((2, 2, 3), 2, (0, 0, 1), 1, (4, 6, 5)),          # ... the width axis only
    "d211": (2, 1, 0, (2, 1, 1), (5, 4, 4)),                  # dilation on the depth axis
    "d121": (2, 1, 0, (1, 2, 1), (3, 5, 4)),                  # ... the height axis
    "d112": (2, 1, 0, (1, 1, 2), (3, 4, 5)),                  # ... the width axis
    "k233s2p1d112": ((2, 3, 3), 2, 1, (1, 1, 2), (5, 7, 9)),  # padding with per-axis dilation
    "k123s121": ((1, 2, 3), (1, 2, 1), 0, 1, (3, 6, 7)),      # an anisotropic kernel and stride
}
# (B, channels, decay, geometry)
LIVE_CASES = ["b1_c2_d0.25_k2s2", "b4_c2_d0.25_k3s1", "b1_c1_d0_k3s2p1", "b4_c3_d1_p100", "b4_c2_d0_p010", "b1_c2_d1_p001",
              "b4_c2_d0.25_d211", "b1_c2_d0_d121", "b4_c2_d1_d112", "b2_c3_d0.25_k233s2p1d112", "b4_c2_d0.25_k123s121"]


def parse(case: str):
    b, c, d, g = case.split("_", 3)
    return int(b[1:]), int(c[1:]), float(d[1:]), g


def _triple(x):
    return tuple(x) if isinstance(x, tuple) else (x, x, x)


def pooled_shape(C, vol, geom):
    k, s, p, d, _ = GEOMS[geom]
    k, s, p, d = (_triple(v) for v in (k, s, p, d))
    return (C, *((n + 2 * p[i] - d[i] * (k[i] - 1) - 1) // s[i] + 1 for i, n in enumerate(vol)))


def pool_kwargs(geom):
    k, s, p, d, _ = GEOMS[geom]
    return dict(kernel_size=k, stride=s, padding=p, dilation=d)


def conv_pool_net(ns, case: str, T: int = 24):
    """Input [2, D, H, W] -> Conv3dConnection (C filters, 3 x 3 x 3, padding 1) -> LIFNodes [C, D, H, W] ->
    MaxPoo3dConnection -> LIFNodes [C, Dout, Hout, Wout] (one pooled spike makes it fire) -> dense Connection ->
    LIFNodes(10).  Returns (net, inputs, T)."""
    B, C, decay, geom = parse(case)
    vol = GEOMS[geom][4]
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    out = pooled_shape(C, vol, geom)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(shape=[2, *vol])
    C1 = ns.nodes.LIFNodes(shape=[C, *vol], thresh=-60.0, tc_decay=20.0, refrac=2)
    P = ns.nodes.LIFNodes(shape=list(out), thresh=-64.5, rest=-65.0, reset=-65.0, refrac=1)
    Y = ns.nodes.LIFNodes(10, thresh=-62.0, refrac=2)
    for name, layer in (("X", X), ("C1", C1), ("P", P), ("Y", Y)):
        net.add_layer(layer, name)
    conv = ns.topology.Conv3dConnection(X, C1, kernel_size=3, stride=1, padding=1, w=1.2 * torch.rand(C, 2, 3, 3, 3, generator=g),
                                        b=0.1 * torch.rand(C, generator=g))
    pool = ns.topology.MaxPoo3dConnection(C1, P, decay=decay, **pool_kwargs(geom))
    dense = ns.topology.Connection(P, Y, w=0.08 * torch.rand(P.n, 10, generator=g))
    net.add_connection(conv, "X", "C1")
    net.add_connection(pool, "C1", "P")
    net.add_connection(dense, "P", "Y")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 2, *vol, generator=g) < 0.2).to(torch.uint8)
    return net, {"X": x}, T


def tie_net(ns, B: int = 4, T: int = 24, decay: float = 0.0):
    """Input [3, 4, 4, 4] -> MaxPoo3dConnection (2 x 2 x 2, stride 2) -> LIFNodes [3, 2, 2, 2]: all-zero rates at t = 0,
    and the eight inputs of every window spike equally often in a permuted order, so that the rates tie in most windows
    and the first element of the window in (d, h, w) order decides."""
    g = torch.Generator().manual_seed(78)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(shape=[3, 4, 4, 4])
    P = ns.nodes.LIFNodes(shape=[3, 2, 2, 2], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=0)
    net.add_layer(X, "X"); net.add_layer(P, "P")
    net.add_connection(ns.topology.MaxPoo3dConnection(X, P, kernel_size=2, stride=2, decay=decay), "X", "P")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    base = (torch.rand(T, B, 3, 2, 2, 2, generator=g) < 0.3)
    x = torch.zeros(T, B, 3, 4, 4, 4, dtype=torch.bool)
    for q in range(8):
        dz, dy, dx = q >> 2, (q >> 1) & 1, q & 1
        perm = torch.randperm(T, generator=g) if q else torch.arange(T)
        x[:, :, :, dz::2, dy::2, dx::2] = base[perm]
    x[0] = False
    return net, {"X": x.to(torch.uint8)}, T


def variant_net(ns, B: int = 3, T: int = 14, one_spike: bool = False, target_first: bool = False, decay: float = 0.25):
    """Input [2, 3, 4, 6] -> dense Connection -> source [2, 3, 4, 6] -> MaxPoo3dConnection (3 x 3 x 3, stride 2, padding
    1) -> LIFNodes [2, 2, 2, 3].
      one_spike      the source is DiehlAndCookNodes(one_spike=True): its spikes are final only after the per-sample arg-max,
                     so its rates are written in phase 2
      target_first   the pooled layer is added before its source, so in one-step mode it reads the source's previous spikes
    Returns (net, inputs, T)."""
    g = torch.Generator().manual_seed(93 + 2 * one_spike + target_first)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(shape=[2, 3, 4, 6])
    if one_spike:
        S = ns.nodes.DiehlAndCookNodes(shape=[2, 3, 4, 6], one_spike=True, thresh=-58.0, refrac=1)
    else:
        S = ns.nodes.LIFNodes(shape=[2, 3, 4, 6], thresh=-58.0, refrac=1)
    P = ns.nodes.LIFNodes(shape=[2, 2, 2, 3], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=0)
    for name, layer in ((("X", X), ("P", P), ("S", S)) if target_first else (("X", X), ("S", S), ("P", P))):
        net.add_layer(layer, name)
    net.add_connection(ns.topology.Connection(X, S, w=(1.5 if one_spike else 0.3) * torch.rand(144, 144, generator=g)), "X", "S")
    net.add_connection(ns.topology.MaxPoo3dConnection(S, P, kernel_size=3, stride=2, padding=1, decay=decay), "S", "P")
    net.add_monitor(ns.monitors.Monitor(S, ["s"], time=T), "Ss")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    x = (torch.rand(2, T, B, 2, 3, 4, 6, generator=g) < 0.3).to(torch.uint8)
    return net, {"X": x}, T


def twin_net(ns, three_d: bool, T: int = 20, one_spike: bool = False, decay: float = 0.25):
    """Input [1, H, W] -> dense Connection -> source -> pooling (kernel 2 x 3, stride (2, 1), padding (1, 1)) -> LIFNodes:
    with ``three_d`` the source is [1, 1, H, W] and the pool a MaxPoo3dConnection with kernel (1, 2, 3), otherwise
    [1, H, W] and a MaxPool2dConnection — the same computation, neuron for neuron.  One channel at batch size 1: the
    only degenerate-depth shape the reference's ``fr += s.float().squeeze()`` can add."""
    H, W = 6, 8
    g = torch.Generator().manual_seed(17 + one_spike)
    lead = (1,) if three_d else ()
    net = ns.Network(dt=1.0, batch_size=1, learning=False)
    X = ns.nodes.Input(shape=[1, H, W])
    if one_spike:
        S = ns.nodes.DiehlAndCookNodes(shape=[1, *lead, H, W], one_spike=True, thresh=-58.0, refrac=1)
    else:
        S = ns.nodes.LIFNodes(shape=[1, *lead, H, W], thresh=-58.0, refrac=1)
    Hout, Wout = (H + 2 - 2) // 2 + 1, (W + 2 - 3) // 1 + 1
    P = ns.nodes.LIFNodes(shape=[1, *lead, Hout, Wout], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=0)
    for name, layer in (("X", X), ("S", S), ("P", P)):
        net.add_layer(layer, name)
    net.add_connection(ns.topology.Connection(X, S, w=(1.5 if one_spike else 0.6) * torch.rand(H * W, H * W, generator=g)), "X", "S")
    if three_d:
        pool = ns.topology.MaxPoo3dConnection(S, P, kernel_size=(1, 2, 3), stride=(1, 2, 1), padding=(0, 1, 1), decay=decay)
    else:
        pool = ns.topology.MaxPool2dConnection(S, P, kernel_size=(2, 3), stride=(2, 1), padding=(1, 1), decay=decay)
    net.add_connection(pool, "S", "P")
    net.add_monitor(ns.monitors.Monitor(S, ["s"], time=T), "Ss")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    x = (torch.rand(2, T, 1, 1, H, W, generator=g) < 0.3).to(torch.uint8)
    return net, {"X": x}, T


def bench_net(ns, B: int, T: int = 250, pool: bool = True, seed: int = 0):
    """The benchmark's network (bench_maxpool3d.py): Input [2, 8, 32, 32] Bernoulli(0.1) -> Conv3dConnection (16
    filters, kernel (3, 5, 5)) -> LIFNodes [16, 6, 28, 28] -> MaxPoo3dConnection (kernel 2, stride 2, decay 1) ->
    LIFNodes [16, 3, 14, 14] -> dense Connection -> LIFNodes(10); without ``pool`` the convolution's layer feeds the dense
    Connection directly.  Returns (net, inputs, T) with inputs["X"] of [2 windows, T, B, 2, 8, 32, 32]."""
    g = torch.Generator().manual_seed(seed)
    w_conv = 0.5 * torch.rand(16, 2, 3, 5, 5, generator=g)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(shape=[2, 8, 32, 32])
    C1 = ns.nodes.LIFNodes(shape=[16, 6, 28, 28], thresh=-60.0, refrac=2)
    Y = ns.nodes.LIFNodes(10, thresh=-62.0, refrac=2)
    net.add_layer(X, "X"); net.add_layer(C1, "C1")
    net.add_connection(ns.topology.Conv3dConnection(X, C1, kernel_size=(3, 5, 5), w=w_conv, b=torch.zeros(16)), "X", "C1")
    last, name = C1, "C1"
    if pool:
        P = ns.nodes.LIFNodes(shape=[16, 3, 14, 14], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=1)
        net.add_layer(P, "P")
        net.add_connection(ns.topology.MaxPoo3dConnection(C1, P, kernel_size=2, stride=2, decay=1.0), "C1", "P")
        last, name = P, "P"
        net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    net.add_layer(Y, "Y")
    net.add_connection(ns.topology.Connection(last, Y, w=0.002 * torch.rand(last.n, 10, generator=g)), name, "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 2, 8, 32, 32, generator=g) < 0.1).to(torch.uint8)
    return net, {"X": x}, T


def run_two_windows(net, inputs, T, reset: bool = True, **kw):
    """maxpool_nets.run_two_windows for 3-D inputs: a [2 windows, T, B, C, D, H, W] input gives each window its own
    spikes, any other one is run in both windows."""
    states = []
    for w in range(2):
        net.run(inputs={k: (v[w] if v.dim() == 7 else v).clone() for k, v in inputs.items()}, time=T, **kw)
        states.append(state(net))
        if w == 0 and reset:
            net.reset_state_variables()
    return states


def one_spike_net(ns, B: int = 3, T: int = 20, decay: float = 0.25):
    """Input [2, 3, 4, 6] -> Connection (20 * identity) -> DiehlAndCookNodes(one_spike) [2, 3, 4, 6] ->
    MaxPoo3dConnection (2 x 2 x 3, stride (1, 2, 3), padding (1, 0, 1)) -> LIFNodes [2, 4, 2, 2].  At most one input
    element of a sample spikes per step, and only its own source neuron can cross threshold: the one_spike winner is
    the only candidate, so the reference's torch.multinomial draw is deterministic.  The source's final spikes, and so
    the rates it feeds, are written in phase 2 of the window kernel."""
    g = torch.Generator().manual_seed(61)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(shape=[2, 3, 4, 6])
    S = ns.nodes.DiehlAndCookNodes(shape=[2, 3, 4, 6], one_spike=True, thresh=-58.0, refrac=1)
    P = ns.nodes.LIFNodes(shape=[2, 4, 2, 2], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=0)
    for name, layer in (("X", X), ("S", S), ("P", P)):
        net.add_layer(layer, name)
    net.add_connection(ns.topology.Connection(X, S, w=20.0 * torch.eye(144)), "X", "S")
    net.add_connection(ns.topology.MaxPoo3dConnection(S, P, kernel_size=(2, 2, 3), stride=(1, 2, 3), padding=(1, 0, 1), decay=decay),
                       "S", "P")
    net.add_monitor(ns.monitors.Monitor(S, ["s"], time=T), "Ss")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "Ps")
    x = torch.zeros(2, T, B, 144, dtype=torch.uint8)
    idx = torch.randint(0, 144, (2, T, B, 1), generator=g)
    x.scatter_(3, idx, (torch.rand(2, T, B, 1, generator=g) < 0.8).to(torch.uint8))
    return net, {"X": x.view(2, T, B, 2, 3, 4, 6)}, T
