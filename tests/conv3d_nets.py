"""Networks with a Conv3dConnection, shared by tests/test_conv3d.py (CPU: oracle, emulated kernel, stored live-reference
results) and tests/test_gpu_conv3d.py (the CUDA library).  ``ns`` is a ``cases.namespace``: the same builder makes the
reference's network and ours, with seeded weights passed as ``w=`` / ``b=``."""
from __future__ import annotations

import torch

# name -> builder keyword arguments of example_net (key "example") or multi_net
LIVE_CASES = {
    "example_b1_nolearn": dict(example=True, learning=False),              # conv3d_MNIST's network, short window
    "example_b1_noop": dict(example=True, rule="NoOp", weight_decay=2e-3),  # learning.NoOp's decay, then the norm
    "c2_nolearn": dict(learning=False),                                     # Cin = 2, anisotropic geometry, B = 4
    "c2_noop": dict(rule="NoOp", weight_decay=1e-2),
    "c2_zero_rate_postpre": dict(rule="PostPre", nu=(0.0, 0.0), weight_decay=1e-2, wmin=0.05, wmax=0.45),
    "c2_zero_rate_wdep": dict(rule="WeightDependentPostPre", nu=(0.0, 0.0), weight_decay=1e-2, wmin=0.05, wmax=0.45),
    "c2_zero_row": dict(learning=False, zero_row=True),                     # normalize over a filter that sums to zero
}

TILE, CONV_STAGE_WORDS, CONV_STAGE_TAPS = 32, 4096, 4096


def example_net(ns, B: int = 1, T: int = 20, rate: float = 0.05, learning: bool = True, rule: str = "PostPre", nu=(1e-4, 1e-2),
                weight_decay: float = 0.0, one_spike: bool = False, seed: int = 5, **_):
    """reference examples/mnist/conv3d_MNIST.py: Input [1, 28, 28, 28] -> Conv3dConnection (kernel 16, stride 4, 25
    filters, norm 0.4 * 16**3, wmax 1) -> DiehlAndCookNodes [25, 4, 4, 4], plus the recurrent inhibition (-100 between
    different filters at the same position).  The input is a seeded Bernoulli(rate) [28, 28] image per step, replicated
    along depth (the example's digit).  ``one_spike`` is off by default: the reference draws its winner with
    torch.multinomial.  Returns (net, inputs, T); inputs["X"] is [2 windows, T, B, 1, 28, 28, 28]."""
    g = torch.Generator().manual_seed(seed)
    k, s, F_ = 16, 4, 25
    c = (28 - k) // s + 1
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(n=28 ** 3, shape=(1, 28, 28, 28), traces=True)
    Y = ns.nodes.DiehlAndCookNodes(n=F_ * c ** 3, shape=(F_, c, c, c), traces=True, one_spike=one_spike)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    kw = dict(nu=list(nu), weight_decay=weight_decay, update_rule=getattr(ns.learning, rule))
    conv = ns.topology.Conv3dConnection(X, Y, kernel_size=k, stride=s, norm=0.4 * k ** 3, wmax=1.0,
                                        w=torch.rand(F_, 1, k, k, k, generator=g), **kw)
    w = torch.zeros(F_, c, c, c, F_, c, c, c)
    for f1 in range(F_):
        for f2 in range(F_):
            if f1 != f2:
                for i in range(c):
                    for j in range(c):
                        for m in range(c):
                            w[f1, i, j, m, f2, i, j, m] = -100.0
    net.add_connection(conv, "X", "Y")
    net.add_connection(ns.topology.Connection(Y, Y, w=w.view(Y.n, Y.n)), "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    img = (torch.rand(2, T, B, 1, 1, 28, 28, generator=g) < rate).to(torch.uint8)
    return net, {"X": img.expand(2, T, B, 1, 28, 28, 28).contiguous()}, T


def multi_net(ns, rule: str = "NoOp", B: int = 4, T: int = 24, learning: bool = True, nu=(0.0, 0.0), weight_decay: float = 0.0,
              wmin: float = -float("inf"), wmax: float = float("inf"), zero_row: bool = False, seed: int = 11, **_):
    """Input [2, 7, 9, 8] -> Conv3dConnection (3 filters, kernel (3, 2, 4), stride (2, 3, 1), padding (1, 0, 2): a
    non-cubic source, H = 9 not a multiple of its stride, a non-zero bias, norm) -> LIFNodes [3, 4, 3, 9] -> dense
    Connection -> LIFNodes(6).  ``zero_row``: one (out, in) filter of w is zero (normalize turns it into NaN)."""
    g = torch.Generator().manual_seed(seed)
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=[2, 7, 9, 8], traces=True)
    Y = ns.nodes.LIFNodes(shape=[3, 4, 3, 9], traces=True, thresh=-60.0, refrac=2)
    Z = ns.nodes.LIFNodes(6, traces=True, thresh=-62.0)
    for name, layer in (("X", X), ("Y", Y), ("Z", Z)):
        net.add_layer(layer, name)
    w = 0.5 * torch.rand(3, 2, 3, 2, 4, generator=g)
    if zero_row:
        w[1, 0].zero_()
    conv = ns.topology.Conv3dConnection(X, Y, kernel_size=(3, 2, 4), stride=(2, 3, 1), padding=(1, 0, 2), nu=list(nu),
                                        weight_decay=weight_decay, update_rule=getattr(ns.learning, rule), norm=5.0,
                                        wmin=wmin, wmax=wmax, reduction=torch.sum, w=w, b=0.2 * torch.rand(3, generator=g))
    net.add_connection(conv, "X", "Y")
    net.add_connection(ns.topology.Connection(Y, Z, w=0.2 * torch.rand(Y.n, 6, generator=g)), "Y", "Z")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    net.add_monitor(ns.monitors.Monitor(Z, ["s"], time=T), "Zs")
    x = (torch.rand(2, T, B, 2, 7, 9, 8, generator=g) < 0.3).to(torch.uint8)
    return net, {"X": x}, T


def wide_net(ns, B: int = 3, T: int = 9, seed: int = 17, **_):
    """Input [3, 6, 5, 40] -> Conv3dConnection (4 filters, kernel (5, 4, 33): kw > 32, stride (1, 1, 2), padding (0, 0,
    1), NoOp decay, norm) -> LIFNodes [4, 2, 2, 5].  20 neurons per filter: the 32-neuron tiles cross filters, and the
    tiles spanning three filters (3 x 1980 taps) cannot stage their taps."""
    g = torch.Generator().manual_seed(seed)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    X = ns.nodes.Input(shape=[3, 6, 5, 40], traces=True)
    Y = ns.nodes.LIFNodes(shape=[4, 2, 2, 5], traces=True, thresh=-58.0)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    conv = ns.topology.Conv3dConnection(X, Y, kernel_size=(5, 4, 33), stride=(1, 1, 2), padding=(0, 0, 1), weight_decay=5e-3, norm=90.0,
                                        w=0.1 * torch.rand(4, 3, 5, 4, 33, generator=g), b=torch.rand(4, generator=g))
    net.add_connection(conv, "X", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 3, 6, 5, 40, generator=g) < 0.2).to(torch.uint8)
    return net, {"X": x}, T


def build_case(ns, case: str, **over):
    kw = dict(LIVE_CASES[case], **over)
    return example_net(ns, **kw) if kw.pop("example", False) else multi_net(ns, **kw)


def windows_of(case: str) -> int:
    """A zero filter turns into NaN at the first window's normalize; F.conv3d then makes every output of that filter NaN,
    which the spike gather does only where a tap spiked: that case stops after one window."""
    return 1 if LIVE_CASES.get(case, {}).get("zero_row") else 2


def gather_paths(conn, B: int) -> dict:
    """phase 1's staging of the Conv3dConnection input (the first into its target), for a batch of B <= 32 (one sample
    chunk of B samples on the GPU and under the emulation).  ``st_bits``: the chunk's source bit rows are staged;
    ``st_taps_all`` / ``st_taps_some_off``: every 32-neuron tile stages the taps of its filters / some tile does not;
    ``tile_crosses_filter``: some tile holds neurons of two filters."""
    assert B <= 32
    ns, nt = conn.source.n, conn.target.n
    L = nt // conn.out_channels
    K = conn.in_channels * conn.kernel_size[0] * conn.kernel_size[1] * conn.kernel_size[2]
    taps, cross = [], False
    for tile in range((nt + TILE - 1) // TILE):
        co_base, co_hi = (tile * TILE) // L, min(nt - 1, tile * TILE + TILE - 1) // L
        taps.append((co_hi - co_base + 1) * K <= CONV_STAGE_TAPS)
        cross |= co_hi > co_base
    return dict(st_bits=B * ((ns + 31) // 32) <= CONV_STAGE_WORDS, st_taps_all=all(taps), st_taps_some_off=not all(taps),
                tile_crosses_filter=cross, kw_over_32=conn.kernel_size[2] > 32)


def run_windows(net, inputs, T, n: int = 2, reset: bool = True, **kw):
    """``n`` windows with reset_state_variables() between them; the state after each."""
    states = []
    for w in range(n):
        net.run(inputs={k: v[w].clone() for k, v in inputs.items()}, time=T, **kw)
        states.append(state(net))
        if w + 1 < n and reset:
            net.reset_state_variables()
    return states


def state(net) -> dict:
    out = {}
    for name in ("Ys", "Zs"):
        if name in net.monitors:
            out[name] = net.monitors[name].get("s").to(torch.uint8).cpu().clone()
    for lname, layer in net.layers.items():
        out[f"{lname}/s"] = layer.s.to(torch.uint8).cpu().clone()
        for var in ("v", "refrac_count", "x", "theta"):
            v = getattr(layer, var, None)
            if isinstance(v, torch.Tensor) and v.numel():
                out[f"{lname}/{var}"] = v.detach().cpu().clone()
    out["XY/w"] = net.connections[("X", "Y")].w.detach().cpu().clone()   # (the other weights never change)
    return out
