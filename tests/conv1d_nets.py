"""Networks with a Conv1dConnection, shared by tests/test_conv1d.py (CPU: oracle, emulated kernel, stored live-reference
results) and tests/test_gpu_conv1d.py (the CUDA library).  ``ns`` is a ``cases.namespace``: the same builder makes the
reference's network and ours, with seeded weights passed as ``w=`` / ``b=``."""
from __future__ import annotations

import torch

RULES = ["PostPre", "WeightDependentPostPre", "Hebbian"]
# name -> builder keyword arguments of example_net (key "example"), multi_net or (key "wide") wide_net
LIVE_CASES = {
    "example_b1": dict(example=True),                                    # conv1d_MNIST's network, short window
    **{f"c2_{r}": dict(rule=r) for r in RULES},                         # Cin = 2, kernel 4, stride 2, padding 1, B = 4
    "c2_NoOp": dict(rule="NoOp", weight_decay=1e-2),
    "c2_mean": dict(rule="PostPre", reduction="mean"),
    "c2_nolearn": dict(rule="PostPre", learning=False),
    "c2_bias": dict(rule="Hebbian", bias=True),
    "c2_zero_row": dict(rule="NoOp", learning=False, zero_row=True),    # normalize over a filter that sums to zero
    "wide_k40": dict(wide=True),                                         # kernel longer than 32 taps
}

TILE, CONV_STAGE_WORDS, CONV_STAGE_TAPS = 32, 4096, 4096


def example_net(ns, B: int = 1, T: int = 20, L_in: int = 784, rate: float = 0.05, learning: bool = True, rule: str = "PostPre",
                one_spike: bool = False, seed: int = 5, **_):
    """reference examples/mnist/conv1d_MNIST.py: Input [1, L_in] -> Conv1dConnection (kernel 56, stride 28, 25 filters,
    PostPre nu (1e-4, 1e-2), norm 0.4 * 56, wmax 1) -> DiehlAndCookNodes [25, (L_in - 56) / 28 + 1], plus the recurrent
    inhibition (-100 between different filters at the same position).  ``one_spike`` is off by default: the reference
    draws its winner with torch.multinomial.  Returns (net, inputs, T); inputs["X"] is [2 windows, T, B, 1, L_in]."""
    g = torch.Generator().manual_seed(seed)
    k, s, F_ = 56, 28, 25
    c = (L_in - k) // s + 1
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(n=L_in, shape=(1, L_in), traces=True)
    Y = ns.nodes.DiehlAndCookNodes(n=F_ * c, shape=(F_, c), traces=True, one_spike=one_spike)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    conv = ns.topology.Conv1dConnection(X, Y, kernel_size=k, stride=s, update_rule=getattr(ns.learning, rule), norm=0.4 * k,
                                        nu=[1e-4, 1e-2], wmax=1.0, reduction=None if B == 1 else torch.sum,
                                        w=torch.rand(F_, 1, k, generator=g))
    w = torch.zeros(F_, c, F_, c)
    for f1 in range(F_):
        for f2 in range(F_):
            if f1 != f2:
                for i in range(c):
                    w[f1, i, f2, i] = -100.0
    net.add_connection(conv, "X", "Y")
    net.add_connection(ns.topology.Connection(Y, Y, w=w.view(Y.n, Y.n)), "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 1, L_in, generator=g) < rate).to(torch.uint8)
    return net, {"X": x}, T


def multi_net(ns, rule: str = "PostPre", B: int = 4, T: int = 24, learning: bool = True, weight_decay: float = 0.0,
              reduction: str = "sum", bias: bool = False, zero_row: bool = False, cin: int = 2, seed: int = 11, **_):
    """Input [cin, 20] -> Conv1dConnection (3 filters, kernel 4, stride 2, padding 1, w in [0, 1], norm) -> LIFNodes
    [3, 10] -> dense Connection -> LIFNodes(6).  ``bias``: a non-zero b; ``zero_row``: one (out, in) filter of w is zero
    (normalize turns it into NaN)."""
    g = torch.Generator().manual_seed(seed + (RULES.index(rule) if rule in RULES else 7))
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=[cin, 20], traces=True)
    Y = ns.nodes.LIFNodes(shape=[3, 10], traces=True, thresh=-60.0, refrac=2)
    Z = ns.nodes.LIFNodes(6, traces=True, thresh=-62.0)
    for name, layer in (("X", X), ("Y", Y), ("Z", Z)):
        net.add_layer(layer, name)
    w = 0.5 * torch.rand(3, cin, 4, generator=g)
    if zero_row:
        w[1, 0].zero_()
    kw = dict(nu=(0.02, 0.05), wmin=0.0, wmax=1.0, norm=2.0, reduction=torch.mean if reduction == "mean" else torch.sum,
              update_rule=getattr(ns.learning, rule), w=w)
    if rule == "NoOp":
        kw["weight_decay"] = weight_decay
    if bias:
        kw["b"] = torch.rand(3, generator=g)
    conv = ns.topology.Conv1dConnection(X, Y, kernel_size=4, stride=2, padding=1, **kw)
    net.add_connection(conv, "X", "Y")
    net.add_connection(ns.topology.Connection(Y, Z, w=0.5 * torch.rand(Y.n, 6, generator=g)), "Y", "Z")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    net.add_monitor(ns.monitors.Monitor(Z, ["s"], time=T), "Zs")
    x = (torch.rand(2, T, B, cin, 20, generator=g) < 0.3).to(torch.uint8)
    return net, {"X": x}, T


def wide_net(ns, B: int = 3, T: int = 12, rule: str = "PostPre", seed: int = 17, **_):
    """Input [3, 90] -> Conv1dConnection (4 filters, kernel 40 > 32, stride 3, padding 2, PostPre, norm) -> LIFNodes
    [4, 19].  19 neurons per filter: the 32-neuron tiles cross filters."""
    g = torch.Generator().manual_seed(seed)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    X = ns.nodes.Input(shape=[3, 90], traces=True)
    Y = ns.nodes.LIFNodes(shape=[4, 19], traces=True, thresh=-58.0)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    conv = ns.topology.Conv1dConnection(X, Y, kernel_size=40, stride=3, padding=2, nu=(1e-3, 5e-3), wmin=0.0, wmax=1.0, norm=12.0,
                                        reduction=torch.sum, update_rule=getattr(ns.learning, rule),
                                        w=0.1 * torch.rand(4, 3, 40, generator=g), b=torch.rand(4, generator=g))
    net.add_connection(conv, "X", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 3, 90, generator=g) < 0.2).to(torch.uint8)
    return net, {"X": x}, T


def long_net(ns, B: int = 32, T: int = 250, L_in: int = 4096, rate: float = 0.02, seed: int = 23, **_):
    """The long-sequence network: Input [4, L_in] -> Conv1dConnection (kernel 9, stride 1, padding 4, 32 filters,
    PostPre, w in [0, 1], norm) -> LIFNodes [32, L_in].  Returns (net, inputs, T); inputs["X"] is [1, T, B, 4, L_in]."""
    g = torch.Generator().manual_seed(seed)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    X = ns.nodes.Input(shape=[4, L_in], traces=True)
    Y = ns.nodes.LIFNodes(shape=[32, L_in], traces=True, thresh=-60.0, refrac=2)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    conv = ns.topology.Conv1dConnection(X, Y, kernel_size=9, stride=1, padding=4, nu=(1e-4, 1e-3), wmin=0.0, wmax=1.0,
                                        norm=0.4 * 36, reduction=torch.sum, update_rule=ns.learning.PostPre,
                                        w=torch.rand(32, 4, 9, generator=g))
    net.add_connection(conv, "X", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(1, T, B, 4, L_in, generator=g) < rate).to(torch.uint8)
    return net, {"X": x}, T


def build_case(ns, case: str, **over):
    kw = dict(LIVE_CASES[case], **over)
    if kw.pop("example", False):
        return example_net(ns, **kw)
    if kw.pop("wide", False):
        return wide_net(ns, **kw)
    return multi_net(ns, **kw)


def windows_of(case: str) -> int:
    """A zero filter turns into NaN at the first window's normalize; F.conv1d then makes every output of that filter NaN,
    which the spike gather does only where a tap spiked: that case stops after one window."""
    return 1 if LIVE_CASES.get(case, {}).get("zero_row") else 2


def gather_paths(conn, B: int) -> dict:
    """phase 1's staging of the Conv1dConnection input (the first into its target), for a batch of B <= 32 (one sample
    chunk of B samples on the GPU and under the emulation).  ``st_bits``: the chunk's source bit rows are staged;
    ``st_taps_all`` / ``st_taps_some_off``: every 32-neuron tile stages the taps of its filters / some tile does not."""
    assert B <= 32
    ns, nt = conn.source.n, conn.target.n
    L = nt // conn.out_channels
    K = conn.in_channels * conn.kernel_size
    taps = []
    for tile in range((nt + TILE - 1) // TILE):
        co_base, co_hi = (tile * TILE) // L, min(nt - 1, tile * TILE + TILE - 1) // L
        taps.append((co_hi - co_base + 1) * K <= CONV_STAGE_TAPS)
    return dict(st_bits=B * ((ns + 31) // 32) <= CONV_STAGE_WORDS, st_taps_all=all(taps), st_taps_some_off=not all(taps))


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
