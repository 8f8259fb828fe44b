"""Networks with a LocalConnection2D, shared by tests/test_local2d.py (CPU: oracle, emulated kernel, stored live-reference
results) and tests/test_gpu_local2d.py (the CUDA library).  ``ns`` is a ``cases.namespace``: the same builder makes the
reference's network and ours.  The reference's constructor refuses ``w=`` (it reads an attribute it never sets), so the
weights are drawn by the constructor and then overwritten in place with seeded values, identically on both sides."""
from __future__ import annotations

import torch

RULES = ["PostPre", "WeightDependentPostPre", "Hebbian", "NoOp"]
# name -> builder keyword arguments of multi_net
LIVE_CASES = {
    "example_b1": None,                                            # the loc2d_mnist network, short window
    **{f"c2_{r}": dict(rule=r) for r in RULES},                   # Cin = 2, rectangular geometry, B = 4, reduction=sum
    "c2_nolearn": dict(rule="PostPre", learning=False),
    "c2_zero_row": dict(rule="NoOp", learning=False, zero_row=True),   # normalize over a row that sums to zero
}


def _set_w(conn, g, scale=1.0):
    with torch.no_grad():
        conn.w.copy_(scale * torch.rand(conn.w.shape, generator=g))


def example_net(ns, B: int = 1, T: int = 40, H: int = 20, W: int = 20, rate: float = 0.15, learning: bool = True, seed: int = 5):
    """reference examples/mnist/loc2d_mnist.py: Input [1, H, W] -> LocalConnection2D (kernel 12, stride 4, 50 filters,
    PostPre nu (1e-4, 1e-2), w in [0, 1], norm 0.2 * 144) -> AdaptiveLIFNodes [50, Hout, Wout], plus the recurrent
    inhibition (-25 between different filters at the same position).  Returns (net, inputs, T); inputs["X"] is
    [2 windows, T, B, 1, H, W] Bernoulli(rate) spikes."""
    g = torch.Generator().manual_seed(seed)
    k, s, F_ = 12, 4, 50
    ho, wo = (H - k) // s + 1, (W - k) // s + 1
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=[1, H, W], traces=True, tc_trace=20)
    Y = ns.nodes.AdaptiveLIFNodes(shape=[F_, ho, wo], traces=True, rest=-65.0, reset=-60.0, thresh=-52.0, refrac=5, tc_trace=20.0,
                                  theta_plus=0.05, tc_theta_decay=1e6)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    lc = ns.topology.LocalConnection2D(X, Y, kernel_size=k, stride=s, n_filters=F_, nu=(1e-4, 1e-2), update_rule=ns.learning.PostPre,
                                       wmin=0.0, wmax=1.0, norm=0.2 * k * k, reduction=None if B == 1 else torch.sum)
    _set_w(lc, g)
    w_inh = torch.zeros(F_, ho, wo, F_, ho, wo)
    for c in range(F_):
        for a in range(ho):
            for b in range(wo):
                w_inh[c, a, b, :, a, b] = -25.0
                w_inh[c, a, b, c, a, b] = 0
    net.add_connection(lc, "X", "Y")
    net.add_connection(ns.topology.Connection(Y, Y, w=w_inh.reshape(Y.n, Y.n)), "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2, T, B, 1, H, W, generator=g) < rate).to(torch.uint8)
    return net, {"X": x}, T


def multi_net(ns, rule: str = "PostPre", B: int = 4, T: int = 24, learning: bool = True, zero_row: bool = False, weight_decay: float = 0.0,
              seed: int = 11):
    """Input [2, 11, 10] -> LocalConnection2D (kernel (3, 4), stride (2, 3): H = 11 is not a multiple of the stride,
    3 filters, reduction=torch.sum, w in [0, 1], norm) -> LIFNodes [3, 5, 3] -> dense Connection -> LIFNodes(6).  ``NoOp``
    runs with weight_decay 0.01.  ``zero_row``: one kernel row of w is zero (normalize turns it into NaN)."""
    g = torch.Generator().manual_seed(seed + RULES.index(rule))
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=[2, 11, 10], traces=True)
    Y = ns.nodes.LIFNodes(shape=[3, 5, 3], traces=True, thresh=-60.0, refrac=2)
    Z = ns.nodes.LIFNodes(6, traces=True, thresh=-62.0)
    for name, layer in (("X", X), ("Y", Y), ("Z", Z)):
        net.add_layer(layer, name)
    kw = dict(nu=(2e-3, 5e-3), wmin=0.0, wmax=1.0, norm=3.0, reduction=torch.sum, update_rule=getattr(ns.learning, rule))
    if rule == "NoOp":
        kw["weight_decay"] = 0.01 if not weight_decay else weight_decay
    lc = ns.topology.LocalConnection2D(X, Y, kernel_size=(3, 4), stride=(2, 3), n_filters=3, **kw)
    _set_w(lc, g, 0.5)
    if zero_row:
        with torch.no_grad():
            lc.w[1, 7].zero_()
    net.add_connection(lc, "X", "Y")
    net.add_connection(ns.topology.Connection(Y, Z, w=0.5 * torch.rand(Y.n, 6, generator=g)), "Y", "Z")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    net.add_monitor(ns.monitors.Monitor(Z, ["s"], time=T), "Zs")
    x = (torch.rand(2, T, B, 2, 11, 10, generator=g) < 0.3).to(torch.uint8)
    return net, {"X": x}, T


def build_case(ns, case: str):
    kw = LIVE_CASES[case]
    return example_net(ns) if kw is None else multi_net(ns, **kw)


def windows_of(case: str) -> int:
    """A zero row turns into NaN at the first window's normalize; the reference's s_unfold * w then makes every input of
    its targets NaN, which the spike gather does not (DESIGN.md section 8): that case stops after one window."""
    return 1 if LIVE_CASES.get(case, {}) and LIVE_CASES[case].get("zero_row") else 2


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
    for (s, t), c in net.connections.items():
        out[f"{s}{t}/w"] = c.w.detach().cpu().clone()
    return out
