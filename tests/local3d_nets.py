"""Networks with a LocalConnection3D, shared by tests/test_local3d.py (CPU: oracle, emulated kernel, stored live-reference
results) and tests/test_gpu_local3d.py (the CUDA library).  ``ns`` is a ``cases.namespace``: the same builder makes the
reference's network and ours.  The reference's constructor refuses ``w=`` (it reads an attribute it never sets), so the
weights are drawn by the constructor and then overwritten in place with seeded values, identically on both sides."""
from __future__ import annotations

import torch

RULES = ["PostPre", "WeightDependentPostPre", "Hebbian", "NoOp"]
# name -> builder keyword arguments of multi_net
LIVE_CASES = {
    "example_b1": None,                                            # the loc3d_mnist network, short window
    **{f"c2_{r}": dict(rule=r) for r in RULES},                   # Cin = 2, (3, 2, 4) kernel, (2, 1, 3) stride, B = 4
    "c2_nolearn": dict(rule="PostPre", learning=False),
    "c2_mean": dict(rule="PostPre", reduction="mean"),
    "c2_zero_row": dict(rule="NoOp", learning=False, zero_row=True),   # normalize over a row that sums to zero
}


def _set_w(conn, g, scale=1.0):
    with torch.no_grad():
        conn.w.copy_(scale * torch.rand(conn.w.shape, generator=g))


def example_net(ns, B: int = 1, T: int = 30, S: int = 20, rate: float = 0.02, w_scale: float = 0.1, learning: bool = True,
                seed: int = 5, reduction=None):
    """reference examples/mnist/loc3d_mnist.py: Input [1, S, S, S] -> LocalConnection3D (kernel 16, stride 2, 25 filters,
    PostPre nu (1e-4, 1e-2), w in [0, 1], norm 0.2 * 16^3) -> AdaptiveLIFNodes [25, c, c, c], plus the recurrent
    inhibition (-25 between different filters at the same position).  Returns (net, inputs, T); inputs["X"] is
    [2 windows, T, B, 1, S, S, S] Bernoulli(rate) spikes of an [S, S] image replicated along the first spatial axis, as the
    example replicates MNIST.  The first window's weights are drawn in [0, w_scale), so that its targets do not all fire
    at once."""
    g = torch.Generator().manual_seed(seed)
    k, s, F_ = 16, 2, 25
    c = (S - k) // s + 1
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(shape=[1, S, S, S], traces=True)
    Y = ns.nodes.AdaptiveLIFNodes(shape=[F_, c, c, c], traces=True, rest=-65.0, reset=-60.0, thresh=-52.0, refrac=5, tc_trace=20.0,
                                  theta_plus=0.05, tc_theta_decay=1e6)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    if reduction is None and B > 1:
        reduction = torch.sum
    lc = ns.topology.LocalConnection3D(X, Y, kernel_size=k, stride=s, n_filters=F_, nu=(1e-4, 1e-2), update_rule=ns.learning.PostPre,
                                       wmin=0.0, wmax=1.0, norm=0.2 * k ** 3, reduction=reduction)
    _set_w(lc, g, w_scale)
    P = c ** 3
    w_inh = torch.full((F_, P, F_, P), 0.0)
    for p in range(P):
        w_inh[:, p, :, p] = -25.0
        w_inh[torch.arange(F_), p, torch.arange(F_), p] = 0.0
    net.add_connection(lc, "X", "Y")
    net.add_connection(ns.topology.Connection(Y, Y, w=w_inh.reshape(Y.n, Y.n)), "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    img = (torch.rand(2, T, B, 1, 1, S, S, generator=g) < rate).to(torch.uint8)
    return net, {"X": img.repeat(1, 1, 1, 1, S, 1, 1)}, T


def multi_net(ns, rule: str = "PostPre", B: int = 4, T: int = 24, learning: bool = True, zero_row: bool = False, reduction: str = "sum",
              shape=(2, 7, 5, 11), kernel=(3, 2, 4), stride=(2, 1, 3), filters: int = 3, seed: int = 11):
    """Input [2, 7, 5, 11] -> LocalConnection3D (kernel (3, 2, 4), stride (2, 1, 3): D = 11 is not a multiple of the
    stride, 3 filters, w in [0, 1], norm) -> LIFNodes [3, 3, 4, 3] with a low threshold, so that the target spikes inside
    the window -> dense Connection -> LIFNodes(6).  ``NoOp`` runs with weight_decay 0.01.  ``zero_row``: one kernel row of w
    is zero (normalize turns it into NaN)."""
    g = torch.Generator().manual_seed(seed + RULES.index(rule))
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    conv = [(n - k) // s + 1 for n, k, s in zip(shape[1:], kernel, stride)]
    X = ns.nodes.Input(shape=list(shape), traces=True)
    Y = ns.nodes.LIFNodes(shape=[filters, *conv], traces=True, thresh=-60.0, refrac=2)
    Z = ns.nodes.LIFNodes(6, traces=True, thresh=-62.0)
    for name, layer in (("X", X), ("Y", Y), ("Z", Z)):
        net.add_layer(layer, name)
    kw = dict(nu=(2e-3, 5e-3), wmin=0.0, wmax=1.0, norm=3.0, reduction={"sum": torch.sum, "mean": torch.mean}[reduction],
              update_rule=getattr(ns.learning, rule))
    if rule == "NoOp":
        kw["weight_decay"] = 0.01
    lc = ns.topology.LocalConnection3D(X, Y, kernel_size=kernel, stride=stride, n_filters=filters, **kw)
    _set_w(lc, g, 0.5)
    if zero_row:
        with torch.no_grad():
            lc.w[1, 7].zero_()
    net.add_connection(lc, "X", "Y")
    net.add_connection(ns.topology.Connection(Y, Z, w=0.5 * torch.rand(Y.n, 6, generator=g)), "Y", "Z")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    net.add_monitor(ns.monitors.Monitor(Z, ["s"], time=T), "Zs")
    x = (torch.rand(2, T, B, *shape, generator=g) < 0.3).to(torch.uint8)
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


def shrink(flat: dict, seed: int = 3, k: int = 20000) -> dict:
    """The example's 2.76 M weights as what is stored of them: the per-row sums of w viewed as [cin * n, K], and k
    elements at seeded positions."""
    out = {}
    for name, v in flat.items():
        if name.endswith("XY/w") and v.numel() > 10 ** 6:
            rows = v.reshape(-1, v.shape[-1])
            idx = torch.randperm(v.numel(), generator=torch.Generator().manual_seed(seed))[:k]
            out[name.replace("/w", "/wrowsum")] = rows.double().sum(-1).float()
            out[name.replace("/w", "/wpick")] = v.reshape(-1)[idx]
        else:
            out[name] = v
    return out
