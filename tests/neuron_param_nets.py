"""Networks whose LIFNodes / AdaptiveLIFNodes / DiehlAndCookNodes populations carry per-neuron parameter tensors, shared
by tests/test_neuron_params.py (CPU: oracle, emulated kernel, stored live-reference results) and
tests/test_gpu_neuron_params.py (the CUDA library).  ``ns`` is a ``cases.namespace``: the same builder makes the
reference's network and ours."""
from __future__ import annotations

import torch

# case -> (population, batch size, extras)
CASES = {
    "lif_b1":     ("LIFNodes", 1, ""),
    "lif_b4":     ("LIFNodes", 4, ""),
    "dc":         ("DiehlAndCookNodes", 3, ""),
    "alif":       ("AdaptiveLIFNodes", 2, ""),
    "conv_chan":  ("LIFNodes", 2, "conv"),
    "traces":     ("LIFNodes", 3, "traces"),
    "ei":         ("LIFNodes", 2, "ei"),
}
LIVE_CASES = list(CASES)
N_IN, N = 40, 30


def _vec(g, n, lo, hi):
    return lo + (hi - lo) * torch.rand(n, generator=g)


def population(ns, kind: str, n: int, g: torch.Generator, shape=None, traces_additive: bool = False, per_trace: bool = False,
               one_spike: bool = False):
    """A population of ``kind`` whose threshold, rest and membrane time constant (LIF), or threshold, theta increment and
    theta time constant (DC / AdaptiveLIF), are per-neuron tensors; with ``per_trace`` also tc_trace and trace_scale."""
    kw = dict(traces=True, traces_additive=traces_additive, refrac=3)
    kw["shape"] = shape if shape is not None else None
    kw["n"] = None if shape is not None else n
    if per_trace:
        kw.update(tc_trace=_vec(g, n, 5.0, 30.0), trace_scale=_vec(g, n, 0.5, 1.5))
    if kind == "LIFNodes":
        return ns.nodes.LIFNodes(thresh=_vec(g, n, -60.0, -54.0), rest=_vec(g, n, -67.0, -63.0), tc_decay=_vec(g, n, 20.0, 120.0), **kw)
    extra = dict(thresh=_vec(g, n, -58.0, -54.0), theta_plus=_vec(g, n, 0.0, 0.4), tc_theta_decay=_vec(g, n, 50.0, 500.0),
                 tc_decay=30.0)
    if kind == "AdaptiveLIFNodes":
        return ns.nodes.AdaptiveLIFNodes(**extra, **kw)
    return ns.nodes.DiehlAndCookNodes(one_spike=one_spike, **extra, **kw)


def live_net(ns, case: str, T: int = 30):
    """Input(40) -> the case's population (30 neurons) through a PostPre Connection, plus a static recurrent inhibitory
    Connection; case "conv": Input [2, 8, 8] -> Conv2dConnection -> LIFNodes [3, 4, 4] with a per-channel [3, 1, 1]
    threshold; case "ei": a recurrent WeightDependentPostPre E/I Connection with sign bounds per row.  Returns
    (net, inputs, T)."""
    kind, B, extra = CASES[case]
    L = ns.learning
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    if extra == "conv":
        X = ns.nodes.Input(shape=[2, 8, 8], traces=True)
        Y = ns.nodes.LIFNodes(shape=[3, 4, 4], traces=True, refrac=2, thresh=torch.tensor([-60.0, -57.0, -54.0]).view(3, 1, 1),
                              rest=-65.0, tc_decay=40.0)
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        conv = ns.topology.Conv2dConnection(X, Y, kernel_size=3, stride=2, padding=1, update_rule=L.PostPre, nu=(1e-3, 1e-3),
                                            reduction=torch.sum, wmin=-1.0, wmax=3.0)
        with torch.no_grad():
            conv.w.copy_(2.5 * torch.rand(conv.w.shape, generator=g))
        net.add_connection(conv, "X", "Y")
        n_in, n = 128, 48
    else:
        X = ns.nodes.Input(N_IN, traces=True)
        Y = population(ns, kind, N, g, traces_additive=extra == "traces", per_trace=extra == "traces")
        net.add_layer(X, "X"); net.add_layer(Y, "Y")
        w1 = 3.0 * torch.rand(N_IN, N, generator=g)
        net.add_connection(ns.topology.Connection(X, Y, w=w1, update_rule=L.PostPre, nu=(1e-2, 1e-2), reduction=torch.sum,
                                                  wmin=0.0, wmax=3.0), "X", "Y")
        n_in, n = N_IN, N
    if extra == "ei":
        inh = torch.rand(n, 1, generator=g) < 0.25
        lo = torch.where(inh, torch.full((n, 1), -1.0), torch.zeros(n, 1))
        hi = torch.where(inh, torch.zeros(n, 1), torch.ones(n, 1))
        w_r = torch.where(inh, -torch.rand(n, n, generator=g), torch.rand(n, n, generator=g)) * 0.8
        yy = ns.topology.Connection(Y, Y, w=w_r, wmin=lo, wmax=hi, update_rule=L.WeightDependentPostPre, nu=(5e-2, 5e-2),
                                    reduction=torch.sum)
    else:
        yy = ns.topology.Connection(Y, Y, w=-1.5 * torch.rand(n, n, generator=g), wmin=-2.0, wmax=0.0)
    net.add_connection(yy, "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2 * T, B, *X.shape, generator=g) < 0.25).to(torch.uint8)
    return net, {"X": x}, T


def window_inputs(inputs, T, k):
    return {name: v[k * T:(k + 1) * T] for name, v in inputs.items()}


def live_state(net) -> dict:
    Y = net.layers["Y"]
    out = {"Ys": net.monitors["Ys"].get("s").to(torch.uint8).cpu(), "Y/v": Y.v.detach().clone().cpu(),
           "Y/x": Y.x.detach().clone().cpu()}
    if hasattr(Y, "theta"):
        out["Y/theta"] = Y.theta.detach().clone().cpu()
    for (s, t), c in net.connections.items():
        out[f"{s}{t}/w"] = c.w.detach().clone().cpu()
    return out


def run_two_windows(net, inputs, T, reference=False, **run_kw) -> dict:
    """Two windows without a reset in between."""
    out = {}
    for k in range(2):
        net.run(inputs=window_inputs(inputs, T, k), time=T, **({} if reference else run_kw))
        out.update({f"{k}/{name}": v for name, v in live_state(net).items()})
    return out


def snapshot(net) -> dict:
    """Every layer state and every weight, as numpy arrays (for bit-for-bit comparisons)."""
    out = {}
    for lname, layer in net.layers.items():
        Bz = layer.s.shape[0]
        out[f"L/{lname}/s"] = layer.s.reshape(Bz, -1).to(torch.uint8).cpu().numpy()
        for var in ("v", "refrac_count", "x"):
            val = getattr(layer, var, None)
            if isinstance(val, torch.Tensor) and val.numel() > 0:
                out[f"L/{lname}/{var}"] = val.detach().reshape(Bz, -1).float().cpu().numpy()
        if isinstance(getattr(layer, "theta", None), torch.Tensor):
            out[f"L/{lname}/theta"] = layer.theta.detach().cpu().numpy().copy()
    for (s, t), c in net.connections.items():
        out[f"C/{s}{t}/w"] = c.w.detach().cpu().numpy().copy()
    if "Ys" in net.monitors:
        out["M/Ys"] = net.monitors["Ys"].get("s").to(torch.uint8).cpu().numpy()
    return out


def dc2015_like(ns, n: int, B: int, T: int, n_in: int = 784, seed: int = 0, device: str = "cpu", constant: bool = False,
                one_spike: bool = True):
    """A DiehlAndCook2015-shaped network: Input(n_in) -> DiehlAndCookNodes(n) (PostPre, norm) with per-neuron thresholds
    and theta increments, an inhibitory LIFNodes(n) layer one-to-one and all-to-all back, Poisson input.
    ``constant``: the tensors hold the model's scalars (thresh -52, theta_plus 0.05).  Returns (net, x)."""
    g = torch.Generator().manual_seed(seed)
    L = ns.learning
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    X = ns.nodes.Input(n_in, traces=True, tc_trace=20.0)
    thresh = torch.full((n,), -52.0) if constant else -52.0 - 3.0 * torch.rand(n, generator=g)
    tplus = torch.full((n,), 0.05) if constant else 0.02 + 0.06 * torch.rand(n, generator=g)
    E = ns.nodes.DiehlAndCookNodes(n, traces=True, rest=-65.0, reset=-60.0, thresh=thresh, refrac=5, tc_decay=100.0,
                                   tc_trace=20.0, theta_plus=tplus, tc_theta_decay=1e7, one_spike=one_spike)
    I = ns.nodes.LIFNodes(n, traces=False, rest=-60.0, reset=-45.0, thresh=-40.0, tc_decay=10.0, refrac=2)
    net.add_layer(X, "X"); net.add_layer(E, "Ae"); net.add_layer(I, "Ai")
    w = 0.3 * torch.rand(n_in, n, generator=g)
    net.add_connection(ns.topology.Connection(X, E, w=w, update_rule=L.PostPre, nu=(1e-4, 1e-2), reduction=torch.sum,
                                              wmin=0.0, wmax=1.0, norm=78.4), "X", "Ae")
    net.add_connection(ns.topology.Connection(E, I, w=22.5 * torch.eye(n), wmin=0.0, wmax=22.5), "Ae", "Ai")
    net.add_connection(ns.topology.Connection(I, E, w=-120.0 * (torch.ones(n, n) - torch.eye(n)), wmin=-120.0, wmax=0.0), "Ai", "Ae")
    rate = 0.25 * torch.rand(n_in, generator=g)
    x = (torch.rand(T, B, n_in, generator=g) < rate).to(torch.uint8)
    if device != "cpu":
        net.to(device)
        x = x.to(device)
    return net, x
