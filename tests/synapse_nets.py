"""Networks whose dense Connection carries per-synapse wmin / wmax tensors or learning-rate tensors, shared by
tests/test_synapse_tensors.py (CPU: oracle, emulated kernel, stored live-reference results) and
tests/test_gpu_synapse_tensors.py (the CUDA library).  ``ns`` is a ``cases.namespace``: the same builder makes the
reference's network and ours."""
from __future__ import annotations

import torch

INF = float("inf")
# case -> (rule, batch size, bound form, rate form, extras)
CASES = {
    "pp_full":      ("PostPre", 2, "full", "tgt", ""),
    "pp_tgt_mean":  ("PostPre", 3, "tgt", "tgt", "mean"),
    "pp_src_decay": ("PostPre", 2, "src", None, "decay"),
    "wdep_src":     ("WeightDependentPostPre", 2, "src", "full", "decay"),
    "wdep_full":    ("WeightDependentPostPre", 3, "full", "full", "mask"),
    "hebb_full":    ("Hebbian", 2, "full", "full", "mask"),
    "hebb_tgt":     ("Hebbian", 1, "tgt", "src", ""),
    "mstdp_b1":     ("MSTDP", 1, "full", "full", ""),
    "mstdp_b4":     ("MSTDP", 4, "src", "full", "mean"),
    "mstdpet":      ("MSTDPET", 1, "tgt", "full", ""),
    "ei":           ("WeightDependentPostPre", 2, "sign", None, "outside"),
}
LIVE_CASES = list(CASES)
WINDOW_KWARGS = [dict(reward=1.0), dict(reward=-0.5)]
N_IN, N = 40, 30


def learning(ns):
    return ns.learning


def bounds(form: str, ns_: int, nt: int, g: torch.Generator, inf: bool = True):
    """(wmin, wmax) of the given broadcast form, mixing finite and (with ``inf``) infinite entries."""
    big = INF if inf else 4.0
    if form == "full":
        lo = -0.5 - torch.rand(ns_, nt, generator=g)
        hi = 1.0 + 2.0 * torch.rand(ns_, nt, generator=g)
        lo[torch.rand(ns_, nt, generator=g) < 0.2] = -big
        hi[torch.rand(ns_, nt, generator=g) < 0.2] = big
        return lo, hi
    if form == "tgt":
        lo = -0.3 - torch.rand(nt, generator=g)
        hi = 1.0 + 2.0 * torch.rand(nt, generator=g)
        hi[::5] = big
        return lo, hi
    if form == "src":
        lo = -0.2 - torch.rand(ns_, 1, generator=g)
        hi = 0.8 + 2.0 * torch.rand(ns_, 1, generator=g)
        lo[::7] = -big
        return lo, hi
    raise ValueError(form)


def rates(form, rule: str, ns_: int, nt: int, g: torch.Generator):
    """The rule's nu: a pair of floats (form None) or of tensors, with zero entries."""
    scale = {"PostPre": 2e-2, "WeightDependentPostPre": 5e-2, "Hebbian": 1e-3, "MSTDP": 5e-2, "MSTDPET": 0.3}[rule]
    if form is None:
        return (scale, 0.5 * scale)
    shape = {"full": (ns_, nt), "tgt": (nt,), "src": (ns_, 1)}[form]
    out = []
    for k in range(2):
        r = scale * torch.rand(*shape, generator=g)
        r[torch.rand(*shape, generator=g) < 0.25] = 0.0
        out.append(r)
    return tuple(out)


def sign_bounds(n: int, frac_inh: float, g: torch.Generator):
    """Per-row sign bounds of a recurrent E/I matrix: rows of excitatory sources in [0, 1], inhibitory ones in [-1, 0]."""
    inh = torch.rand(n, 1, generator=g) < frac_inh
    lo = torch.where(inh, torch.full((n, 1), -1.0), torch.zeros(n, 1))
    hi = torch.where(inh, torch.zeros(n, 1), torch.ones(n, 1))
    return lo, hi, inh


def live_net(ns, case: str, T: int = 30):
    """Input(40) -> LIFNodes(30) through a Connection with the case's rule, bounds and rates, plus a recurrent LIF -> LIF
    Connection (static, or in case "ei" a WeightDependentPostPre E/I matrix with sign bounds per row whose user w starts
    outside its bounds).  Returns (net, inputs, T, masks)."""
    rule, B, bform, nform, extra = CASES[case]
    L = learning(ns)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    X = ns.nodes.Input(N_IN, traces=True)
    Y = ns.nodes.LIFNodes(N, traces=True, thresh=-58.0, tc_decay=30.0, refrac=3)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    kw = dict(update_rule=getattr(L, rule), nu=rates(nform, rule, N_IN, N, g), weight_decay=2e-3 if extra == "decay" else 0.0)
    if extra == "mean":
        kw["reduction"] = torch.mean
    elif B > 1:
        kw["reduction"] = torch.sum
    if rule.startswith("MSTDP"):
        kw.update(tc_plus=15.0, tc_minus=25.0, tc_e_trace=10.0)
    w1 = 3.0 * torch.rand(N_IN, N, generator=g) - 0.3
    if bform == "sign":
        xy = ns.topology.Connection(X, Y, w=w1.abs(), update_rule=getattr(L, "PostPre"), nu=(1e-2, 1e-2),
                                    reduction=torch.sum, wmin=0.0, wmax=2.0)
    else:
        # (WeightDependentPostPre: finite bounds, its update turns the synapses of an infinite one into NaN)
        lo, hi = bounds(bform, N_IN, N, g, inf=rule != "WeightDependentPostPre")
        xy = ns.topology.Connection(X, Y, w=w1, wmin=lo, wmax=hi, **kw)
    net.add_connection(xy, "X", "Y")
    if case == "ei":
        lo, hi, inh = sign_bounds(N, 0.2, g)
        w_r = torch.where(inh, -torch.rand(N, N, generator=g), torch.rand(N, N, generator=g)) * 0.8
        yy = ns.topology.Connection(Y, Y, w=w_r, wmin=lo, wmax=hi, update_rule=getattr(L, rule), nu=(5e-2, 5e-2),
                                    reduction=torch.sum)
        with torch.no_grad():   # a user w outside its bounds: the first update clamps it
            yy.w.copy_(yy.w * 1.6 + 0.1)
    else:
        yy = ns.topology.Connection(Y, Y, w=-1.5 * torch.rand(N, N, generator=g), wmin=-2.0, wmax=0.0)
    net.add_connection(yy, "Y", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s"], time=T), "Ys")
    x = (torch.rand(2 * T, B, N_IN, generator=g) < 0.25).to(torch.uint8)
    masks = None
    if extra == "mask":
        masks = {("X", "Y"): torch.rand(N_IN, N, generator=g) < 0.1}
    return net, {"X": x}, T, masks


def to_device(net, device):
    """``net.to(device)`` and the rules' rate tensors with it: a rule is not a ``Module``, so ``Network.to`` leaves its
    ``nu`` where it is (and the reference's first update then fails on it, as ours does)."""
    net.to(device)
    for c in net.connections.values():
        r = getattr(c, "update_rule", None)
        if r is not None and r.nu.dim() > 1:
            r.nu = r.nu.to(device)
    return net


def window_inputs(inputs, T, k):
    return {name: v[k * T:(k + 1) * T] for name, v in inputs.items()}


def live_state(net) -> dict:
    out = {"Ys": net.monitors["Ys"].get("s").to(torch.uint8).cpu(),
           "Y/v": net.layers["Y"].v.detach().clone().cpu(), "Y/x": net.layers["Y"].x.detach().clone().cpu()}
    for (s, t), c in net.connections.items():
        out[f"{s}{t}/w"] = c.w.detach().clone().cpu()
    return out


def run_two_windows(net, inputs, T, case, masks=None, reference=False, one_step=False, **run_kw) -> dict:
    """Two windows without a reset in between; the reward of WINDOW_KWARGS[k] for the reward-modulated rules."""
    rule = CASES[case][0]
    out = {}
    for k in range(2):
        kw = dict(WINDOW_KWARGS[k]) if rule.startswith("MSTDP") else {}
        if masks is not None:
            kw["masks"] = {key: (m.to(net.connections[key].w.device)) for key, m in masks.items()}
        if not reference:
            kw.update(one_step=one_step, **run_kw)
        net.run(inputs=window_inputs(inputs, T, k), time=T, **kw)
        out.update({f"{k}/{name}": v for name, v in live_state(net).items()})
    return out


def snapshot(net) -> dict:
    """Every layer state, every weight and the rule state, as numpy arrays (for bit-for-bit comparisons)."""
    out = {}
    for lname, layer in net.layers.items():
        Bz = layer.s.shape[0]
        out[f"L/{lname}/s"] = layer.s.reshape(Bz, -1).to(torch.uint8).cpu().numpy()
        for var in ("v", "refrac_count", "x"):
            val = getattr(layer, var, None)
            if isinstance(val, torch.Tensor) and val.numel() > 0:
                out[f"L/{lname}/{var}"] = val.detach().reshape(Bz, -1).float().cpu().numpy()
    for (s, t), c in net.connections.items():
        out[f"C/{s}{t}/w"] = c.w.detach().cpu().numpy().copy()
        for name in ("p_plus", "p_minus", "eligibility_trace", "_spre", "_spost"):
            v = getattr(c.update_rule, name, None)
            if isinstance(v, torch.Tensor):
                out[f"R/{s}{t}/{name}"] = v.detach().cpu().numpy().copy()
    if "Ys" in net.monitors:
        out["M/Ys"] = net.monitors["Ys"].get("s").to(torch.uint8).cpu().numpy()
    return out


def ei_network(ns, n: int, B: int, T: int, frac_inh: float = 0.2, n_in: int = 784, seed: int = 0, device: str = "cpu",
               full_bounds: bool = False, scalar_twin: bool = False):
    """The benchmark workload: Input(n_in) -> LIFNodes(n) with PostPre and a per-target nu, plus a recurrent n x n
    WeightDependentPostPre Connection with sign bounds per source row (``frac_inh`` inhibitory sources), Poisson input.
    ``full_bounds``: the same bounds materialised as [n, n] tensors.  ``scalar_twin``: scalar bounds [-1, 1] on the
    recurrent matrix and a scalar nu on the input one instead (the network the tensors extend).  Returns (net, x)."""
    g = torch.Generator().manual_seed(seed)
    L = learning(ns)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    X = ns.nodes.Input(n_in, traces=True)
    Y = ns.nodes.LIFNodes(n, traces=True, thresh=-52.0, refrac=5)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    nu_t = 1e-4 * (0.5 + torch.rand(n, generator=g))
    nu = (1e-4, 1e-4) if scalar_twin else (nu_t, nu_t.clone())
    w_in = 0.3 * torch.rand(n_in, n, generator=g)
    xy = ns.topology.Connection(X, Y, w=w_in, update_rule=L.PostPre, nu=nu, reduction=torch.sum, wmin=0.0, wmax=1.0)
    lo, hi, inh = sign_bounds(n, frac_inh, g)
    w_r = torch.where(inh, -torch.rand(n, n, generator=g), torch.rand(n, n, generator=g)) * (2.0 / n)
    if scalar_twin:
        lo, hi = -1.0, 1.0
    elif full_bounds:
        lo, hi = lo.expand(n, n).contiguous(), hi.expand(n, n).contiguous()
    yy = ns.topology.Connection(Y, Y, w=w_r, wmin=lo, wmax=hi, update_rule=L.WeightDependentPostPre, nu=(1e-3, 1e-3),
                                reduction=torch.sum)
    net.add_connection(xy, "X", "Y")
    net.add_connection(yy, "Y", "Y")
    rate = 0.02 * torch.rand(n_in, generator=g)
    x = (torch.rand(T, B, n_in, generator=g) < rate).to(torch.uint8)
    if device != "cpu":
        to_device(net, device)
        x = x.to(device)
    return net, x


def constant_twin(ns, n: int, B: int, T: int, **kw):
    """``ei_network(scalar_twin=True)`` with its scalar bounds and rates as constant tensors of the same values."""
    net, x = ei_network(ns, n, B, T, scalar_twin=True, **kw)
    dev = x.device
    xy, yy = net.connections[("X", "Y")], net.connections[("Y", "Y")]
    with torch.no_grad():
        yy.wmin = torch.nn.Parameter(torch.full((n, n), -1.0, device=dev), requires_grad=False)
        yy.wmax = torch.nn.Parameter(torch.full((n, 1), 1.0, device=dev), requires_grad=False)
        yy.update_rule.wmin, yy.update_rule.wmax = yy.wmin, yy.wmax
        xy.update_rule.nu = torch.stack([torch.full((n,), 1e-4, device=dev), torch.full((n,), 1e-4, device=dev)])
        xy.update_rule._nu_tensors = True
    return net, x

