"""Networks with a MeanFieldConnection, shared by tests/test_meanfield.py (CPU: oracle, emulated kernel, stored
live-reference results) and tests/test_gpu_meanfield.py (the CUDA library).  ``ns`` is a ``cases.namespace``: the same
builder makes the reference's network and ours.

A case is ``b{B}_{source}_{w form}_{order}``:
  source   in (the Input), lif (a LIFNodes layer), dc1 (DiehlAndCookNodes with one_spike), clamp (the LIF layer with
           clamp / unclamp masks in the run), self (the target itself, a recurrent self-loop)
  w form   0d, n ([W], the last axis), 1w ([1, W]), c1 ([C, 1]), full ([B, C, W], per sample)
  order    mf (the mean-field connection only), mf_dense / dense_mf (with a dense Connection into the same target, in
           that insertion order)
The target is McCullochPitts [C, W] = [2, 4], whose v is its input: the raw sum is compared bit for bit.  At B > 1
sample 0 of the Input never spikes, so it receives nothing but the batch mean (the batch coupling)."""
from __future__ import annotations

import torch

C_, W_ = 2, 4
N_IN = 24

LIVE_CASES = [
    "b1_in_0d_mf", "b3_in_n_mf", "b8_in_1w_mf", "b3_in_c1_mf", "b3_in_full_mf", "b8_in_full_mf_dense",
    "b3_lif_n_dense_mf", "b3_lif_0d_mf_dense", "b8_dc1_c1_mf", "b3_clamp_1w_mf", "b3_self_n_mf_dense", "b1_self_full_dense_mf",
]


def parse(case: str):
    b, src, form, order = case.split("_", 3)
    return int(b[1:]), src, form, order


def w_of(form: str, B: int, g: torch.Generator) -> torch.Tensor:
    shape = {"0d": (), "n": (W_,), "1w": (1, W_), "c1": (C_, 1), "full": (B, C_, W_)}[form]
    return (torch.rand(shape, generator=g) * 4.0 - 1.0).float()   # both signs


def mf_net(ns, case: str, T: int = 21):
    """Input [N_IN] -> (dense) LIFNodes A [8] / DiehlAndCookNodes D [8] (one_spike); MeanFieldConnection from the case's
    source, and optionally a dense Input -> target Connection, into McCullochPitts Y [C, W].  Returns (net, inputs, T,
    run_kwargs)."""
    B, src, form, order = parse(case)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    X = ns.nodes.Input(n=N_IN, traces=True)
    net.add_layer(X, name="X")
    if src in ("lif", "clamp"):
        A = ns.nodes.LIFNodes(n=8, thresh=-62.0, refrac=1, traces=True)
        net.add_layer(A, name="A")
        net.add_connection(ns.topology.Connection(X, A, w=torch.rand(N_IN, 8, generator=g) * 6.0), source="X", target="A")
    if src == "dc1":
        D = ns.nodes.DiehlAndCookNodes(n=8, thresh=-60.0, one_spike=True, traces=True)
        net.add_layer(D, name="A")
        wd = torch.zeros(N_IN, 8)
        wd[:, 3] = torch.rand(N_IN, generator=g) * 8.0   # one candidate per step: the winner needs no tie-break
        net.add_connection(ns.topology.Connection(X, D, w=wd), source="X", target="A")
    Y = ns.nodes.McCullochPitts(shape=[C_, W_], thresh=0.05)
    net.add_layer(Y, name="Y")
    source = {"in": X, "lif": net.layers.get("A"), "clamp": net.layers.get("A"), "dc1": net.layers.get("A"), "self": Y}[src]
    sname = {"in": "X", "lif": "A", "clamp": "A", "dc1": "A", "self": "Y"}[src]
    mf = ns.topology.MeanFieldConnection(source, Y, w=w_of(form, B, g))
    dense = ns.topology.Connection(X, Y, w=torch.rand(N_IN, C_ * W_, generator=g) * 0.3 - 0.05)
    if order == "dense_mf":
        net.add_connection(dense, source="X", target="Y")
    net.add_connection(mf, source=sname, target="Y")
    if order == "mf_dense":
        net.add_connection(dense, source="X", target="Y")
    net.add_monitor(ns.monitors.Monitor(Y, state_vars=("s", "v"), time=T), name="Y")
    p = torch.rand(B, N_IN, generator=g) * 0.35
    if B > 1:
        p[0] = 0.0   # a silent sample: all it receives is the batch mean
    x = torch.stack([torch.bernoulli(p.expand(T, B, N_IN), generator=g).bool() for _ in range(2)])
    kw = {}
    if src == "clamp":
        kw = dict(clamp={"A": torch.tensor([1, 0, 0, 0, 0, 0, 0, 1], dtype=torch.bool)},
                  unclamp={"A": torch.tensor([0, 1, 1, 0, 0, 0, 0, 0], dtype=torch.bool)})
    return net, {"X": x}, T, kw


def state(net, monitors: bool = True) -> dict:
    out = {"Ys": net.monitors["Y"].get("s").to(torch.uint8).cpu().clone(),
           "Yv": net.monitors["Y"].get("v").detach().cpu().clone()} if monitors else {}
    for lname, layer in net.layers.items():
        out[f"{lname}/s"] = layer.s.to(torch.uint8).cpu().clone()
        for var in ("v", "refrac_count", "x", "theta"):
            v = getattr(layer, var, None)
            if isinstance(v, torch.Tensor) and v.numel():
                out[f"{lname}/{var}"] = v.detach().cpu().clone()
    for (s, t), c in net.connections.items():
        out[f"{s}{t}/w"] = c.w.detach().cpu().clone()
    return out


def run_two_windows(net, inputs, T, reset: bool = True, **kw):
    """Two windows, with reset_state_variables() between them unless ``reset`` is False; the state after each."""
    states = []
    for w in range(2):
        net.run(inputs={k: v[w].clone() for k, v in inputs.items()}, time=T, **kw)
        states.append(state(net))
        if w == 0 and reset:
            net.reset_state_variables()
    return states


def flat(states) -> dict:
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}


def big_net(ns, B: int = 128, T: int = 250, with_mf: bool = True, seed: int = 0):
    """The large case: Input(784) -> LIFNodes(1600) with PostPre, plus a LIF -> LIF MeanFieldConnection with negative
    per-target w into a second LIFNodes(1600) population that also receives the Input.  Returns (net, inputs, T)."""
    g = torch.Generator().manual_seed(seed)
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    X = ns.nodes.Input(n=784, traces=True)
    A = ns.nodes.LIFNodes(n=1600, traces=True, thresh=-52.0)
    Z = ns.nodes.LIFNodes(n=1600, thresh=-52.0)
    net.add_layer(X, name="X")
    net.add_layer(A, name="A")
    net.add_layer(Z, name="Z")
    net.add_connection(ns.topology.Connection(X, A, w=0.3 * torch.rand(784, 1600, generator=g), update_rule=ns.learning.PostPre,
                                              nu=(1e-4, 1e-2), wmin=0.0, wmax=1.0), source="X", target="A")
    net.add_connection(ns.topology.Connection(X, Z, w=0.25 * torch.rand(784, 1600, generator=g)), source="X", target="Z")
    if with_mf:
        net.add_connection(ns.topology.MeanFieldConnection(A, Z, w=-40.0 * torch.rand(1600, generator=g)), source="A", target="Z")
    x = torch.bernoulli(0.05 * torch.ones(T, B, 784), generator=g).bool()
    return net, {"X": x}, T
