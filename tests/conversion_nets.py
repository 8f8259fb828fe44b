"""Networks of ``ann_to_snn`` and of its two layer kinds, shared by tests/test_conversion.py (CPU: oracle, emulated
kernel, stored live-reference results) and tests/test_gpu_conversion.py (the CUDA library).  ``ns`` is a
``cases.namespace``: the same builder makes the reference's network and ours."""
from __future__ import annotations

import importlib

import torch
import torch.nn as nn


def conversion(ns):
    """``bindsnet.conversion`` of the namespace's package."""
    return importlib.import_module("bindsnet_b200.conversion" if ns.kind == "b200" else "bindsnet.conversion")


class FullyConnected(nn.Module):
    """784 -> 256 -> 128 -> 10 with ReLUs applied in forward (no ReLU modules): the shape of the reference's own
    conversion test network."""

    def __init__(self):
        super().__init__()
        self.fc1 = nn.Linear(784, 256)
        self.fc2 = nn.Linear(256, 128)
        self.fc3 = nn.Linear(128, 10)

    def forward(self, x):
        return self.fc3(torch.relu(self.fc2(torch.relu(self.fc1(x)))))


def small_cnn(conv_bias: bool = True):
    """[1, 28, 28] -> conv 4@5x5 -> ReLU -> pool 2 -> conv 8@3x3 -> ReLU -> pool 2 -> flatten -> 32 -> ReLU -> 10."""
    return nn.Sequential(
        nn.Conv2d(1, 4, 5, bias=conv_bias), nn.ReLU(), nn.MaxPool2d(2),
        nn.Conv2d(4, 8, 3), nn.ReLU(), nn.MaxPool2d(2),
        nn.Flatten(), nn.Linear(200, 32), nn.ReLU(), nn.Linear(32, 10),
    )


def lenet5():
    """LeNet-5: [1, 28, 28] -> conv 6@5x5 pad 2 -> ReLU -> pool -> conv 16@5x5 -> ReLU -> pool -> 120 -> 84 -> 10."""
    return nn.Sequential(
        nn.Conv2d(1, 6, 5, padding=2), nn.ReLU(), nn.MaxPool2d(2),
        nn.Conv2d(6, 16, 5), nn.ReLU(), nn.MaxPool2d(2),
        nn.Flatten(), nn.Linear(400, 120), nn.ReLU(), nn.Linear(120, 84), nn.ReLU(), nn.Linear(84, 10),
    )


MODELS = {"fc": (FullyConnected, (784,)), "cnn": (small_cnn, (1, 28, 28)), "lenet5": (lenet5, (1, 28, 28))}


def model(name: str, seed: int = 0):
    torch.manual_seed(seed)
    return MODELS[name][0]()


def images(name: str, n: int, seed: int = 1) -> torch.Tensor:
    """Seeded random images in [0, 1) of the model's input shape."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, *MODELS[name][1], generator=g)


def convert(ns, name: str, data: bool, seed: int = 0, percentile: float = 99.9):
    """``ann_to_snn`` of the seeded model, with ``data_based_normalization`` on 64 seeded images when ``data``."""
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return conversion(ns).ann_to_snn(model(name, seed), input_shape=MODELS[name][1], data=images(name, 64) if data else None,
                                         percentile=percentile)


def set_batch(net, B: int):
    """Batch size B for a converted network (built at batch 1): the reference's pooling connections keep their
    batch-1 rates buffer until reset_state_variables()."""
    net.batch_size = B
    for layer in net.layers.values():
        layer.set_batch_size(B)
    net.reset_state_variables()


def rate_inputs(shape, T: int, B: int, seed: int = 5, windows: int = 2, p: float = 0.25) -> torch.Tensor:
    """[windows, T, B, *shape] Bernoulli(p * pixel) spikes of seeded random images."""
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(windows, 1, B, *shape, generator=g)
    return (torch.rand(windows, T, B, *shape, generator=g) < p * img).to(torch.uint8)


def cnn_net(ns, B: int, T: int = 32, data: bool = True, monitors: bool = True):
    """The small CNN converted (learning off, batch B) with Monitors on both PassThroughNodes layers' s; returns
    (net, inputs, T)."""
    net = convert(ns, "cnn", data)
    net.train(False)
    set_batch(net, B)
    if monitors:
        for name in ("3", "6"):
            net.add_monitor(ns.monitors.Monitor(net.layers[name], ["s"], time=T), "M" + name)
    return net, {"Input": rate_inputs((1, 28, 28), T, B, p=0.6)}, T


def subif_net(ns, case: str, B: int = 3, T: int = 30):
    """Input(24) -> dense Connection -> SubtractiveResetIFNodes(16), thresh 1, reset 0.
      refrac      refrac = 1.5 at dt = 1: 0.5 left after a step, then a negative counter that gates one more step off
      lbound      negative weights and lbound = -0.75
      traces      traces and summed input
      postpre     PostPre on the connection, learning on (traces on both ends)"""
    conv = conversion(ns)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    learning = case == "postpre"
    net = ns.Network(dt=1.0, batch_size=B, learning=learning)
    X = ns.nodes.Input(24, traces=case in ("traces", "postpre"))
    kw = dict(thresh=1.0, reset=0.0, refrac=0)
    if case == "refrac":
        kw["refrac"] = 1.5
    if case == "lbound":
        kw["lbound"] = -0.75
    if case in ("traces", "postpre"):
        kw.update(traces=True, sum_input=True, tc_trace=5.0)
    Y = conv.SubtractiveResetIFNodes(16, **kw)
    net.add_layer(X, "X")
    net.add_layer(Y, "Y")
    w = 0.4 * torch.rand(24, 16, generator=g) - (0.18 if case == "lbound" else 0.05)
    ckw = dict(update_rule=ns.learning.PostPre, nu=(1e-2, 2e-2), wmin=-1.0, wmax=1.0) if learning else {}
    net.add_connection(ns.topology.Connection(X, Y, w=w, **ckw), "X", "Y")
    net.add_monitor(ns.monitors.Monitor(Y, ["s", "v"], time=T), "Ys")
    return net, {"X": rate_inputs((24,), T, B, seed=len(case), p=0.6)}, T


def passthrough_net(ns, B: int = 2, T: int = 20):
    """A PassThroughNodes layer [2, 6, 6] driven by external float 0 / 1 input, then Conv2dConnection (3 x 3) ->
    SubtractiveResetIFNodes [3, 4, 4] and MaxPool2dConnection -> PassThroughNodes [3, 2, 2] -> dense Connection ->
    SubtractiveResetIFNodes(5, sum_input)."""
    conv = conversion(ns)
    g = torch.Generator().manual_seed(23)
    net = ns.Network(dt=1.0, batch_size=B, learning=False)
    P = conv.PassThroughNodes(shape=[2, 6, 6])
    C = conv.SubtractiveResetIFNodes(shape=[3, 4, 4], thresh=1.0, reset=0.0, refrac=0)
    Q = conv.PassThroughNodes(shape=[3, 2, 2])
    Y = conv.SubtractiveResetIFNodes(5, thresh=1.0, reset=0.0, refrac=0, sum_input=True)
    for name, layer in (("P", P), ("C", C), ("Q", Q), ("Y", Y)):
        net.add_layer(layer, name)
    net.add_connection(ns.topology.Conv2dConnection(P, C, kernel_size=3, w=0.5 * torch.rand(3, 2, 3, 3, generator=g),
                                                    b=0.05 * torch.rand(3, generator=g)), "P", "C")
    net.add_connection(ns.topology.MaxPool2dConnection(C, Q, kernel_size=2, stride=2, decay=1), "C", "Q")
    net.add_connection(ns.topology.Connection(Q, Y, w=0.6 * torch.rand(12, 5, generator=g)), "Q", "Y")
    net.add_monitor(ns.monitors.Monitor(P, ["s"], time=T), "MP")
    net.add_monitor(ns.monitors.Monitor(Q, ["s"], time=T), "MQ")
    x = rate_inputs((2, 6, 6), T, B, seed=8, p=0.7).float()
    return net, {"P": x}, T


def run_two_windows(net, inputs, T, reset: bool = True, **kw):
    """Two windows, with reset_state_variables() between them unless ``reset`` is False; the state after each."""
    states = []
    for w in range(2):
        # a copy per window: the reference's Input / PassThroughNodes alias their input as s, and reset_state_variables()
        # zeroes s in place
        net.run(inputs={k: v[w].clone() for k, v in inputs.items()}, time=T, **kw)
        states.append(state(net))
        if w == 0 and reset:
            net.reset_state_variables()
    return states


def state(net) -> dict:
    out = {}
    for mname, mon in net.monitors.items():
        for var in mon.state_vars:
            out[f"{mname}/{var}"] = mon.get(var).detach().cpu().clone()
    for lname, layer in net.layers.items():
        out[f"{lname}/s"] = layer.s.detach().cpu().clone()
        for var in ("v", "refrac_count", "x", "summed"):
            v = getattr(layer, var, None)
            if isinstance(v, torch.Tensor) and v.numel():
                out[f"{lname}/{var}"] = v.detach().cpu().clone()
    for (s, t), c in net.connections.items():
        if hasattr(c, "firing_rates"):
            out[f"{s}-{t}/fr"] = c.firing_rates.detach().cpu().clone()
        else:
            out[f"{s}-{t}/w"] = c.w.detach().cpu().clone()
    return out


def flat(states) -> dict:
    return {f"w{w}/{k}": v for w, st in enumerate(states) for k, v in st.items()}
