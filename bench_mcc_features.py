"""Stochastic-synapse benchmark of the MulticompartmentConnection features, the topology of the reference's
examples/mnist/MCC_reservoir.py: Input(784) -> MCC[Probability, Weight] -> LIFNodes(N) with a recurrent
MCC[Probability, Weight], scalar threshold, T = 250, inputs resident on the device.  Beside it, in the same process and
alternated window by window, the same network with Weight-only pipelines (what the features cost).  Learning on means
MCC_learning.PostPre on the input Weight.  One JSON line per configuration.

    python bench_mcc_features.py [--steps K] [--warmup W] [--configs 4000:32:0,4000:128:1]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events).
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json

import torch

from bench_sparse import device_info
from bindsnet_b200 import _backend
from bindsnet_b200.learning import MCC_learning
from bindsnet_b200.network import Network, nodes, topology
from bindsnet_b200.network.topology_features import Probability, Weight

T, N_IN = 250, 784


def build(n: int, batch: int, learning: bool, features: bool, device, seed: int = 0):
    """Input weights in [0, 1) (mostly excitatory), recurrent weights of mixed sign scaled by 1 / sqrt(n); transmission
    probabilities uniform in [0, 1), as MCC_reservoir.py draws them.  The Weight-only twin holds the same weights."""
    g = torch.Generator(device=device).manual_seed(seed)
    w_in = torch.rand(N_IN, n, generator=g, device=device)
    w_rec = (torch.rand(n, n, generator=g, device=device) - 0.5) * (8.0 / n ** 0.5)
    p_in = torch.rand(N_IN, n, generator=g, device=device)
    p_rec = torch.rand(n, n, generator=g, device=device)
    x = (torch.rand(T, batch, N_IN, generator=g, device=device) < 0.05).to(torch.uint8)
    net = Network(dt=1.0, batch_size=batch, learning=learning)
    X, Y = nodes.Input(N_IN, traces=learning), nodes.LIFNodes(n, thresh=-52.0, traces=learning)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    rule = dict(learning_rule=MCC_learning.PostPre, nu=(1e-4, 1e-3), range=[0.0, 1.0]) if learning else {}
    pin = [Weight("w_in", w_in, **rule)]
    prec = [Weight("w_rec", w_rec)]
    if features:
        pin.insert(0, Probability("p_in", p_in))
        prec.insert(0, Probability("p_rec", p_rec))
    net.add_connection(topology.MulticompartmentConnection(X, Y, device=device, pipeline=pin), "X", "Y")
    net.add_connection(topology.MulticompartmentConnection(Y, Y, device=device, pipeline=prec), "Y", "Y")
    net.to(device)
    return net, {"X": x}


def _window(net, inputs) -> float:
    _backend.kernel_events = []
    net.run(inputs=inputs, time=T)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def measure(n: int, batch: int, learning: bool, steps: int, warmup: int) -> dict:
    dev = torch.device("cuda")
    nets = {k: build(n, batch, learning, k == "features", dev) for k in ("features", "weight_only")}
    for _ in range(warmup):
        for net, inputs in nets.values():
            _window(net, inputs)
    ms = {k: [] for k in nets}
    for _ in range(steps):   # alternated: both arms see the same clocks and the same neighbours on the host
        for k, (net, inputs) in nets.items():
            ms[k].append(_window(net, inputs))
    for net, _ in nets.values():
        net.check_errors()
    line = {"N": n, "B": batch, "T": T, "learning": learning, **device_info()}
    for k, v in ms.items():
        line.update({f"{k}_ms_per_window": sum(v) / len(v), f"{k}_ms_min": min(v), f"{k}_ms_max": max(v),
                     f"{k}_sample_timesteps_per_s": batch * T / (sum(v) / len(v) / 1e3)})
    line["features_over_weight_only"] = line["features_ms_per_window"] / line["weight_only_ms_per_window"]
    del nets
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--configs", default="4000:32:0,4000:32:1,4000:128:0,4000:128:1")
    a = ap.parse_args()
    for item in a.configs.split(","):
        n, b, learn = item.split(":")
        print(json.dumps(measure(int(n), int(b), bool(int(learn)), a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
