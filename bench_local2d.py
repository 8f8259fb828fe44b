"""LocalConnection2D benchmark: the reference's examples/mnist/loc2d_mnist.py network, Input [1, 20, 20] ->
LocalConnection2D (kernel 12, stride 4, 50 filters, PostPre, norm) -> AdaptiveLIFNodes [50, 3, 3] with the recurrent
inhibition, learning on, T = 250, Bernoulli(0.05) input resident on the device.
  B = 1    alternated window by window with a twin whose input connection is the classic LocalConnection (a dense
           [400, 450] matrix held to the same receptive fields by its mask): what the native kind saves.
  B = 128  the batched variant on Input [1, 28, 28] (1250 target neurons), reduction=torch.sum.
One JSON line per measurement, with the median / min / max kernel time per window over ``--steps`` windows after
``--warmup`` windows, and the device name and power limit read in the same run.

    python bench_local2d.py [--steps K] [--warmup W]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events).
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch

from bench_sparse import device_info
from bindsnet_b200 import _backend
from bindsnet_b200.learning import PostPre
from bindsnet_b200.network import Network, nodes, topology

T = 250


def build(batch: int, side: int, local2d: bool, device, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    k, s, F_ = 12, 4, 50
    c = (side - k) // s + 1
    net = Network(dt=1.0, batch_size=batch, learning=True)
    X = nodes.Input(shape=[1, side, side], traces=True, tc_trace=20)
    Y = nodes.AdaptiveLIFNodes(shape=[F_, c, c], traces=True, rest=-65.0, reset=-60.0, thresh=-52.0, refrac=5, tc_trace=20.0,
                               theta_plus=0.05, tc_theta_decay=1e6)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    kw = dict(kernel_size=k, stride=s, n_filters=F_, nu=(1e-4, 1e-2), update_rule=PostPre, wmin=0.0, wmax=1.0, norm=0.2 * k * k,
              reduction=None if batch == 1 else torch.sum)
    if local2d:
        lc = topology.LocalConnection2D(X, Y, **kw)
    else:
        lc = topology.LocalConnection(X, Y, input_shape=(side, side), **kw)
    w_inh = torch.zeros(F_, c, c, F_, c, c)
    for f in range(F_):
        for a in range(c):
            for b in range(c):
                w_inh[f, a, b, :, a, b] = -25.0
                w_inh[f, a, b, f, a, b] = 0
    net.add_connection(lc, "X", "Y")
    net.add_connection(topology.Connection(Y, Y, w=w_inh.reshape(Y.n, Y.n)), "Y", "Y")
    net.to(device)
    x = (torch.rand(T, batch, 1, side, side, generator=g) < 0.05).to(torch.uint8).to(device)
    return net, {"X": x}


def _window(net, inputs) -> float:
    _backend.kernel_events = []
    net.run(inputs=inputs, time=T)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def measure(batch: int, side: int, arms, steps: int, warmup: int) -> dict:
    dev = torch.device("cuda")
    nets = {k: build(batch, side, k == "local2d", dev) for k in arms}
    for _ in range(warmup):
        for net, inputs in nets.values():
            _window(net, inputs)
    ms = {k: [] for k in nets}
    for _ in range(steps):   # alternated: every arm sees the same clocks and the same neighbours on the host
        for k, (net, inputs) in nets.items():
            ms[k].append(_window(net, inputs))
    for net, _ in nets.values():
        net.check_errors()
    line = {"B": batch, "input": [1, side, side], "T": T, "windows": steps, **device_info()}
    for k, v in ms.items():
        med = statistics.median(v)
        line.update({f"{k}_ms_median": med, f"{k}_ms_min": min(v), f"{k}_ms_max": max(v),
                     f"{k}_sample_timesteps_per_s": batch * T / (med / 1e3)})
    if len(ms) == 2:
        line["dense_mask_over_local2d"] = line["dense_mask_ms_median"] / line["local2d_ms_median"]
    del nets
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    print(json.dumps(measure(1, 20, ("local2d", "dense_mask"), a.steps, a.warmup)), flush=True)
    print(json.dumps(measure(128, 28, ("local2d",), a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
