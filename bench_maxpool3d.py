"""3-D max-pooling benchmark: Input [2, 8, 32, 32] (Bernoulli(0.1), resident on the device) -> Conv3dConnection (16
filters, kernel (3, 5, 5)) -> LIFNodes [16, 6, 28, 28] -> MaxPoo3dConnection (kernel 2, stride 2, decay 1) -> LIFNodes
[16, 3, 14, 14] -> dense Connection -> LIFNodes(10), T = 250, learning off (the reference's pooling connections cannot
run in a learning window).  Two comparisons, each alternated window by window in the same process:

  pool / no_pool   the network against its twin without the pool stage (the convolution's layer feeds the dense
                   Connection directly): what the pool stage costs;
  pool3d / pool2d  a MaxPoo3dConnection with a kernel of depth 1 (Input [16, 6, 28, 28] -> kernel (1, 2, 2) -> LIFNodes
                   [16, 6, 14, 14] -> dense -> LIFNodes(10)) against the MaxPool2dConnection that does the same work
                   (Input [96, 28, 28] -> kernel 2 -> LIFNodes [96, 14, 14] -> dense -> LIFNodes(10)): whether the 3-D
                   path costs what the 2-D one costs.

One JSON line per batch size.

    python bench_maxpool3d.py [--steps K] [--warmup W] [--batches 32,128] [--gprof]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events);
each line carries the median, min and max over the timed windows and the device name and power limit read in the same
run.  --gprof then runs one more window of each arm with SNN_B200_GPROF=1, which prints the generic kernel's per-phase
cycles to stderr: the pooled gather runs inside phase 1.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

from bench_sparse import device_info
from bindsnet_b200 import _backend
from bindsnet_b200.network import Network, nodes, topology

T = 250


def build_conv(batch: int, pool: bool, device, seed: int = 0):
    """Weights drawn on the CPU (the constructors clamp them against CPU bounds), then the network moved to ``device``."""
    g = torch.Generator().manual_seed(seed)
    w_conv = 0.5 * torch.rand(16, 2, 3, 5, 5, generator=g)
    x = (torch.rand(T, batch, 2, 8, 32, 32, generator=g) < 0.1).to(torch.uint8).to(device)
    net = Network(dt=1.0, batch_size=batch, learning=False)
    X = nodes.Input(shape=[2, 8, 32, 32])
    C1 = nodes.LIFNodes(shape=[16, 6, 28, 28], thresh=-60.0, refrac=2)
    Y = nodes.LIFNodes(10, thresh=-62.0, refrac=2)
    net.add_layer(X, "X"); net.add_layer(C1, "C1")
    net.add_connection(topology.Conv3dConnection(X, C1, kernel_size=(3, 5, 5), w=w_conv, b=torch.zeros(16)), "X", "C1")
    last, name = C1, "C1"
    if pool:
        P = nodes.LIFNodes(shape=[16, 3, 14, 14], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=1)
        net.add_layer(P, "P")
        net.add_connection(topology.MaxPoo3dConnection(C1, P, kernel_size=2, stride=2, decay=1.0), "C1", "P")
        last, name = P, "P"
    net.add_layer(Y, "Y")
    net.add_connection(topology.Connection(last, Y, w=0.002 * torch.rand(last.n, 10, generator=g)), name, "Y")
    net.to(device)
    return net, {"X": x}


def build_flat(batch: int, three_d: bool, device, seed: int = 1):
    """The same pooling work as a depth-1 MaxPoo3dConnection over [16, 6, 28, 28] or a MaxPool2dConnection over
    [96, 28, 28]: identical inputs, rates and outputs, neuron for neuron."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(T, batch, 96, 28, 28, generator=g) < 0.1).to(torch.uint8)
    w = 0.002 * torch.rand(96 * 14 * 14, 10, generator=g)
    src, tgt = ([16, 6, 28, 28], [16, 6, 14, 14]) if three_d else ([96, 28, 28], [96, 14, 14])
    net = Network(dt=1.0, batch_size=batch, learning=False)
    X = nodes.Input(shape=src)
    P = nodes.LIFNodes(shape=tgt, thresh=-64.5, rest=-65.0, reset=-65.0, refrac=1)
    Y = nodes.LIFNodes(10, thresh=-62.0, refrac=2)
    for name, layer in (("X", X), ("P", P), ("Y", Y)):
        net.add_layer(layer, name)
    if three_d:
        pool = topology.MaxPoo3dConnection(X, P, kernel_size=(1, 2, 2), stride=(1, 2, 2), decay=1.0)
    else:
        pool = topology.MaxPool2dConnection(X, P, kernel_size=2, stride=2, decay=1.0)
    net.add_connection(pool, "X", "P")
    net.add_connection(topology.Connection(P, Y, w=w), "P", "Y")
    net.to(device)
    return net, {"X": x.view(T, batch, *src).to(device)}


def _window(net, inputs) -> float:
    _backend.kernel_events = []
    net.run(inputs=inputs, time=T)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def _alternate(nets, steps: int, warmup: int) -> dict:
    for _ in range(warmup):
        for net, inputs in nets.values():
            _window(net, inputs)
    ms = {k: [] for k in nets}
    for _ in range(steps):   # alternated: both arms see the same clocks and the same neighbours on the host
        for k, (net, inputs) in nets.items():
            ms[k].append(_window(net, inputs))
    for net, _ in nets.values():
        net.check_errors()
    return ms


def measure(batch: int, steps: int, warmup: int, gprof: bool) -> dict:
    dev = torch.device("cuda")
    line = {"B": batch, "T": T, **device_info()}
    groups = {"conv": {k: build_conv(batch, k == "pool", dev) for k in ("pool", "no_pool")},
              "flat": {k: build_flat(batch, k == "pool3d", dev) for k in ("pool3d", "pool2d")}}
    for nets in groups.values():
        for k, v in _alternate(nets, steps, warmup).items():
            line.update({f"{k}_ms_median": statistics.median(v), f"{k}_ms_min": min(v), f"{k}_ms_max": max(v),
                         f"{k}_sample_timesteps_per_s": batch * T / (statistics.median(v) / 1e3)})
    line["pool_over_no_pool"] = line["pool_ms_median"] / line["no_pool_ms_median"]
    line["pool3d_over_pool2d"] = line["pool3d_ms_median"] / line["pool2d_ms_median"]
    if gprof:
        os.environ["SNN_B200_GPROF"] = "1"
        try:
            for nets in groups.values():
                for k, (net, inputs) in nets.items():
                    print(f"[bench_maxpool3d] B={batch} {k}: per-phase cycles", file=sys.stderr, flush=True)
                    _window(net, inputs)
        finally:
            del os.environ["SNN_B200_GPROF"]
    del groups
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batches", default="32,128")
    ap.add_argument("--gprof", action="store_true")
    a = ap.parse_args()
    for b in a.batches.split(","):
        print(json.dumps(measure(int(b), a.steps, a.warmup, a.gprof)), flush=True)


if __name__ == "__main__":
    main()
