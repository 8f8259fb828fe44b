"""Max-pooling benchmark: BASELINE config 4's convolution followed by a MaxPool2dConnection, Input [1, 32, 32] ->
Conv2dConnection (16 filters, 5 x 5) -> LIFNodes [16, 28, 28] -> MaxPool2dConnection (2 x 2, stride 2, decay 1 as
ann_to_snn builds it) -> LIFNodes [16, 14, 14] -> dense Connection -> LIFNodes(10), Bernoulli(0.1) input resident on the
device, learning off (the reference's MaxPool2dConnection cannot run in a learning window).  Beside it, in the same
process and alternated window by window, the twin without the pool stage: the convolution's layer feeds the dense
Connection directly.  One JSON line per batch size.

    python bench_maxpool.py [--steps K] [--warmup W] [--batches 32,128] [--gprof]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events).
--gprof then runs one more window of each arm with SNN_B200_GPROF=1, which prints the generic kernel's per-phase cycles
to stderr: the pooled gather and the rate update run inside phase 1, so the two arms' phase-1 rows give the pooling's
share.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

from bench_sparse import device_info
from bindsnet_b200 import _backend
from bindsnet_b200.network import Network, nodes, topology

T = 250


def build(batch: int, pool: bool, device, seed: int = 0):
    """Weights drawn on the CPU (the constructors clamp them against CPU bounds), then the network moved to ``device``."""
    g = torch.Generator().manual_seed(seed)
    w_conv = 0.9 * torch.rand(16, 1, 5, 5, generator=g)
    x = (torch.rand(T, batch, 1, 32, 32, generator=g) < 0.1).to(torch.uint8).to(device)
    net = Network(dt=1.0, batch_size=batch, learning=False)
    X = nodes.Input(shape=[1, 32, 32])
    C1 = nodes.LIFNodes(shape=[16, 28, 28], thresh=-60.0, refrac=2)
    Y = nodes.LIFNodes(10, thresh=-62.0, refrac=2)
    net.add_layer(X, "X"); net.add_layer(C1, "C1")
    net.add_connection(topology.Conv2dConnection(X, C1, kernel_size=5, w=w_conv), "X", "C1")
    if pool:
        P = nodes.LIFNodes(shape=[16, 14, 14], thresh=-64.5, rest=-65.0, reset=-65.0, refrac=1)
        net.add_layer(P, "P")
        net.add_connection(topology.MaxPool2dConnection(C1, P, kernel_size=2, stride=2, decay=1.0), "C1", "P")
        last = P
    else:
        last = C1
    net.add_layer(Y, "Y")
    net.add_connection(topology.Connection(last, Y, w=0.002 * torch.rand(last.n, 10, generator=g)), "P" if pool else "C1", "Y")
    net.to(device)
    return net, {"X": x}


def _window(net, inputs) -> float:
    _backend.kernel_events = []
    net.run(inputs=inputs, time=T)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def measure(batch: int, steps: int, warmup: int, gprof: bool) -> dict:
    dev = torch.device("cuda")
    nets = {k: build(batch, k == "pool", dev) for k in ("pool", "no_pool")}
    for _ in range(warmup):
        for net, inputs in nets.values():
            _window(net, inputs)
    ms = {k: [] for k in nets}
    for _ in range(steps):   # alternated: both arms see the same clocks and the same neighbours on the host
        for k, (net, inputs) in nets.items():
            ms[k].append(_window(net, inputs))
    for net, _ in nets.values():
        net.check_errors()
    line = {"B": batch, "T": T, **device_info()}
    for k, v in ms.items():
        line.update({f"{k}_ms_per_window": sum(v) / len(v), f"{k}_ms_min": min(v), f"{k}_ms_max": max(v),
                     f"{k}_sample_timesteps_per_s": batch * T / (sum(v) / len(v) / 1e3)})
    line["pool_over_no_pool"] = line["pool_ms_per_window"] / line["no_pool_ms_per_window"]
    if gprof:
        os.environ["SNN_B200_GPROF"] = "1"
        try:
            for k, (net, inputs) in nets.items():
                print(f"[bench_maxpool] B={batch} {k}: per-phase cycles", file=sys.stderr, flush=True)
                _window(net, inputs)
        finally:
            del os.environ["SNN_B200_GPROF"]
    del nets
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
