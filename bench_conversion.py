"""ANN-to-SNN benchmark: a seeded LeNet-5 (conv 6@5x5 pad 2, pool, conv 16@5x5, pool, 120, 84, 10) rescaled by
data_based_normalization on seeded random images and converted by ann_to_snn — Input [1, 28, 28] ->
SubtractiveResetIFNodes [6, 28, 28] -> PassThroughNodes [6, 14, 14] -> SubtractiveResetIFNodes [16, 10, 10] ->
PassThroughNodes [16, 5, 5] -> SubtractiveResetIFNodes 120 -> 84 -> 10 — run with learning off (its pooling
connections cannot run in a learning window) on Poisson spikes of rate images from the on-device encoder, T = 250.
Beside it, in the same process and alternated window by window, the twin in which every PassThroughNodes layer is a
McCullochPitts(thresh=1) layer: on 0 / 1 input the two kinds spike alike, so every window also checks that the layers
downstream of them give identical spikes.  One JSON line per batch size.

    python bench_conversion.py [--steps K] [--warmup W] [--batches 32,128] [--gprof]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events).
--gprof then runs one more window of each arm with SNN_B200_GPROF=1, which prints the generic kernel's per-phase cycles
to stderr.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import warnings

import torch

from bench_sparse import device_info
from bindsnet_b200 import _backend, encoding
from bindsnet_b200.conversion import PassThroughNodes, ann_to_snn
from bindsnet_b200.network import nodes

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
import conversion_nets as cn  # noqa: E402

T = 250
POOLED = ("3", "6")   # the PassThroughNodes layers of the converted LeNet-5


def build(batch: int, twin: bool, device):
    torch.manual_seed(0)
    ann = cn.lenet5()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        net = ann_to_snn(ann, input_shape=(1, 28, 28), data=cn.images("lenet5", 256, seed=1))
    net.train(False)
    if twin:
        for name in POOLED:
            old = net.layers[name]
            mcp = nodes.McCullochPitts(shape=old.shape, thresh=1.0)
            net.add_layer(mcp, name)
            for c in net.connections.values():
                c.source = mcp if c.source is old else c.source
                c.target = mcp if c.target is old else c.target
    assert sum(isinstance(l, PassThroughNodes) for l in net.layers.values()) == (0 if twin else 2)
    cn.set_batch(net, batch)
    net.to(device)
    net.reset_state_variables()
    counters = {name: nodes_counter(net, name) for name in net.layers}
    return net, counters


def nodes_counter(net, name):
    from bindsnet_b200.network.monitors import SpikeCounter

    m = SpikeCounter(net.layers[name])
    net.add_monitor(m, "count_" + name)
    return m


def rates(batch: int, device, seed: int) -> torch.Tensor:
    """Rate images of 0-64 Hz per pixel for the Poisson encoder."""
    g = torch.Generator().manual_seed(seed)
    return (64.0 * torch.rand(batch, 1, 28, 28, generator=g)).to(device)


def _window(net, x) -> float:
    _backend.kernel_events = []
    net.run(inputs={"Input": x}, time=T)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def measure(batch: int, steps: int, warmup: int, gprof: bool) -> dict:
    dev = torch.device("cuda")
    arms = {k: build(batch, k == "mcp_twin", dev) for k in ("passthrough", "mcp_twin")}
    ms = {k: [] for k in arms}
    spikes = {k: {} for k in arms}
    for w in range(warmup + steps):
        x = encoding.poisson(rates(batch, dev, seed=w), time=T, dt=1.0, seed=w)
        counts = {}
        for k, (net, counters) in arms.items():   # alternated: both arms see the same clocks and the same neighbours
            net.reset_state_variables()
            t = _window(net, x)
            counts[k] = {name: m.get().clone() for name, m in counters.items()}
            if w >= warmup:
                ms[k].append(t)
                for name, c in counts[k].items():
                    spikes[k][name] = spikes[k].get(name, 0) + int(c.sum())
        for name in counts["passthrough"]:
            assert torch.equal(counts["passthrough"][name], counts["mcp_twin"][name]), f"window {w}: layer {name} differs from the twin"
    for net, _ in arms.values():
        net.check_errors()
    line = {"B": batch, "T": T, "windows": steps, **device_info(), "identical_to_mcp_twin": True}
    for k, v in ms.items():
        line.update({f"{k}_ms_per_window": sum(v) / len(v), f"{k}_ms_min": min(v), f"{k}_ms_max": max(v),
                     f"{k}_sample_timesteps_per_s": batch * T / (sum(v) / len(v) / 1e3)})
    line["spikes_per_window"] = {name: n / steps for name, n in spikes["passthrough"].items()}
    line["passthrough_over_twin"] = line["passthrough_ms_per_window"] / line["mcp_twin_ms_per_window"]
    if gprof:
        os.environ["SNN_B200_GPROF"] = "1"
        try:
            x = encoding.poisson(rates(batch, dev, seed=0), time=T, dt=1.0, seed=0)
            for k, (net, _) in arms.items():
                print(f"[bench_conversion] B={batch} {k}: per-phase cycles", file=sys.stderr, flush=True)
                _window(net, x)
        finally:
            del os.environ["SNN_B200_GPROF"]
    del arms
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
