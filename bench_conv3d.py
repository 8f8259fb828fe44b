"""Conv3dConnection benchmark: the reference's examples/mnist/conv3d_MNIST.py network, Input [1, 28, 28, 28] ->
Conv3dConnection (kernel 16, stride 4, 25 filters, norm 0.4 * 16**3, wmax 1) -> DiehlAndCookNodes [25, 4, 4, 4] with the
example's -100 recurrent inhibition, learning.NoOp, T = 250.  The input is seeded synthetic Poisson spikes: a random
[28, 28] image of rates up to 64 Hz (the example's intensity / 2), encoded on the device with the package's Poisson
encoder and replicated along depth like the example's digit; it stays resident on the device.
One JSON line per batch size (B = 1 and B = 128) with the median / min / max kernel time per window over ``--steps``
windows after ``--warmup`` windows, the bytes and taps of one step computed from the shapes, and the device name and
power limit read in the same run.

    python bench_conv3d.py [--steps K] [--warmup W]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events).
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch

from bench_sparse import device_info
from bindsnet_b200 import _backend, encoding
from bindsnet_b200.learning import NoOp
from bindsnet_b200.network import Network, nodes, topology

T, K, S, F_, SIDE = 250, 16, 4, 25, 28
C = (SIDE - K) // S + 1


def build(batch: int, device, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    net = Network(dt=1.0, batch_size=batch, learning=True)
    X = nodes.Input(n=SIDE ** 3, shape=(1, SIDE, SIDE, SIDE), traces=True)
    Y = nodes.DiehlAndCookNodes(n=F_ * C ** 3, shape=(F_, C, C, C), traces=True)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    conv = topology.Conv3dConnection(X, Y, kernel_size=K, stride=S, update_rule=NoOp, norm=0.4 * K ** 3, wmax=1.0,
                                     w=torch.rand(F_, 1, K, K, K, generator=g))
    w = torch.zeros(F_, C ** 3, F_, C ** 3)
    for f1 in range(F_):
        for f2 in range(F_):
            if f1 != f2:
                w[f1, torch.arange(C ** 3), f2, torch.arange(C ** 3)] = -100.0
    net.add_connection(conv, "X", "Y")
    net.add_connection(topology.Connection(Y, Y, w=w.view(Y.n, Y.n)), "Y", "Y")
    net.to(device)
    rates = (64.0 * torch.rand(batch, 1, 1, SIDE, SIDE, generator=g)).to(device)
    x = encoding.poisson(rates, time=T, seed=seed + 1)                    # [T, B, 1, 1, 28, 28]
    return net, {"X": x.expand(T, batch, 1, SIDE, SIDE, SIDE).contiguous()}


def _window(net, inputs) -> float:
    _backend.kernel_events = []
    net.run(inputs=inputs, time=T)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def step_traffic(batch: int) -> dict:
    """Per step, from the shapes: every target neuron visits its 16**3 taps (the gather reads the taps of spiking inputs
    only, so this is the upper bound); bytes = source bit rows + the filter taps + the target's state (v, refrac_count,
    x: 3 floats read and written) + the dense recurrent matrix's rows read for the spiking neurons (upper bound: all)."""
    n_src, n_tgt = SIDE ** 3, F_ * C ** 3
    taps = batch * n_tgt * K ** 3
    bytes_ = batch * (n_src // 8) + F_ * K ** 3 * 4 + batch * n_tgt * 3 * 4 * 2 + n_tgt * n_tgt * 4
    return {"taps_per_step": taps, "bytes_per_step_upper": bytes_}


def measure(batch: int, steps: int, warmup: int) -> dict:
    dev = torch.device("cuda")
    net, inputs = build(batch, dev)
    for _ in range(warmup):
        _window(net, inputs)
    ms = []
    for _ in range(steps):
        net.reset_state_variables()
        ms.append(_window(net, inputs))
    net.check_errors()
    spikes = int(inputs["X"].sum())
    med = statistics.median(ms)
    line = {"bench": "conv3d", "B": batch, "input": [1, SIDE, SIDE, SIDE], "target": [F_, C, C, C], "kernel": K, "stride": S,
            "T": T, "windows": steps, "input_spikes_per_step": spikes / T, **step_traffic(batch), **device_info(),
            "ms_median": med, "ms_min": min(ms), "ms_max": max(ms), "sample_timesteps_per_s": batch * T / (med / 1e3)}
    del net, inputs
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    for batch in (1, 128):
        print(json.dumps(measure(batch, a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
