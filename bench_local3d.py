"""LocalConnection3D benchmark: the reference's examples/mnist/loc3d_mnist.py network, Input [1, 20, 20, 20] ->
LocalConnection3D (kernel 16, stride 2, 25 filters, PostPre nu (1e-4, 1e-2), w in [0, 1], norm 0.2 * 16^3) ->
AdaptiveLIFNodes [25, 3, 3, 3] with -25 recurrent inhibition, learning on, T = 250.  The input is seeded Bernoulli(0.05)
spikes of a [20, 20] image replicated along the first spatial axis, as the example replicates MNIST, resident on the
device.
  B = 1    alternated window by window with a twin whose input connection is a dense Connection ([8000, 675] weights)
           held to the same receptive fields by Network.run's masks=: what the native kind saves.
  B = 32   reduction=torch.sum.
One JSON line per measurement, with the median / min / max kernel time per window over ``--steps`` windows after
``--warmup`` windows, and the device name and power limit read in the same run.  Each line also carries the learning
phase's weight traffic computed from the shapes: every step reads and writes all of w (2 x 11.06 MB), which bounds the
learning phase from below at the device's memory bandwidth.

    python bench_local3d.py [--steps K] [--warmup W]

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

T, S, K, STRIDE, F_ = 250, 20, 16, 2, 25
C = (S - K) // STRIDE + 1


def receptive_mask() -> torch.Tensor:
    """[S^3, F_ * C^3] bool, True where the dense twin's weight lies outside target j's receptive field (masked to zero)."""
    m = torch.ones(S, S, S, F_, C, C, C, dtype=torch.bool)
    for a in range(C):
        for b in range(C):
            for c in range(C):
                m[a * STRIDE:a * STRIDE + K, b * STRIDE:b * STRIDE + K, c * STRIDE:c * STRIDE + K, :, a, b, c] = False
    return m.reshape(S ** 3, F_ * C ** 3)


def build(batch: int, local3d: bool, device, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    net = Network(dt=1.0, batch_size=batch, learning=True)
    X = nodes.Input(shape=[1, S, S, S], traces=True)
    Y = nodes.AdaptiveLIFNodes(shape=[F_, C, C, C], traces=True, rest=-65.0, reset=-60.0, thresh=-52.0, refrac=5, tc_trace=20.0,
                               theta_plus=0.05, tc_theta_decay=1e6)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    kw = dict(nu=(1e-4, 1e-2), update_rule=PostPre, wmin=0.0, wmax=1.0, norm=0.2 * K ** 3, reduction=None if batch == 1 else torch.sum)
    masks = {}
    if local3d:
        lc = topology.LocalConnection3D(X, Y, kernel_size=K, stride=STRIDE, n_filters=F_, **kw)
    else:
        m = receptive_mask()
        lc = topology.Connection(X, Y, w=torch.rand(X.n, Y.n, generator=g).masked_fill(m, 0.0), **kw)
        masks[("X", "Y")] = m.to(device)
    P = C ** 3
    w_inh = torch.zeros(F_, P, F_, P)
    for p in range(P):
        w_inh[:, p, :, p] = -25.0
        w_inh[torch.arange(F_), p, torch.arange(F_), p] = 0.0
    net.add_connection(lc, "X", "Y")
    net.add_connection(topology.Connection(Y, Y, w=w_inh.reshape(Y.n, Y.n)), "Y", "Y")
    net.to(device)
    img = (torch.rand(T, batch, 1, 1, S, S, generator=g) < 0.05).to(torch.uint8)
    return net, {"X": img.repeat(1, 1, 1, S, 1, 1).to(device)}, masks


def _window(net, inputs, masks) -> float:
    _backend.kernel_events = []
    net.run(inputs=inputs, time=T, **({"masks": masks} if masks else {}))
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def measure(batch: int, arms, steps: int, warmup: int) -> dict:
    dev = torch.device("cuda")
    nets = {k: build(batch, k == "local3d", dev) for k in arms}
    for _ in range(warmup):
        for net, inputs, masks in nets.values():
            _window(net, inputs, masks)
    ms = {k: [] for k in nets}
    for _ in range(steps):   # alternated: every arm sees the same clocks and the same neighbours on the host
        for k, (net, inputs, masks) in nets.items():
            ms[k].append(_window(net, inputs, masks))
    for net, _, _ in nets.values():
        net.check_errors()
    w_bytes = 4 * F_ * C ** 3 * K ** 3
    line = {"B": batch, "input": [1, S, S, S], "T": T, "windows": steps, **device_info(),
            "w_MB": w_bytes / 1e6, "learning_w_traffic_MB_per_step": 2 * w_bytes / 1e6}
    for k, v in ms.items():
        med = statistics.median(v)
        line.update({f"{k}_ms_median": med, f"{k}_ms_min": min(v), f"{k}_ms_max": max(v),
                     f"{k}_sample_timesteps_per_s": batch * T / (med / 1e3)})
    if "local3d" in ms:
        # the learning phase's weight traffic alone, over the whole window's kernel time: a lower bound of the rate
        line["local3d_w_traffic_GB_per_s"] = 2 * w_bytes * T / (line["local3d_ms_median"] / 1e3) / 1e9
    if len(ms) == 2:
        line["dense_mask_over_local3d"] = line["dense_mask_ms_median"] / line["local3d_ms_median"]
    del nets
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    print(json.dumps(measure(1, ("local3d", "dense_mask"), a.steps, a.warmup)), flush=True)
    print(json.dumps(measure(32, ("local3d",), a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
