"""MeanFieldConnection benchmark: Input(784) (Bernoulli(0.05), resident on the device) -> LIFNodes(1600) with PostPre,
and Input -> LIFNodes(1600) Z with a LIF -> Z MeanFieldConnection of negative per-target w, T = 250, learning on.  Three
arms, alternated window by window in the same process:

  mf        the network as built: the generic window kernel counts A's spikes each step and adds the batch mean;
  no_mf     the same network without the mean-field connection: what the connection costs;
  torch_mf  the mean-field connection written as a user torch subclass (compute = s.float().mean() * w), which sends the
            network to the scripted tier (one step at a time from Python): what a user had to write before.

One JSON line per batch size, with the median, min and max window time (CUDA events around Network.run, then a
synchronise) and the device name and power limit read in the same run.  Nothing is written to the tree.

    python bench_meanfield.py [--steps K] [--warmup W] [--batches 32,128]
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch

from bench_sparse import device_info
from bindsnet_b200.learning import PostPre
from bindsnet_b200.network import Network, nodes, topology

T = 250


class TorchMeanField(topology.AbstractConnection):
    """The mean-field connection as a user would write it without the built-in class (reference topology.py:1972-1981)."""

    def __init__(self, source, target, w):
        super().__init__(source, target)
        self.w = torch.nn.Parameter(w, requires_grad=False)

    def compute(self, s):   # (Network's scripted tier takes [B, *target.shape])
        return (s.float().mean() * self.w).expand(s.shape[0], *self.target.shape)

    def update(self, **kwargs):
        pass

    def normalize(self):
        pass


def build(batch: int, arm: str, device, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    net = Network(dt=1.0, batch_size=batch, learning=True)
    X = nodes.Input(n=784, traces=True)
    A = nodes.LIFNodes(n=1600, traces=True, thresh=-52.0)
    Z = nodes.LIFNodes(n=1600, thresh=-52.0)
    net.add_layer(X, "X"); net.add_layer(A, "A"); net.add_layer(Z, "Z")
    net.add_connection(topology.Connection(X, A, w=0.3 * torch.rand(784, 1600, generator=g), update_rule=PostPre, nu=(1e-4, 1e-2),
                                           wmin=0.0, wmax=1.0), "X", "A")
    net.add_connection(topology.Connection(X, Z, w=0.25 * torch.rand(784, 1600, generator=g)), "X", "Z")
    w = -40.0 * torch.rand(1600, generator=g)
    if arm == "mf":
        net.add_connection(topology.MeanFieldConnection(A, Z, w=w), "A", "Z")
    elif arm == "torch_mf":
        net.add_connection(TorchMeanField(A, Z, w), "A", "Z")
    x = torch.bernoulli(0.05 * torch.ones(T, batch, 784), generator=g).bool().to(device)
    net.to(device)
    return net, {"X": x}


def measure(batch: int, steps: int, warmup: int) -> dict:
    dev = torch.device("cuda")
    arms = ("mf", "no_mf", "torch_mf")
    nets = {a: build(batch, a, dev) for a in arms}
    times = {a: [] for a in arms}
    for k in range(warmup + steps):
        for a in arms:
            net, inputs = nets[a]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            net.run(inputs=inputs, time=T)
            e1.record()
            torch.cuda.synchronize()
            net.check_errors()
            if k >= warmup:
                times[a].append(e0.elapsed_time(e1))
            net.reset_state_variables()
    out = {"bench": "meanfield", "B": batch, "T": T, "steps": steps, **device_info()}
    for a in arms:
        out[f"{a}_ms"] = {"median": statistics.median(times[a]), "min": min(times[a]), "max": max(times[a])}
    out["mf_over_no_mf"] = out["mf_ms"]["median"] / out["no_mf_ms"]["median"]
    out["torch_mf_over_mf"] = out["torch_mf_ms"]["median"] / out["mf_ms"]["median"]
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batches", default="32,128")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_meanfield.py needs a CUDA device")
    for b in (int(v) for v in args.batches.split(",")):
        print(json.dumps(measure(b, args.steps, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
