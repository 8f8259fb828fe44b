"""Averaged MCC PostPre benchmark: the DiehlAndCook2015 MCC network (Input(784) -> 1600 DiehlAndCookNodes with
inhibition) whose input Weight learns with MCC_learning.PostPre(average_update=10), with and without continues_update,
beside the same network without averaging, all on the generic window kernel (tier 1), T = 250, B = 1 and 128.  The
arms alternate window by window in one process; each reports the median of the windows' kernel times (CUDA events
around each window's launch).  Inputs are seeded synthetic Poisson spikes (per-pixel rates up to 60 Hz), resident on
the device.  One JSON line per batch size.  Nothing is written to the tree.

    python bench_mcc_average.py [--steps 7] [--warmup 2] [--batches 1,128]
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch

from bench_sparse import device_info
from bindsnet_b200 import _backend
from bindsnet_b200.learning import MCC_learning
from bindsnet_b200.models import DiehlAndCook2015

N_IN, N = 784, 1600


def build(B: int, k: int, cont: bool, T: int = 250, device: str = "cuda", seed: int = 0):
    """The network with its input Weight's rule averaging over k updates (k = 0: the plain rule), and seeded input."""
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    net = DiehlAndCook2015(n_inpt=N_IN, n_neurons=N, batch_size=B, inpt_shape=(1, 28, 28), inh=120.0)
    with torch.no_grad():
        net.connections[("X", "Ae")].w.copy_(0.3 * torch.rand(N_IN, N, generator=g))
    if k:
        conn = net.connections[("X", "Ae")]
        wf = conn._weight()
        r = wf.learning_rule
        wf.learning_rule = MCC_learning.PostPre(connection=conn, feature_value=wf.value, range=[r.min, r.max],
                                                nu=(float(r.nu[0]), float(r.nu[1])), reduction=r.reduction,
                                                average_update=k, continues_update=cont)
    net.force_tier = 1
    net.to(device)
    rate = 0.06 * torch.rand(B, N_IN, generator=g)   # spikes per step (dt = 1 ms): up to 60 Hz
    x = (torch.rand(T, B, N_IN, generator=g) < rate).to(torch.uint8).view(T, B, 1, 28, 28)
    return net, x.to(device)


def measure(B: int, steps: int, warmup: int, T: int = 250) -> dict:
    arms = {"plain": (0, False), "k10": (10, False), "k10_continues": (10, True)}
    nets = {name: build(B, k, cont, T) for name, (k, cont) in arms.items()}
    times = {name: [] for name in arms}
    for it in range(warmup + steps):
        for name, (net, x) in nets.items():
            _backend.kernel_events = []
            net.run({"X": x}, time=T, one_spike_seed=it)
            torch.cuda.synchronize()
            ev = _backend.kernel_events
            _backend.kernel_events = None
            net.check_errors()
            assert _backend.last_tier == 1
            if it >= warmup:
                times[name].append(sum(a.elapsed_time(b) for a, b in ev))
    med = {name: statistics.median(v) for name, v in times.items()}
    return {"bench": "mcc_average", "B": B, "T": T, "n_neurons": N, "windows": steps,
            "ms_per_window": {k: round(v, 3) for k, v in med.items()},
            "ratio_vs_plain": {k: round(v / med["plain"], 3) for k, v in med.items() if k != "plain"}, **device_info()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batches", default="1,128")
    a = ap.parse_args()
    for B in (int(b) for b in a.batches.split(",")):
        print(json.dumps(measure(B, a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
