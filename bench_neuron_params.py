"""Per-neuron parameter benchmark: the DiehlAndCook2015 metric network (bench.py: n_neurons = 1600, batch 128, T = 250,
learning on, synthetic 28x28 Poisson input) whose excitatory population's thresh and theta_plus are per-neuron tensors
holding the model's scalars (-52 and 0.05), so that it computes what the scalar network computes.

Windows alternate among three copies with the same weights and input:
  pn       per-neuron tensors: the generic window kernel's PN instantiation (tier 1)
  scalar   the scalar network forced to the generic window kernel (tier 1)
  fused    the scalar network on the tier the library selects for it (the fused DiehlAndCook2015 kernel), for context
so that "pn" vs "scalar" is the cost of the per-lane parameter loads.  One JSON line with the median / min / max kernel
time per window of each over the measured windows (default 7), and the device name and power limit read in the same run.

    python bench_neuron_params.py [--steps K] [--warmup W]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events).
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch

from bench import BATCH, N_NEURONS, T_STEPS, make_network, synth_windows
from bench_sparse import device_info
from bindsnet_b200 import _backend

VARIANTS = ("pn", "scalar", "fused")


def build(variant: str, device):
    net = make_network(device)
    E = net.layers["Ae"]
    if variant == "pn":
        E.thresh = torch.full((N_NEURONS,), float(E.thresh), device=device)
        E.theta_plus = torch.full((N_NEURONS,), float(E.theta_plus), device=device)
    net.force_tier = 0 if variant == "fused" else 1
    return net


def _window(net, x) -> float:
    _backend.kernel_events = []
    net.run(inputs={"X": x}, time=T_STEPS)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda")
    nets = {v: build(v, dev) for v in VARIANTS}
    xs = [x.to(dev) for x in synth_windows(2, seed=0)]
    ms = {v: [] for v in VARIANTS}
    tiers = {}
    for k in range(a.warmup + a.steps):
        for v in VARIANTS:   # alternate window by window
            net = nets[v]
            net.reset_state_variables()
            t = _window(net, xs[k % 2])
            tiers[v] = _backend.last_tier
            if k >= a.warmup:
                ms[v].append(t)
    for net in nets.values():
        net.check_errors()
    assert tiers["pn"] == 1 and tiers["scalar"] == 1
    same = torch.equal(nets["pn"].layers["Ae"].theta, nets["scalar"].layers["Ae"].theta) and all(
        torch.equal(nets["pn"].connections[k].w, nets["scalar"].connections[k].w) for k in nets["pn"].connections)
    med = {v: statistics.median(ms[v]) for v in VARIANTS}
    print(json.dumps({"bench": "neuron_params", "B": BATCH, "n_neurons": N_NEURONS, "T": T_STEPS, "windows": a.steps, **device_info(),
                      **{f"ms_median_{v}": med[v] for v in VARIANTS}, **{f"ms_min_{v}": min(ms[v]) for v in VARIANTS},
                      **{f"ms_max_{v}": max(ms[v]) for v in VARIANTS}, "pn_over_scalar": med["pn"] / med["scalar"],
                      "fused_tier": tiers["fused"], "pn_equals_scalar": bool(same)}), flush=True)


if __name__ == "__main__":
    main()
