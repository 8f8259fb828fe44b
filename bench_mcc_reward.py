"""Reward-modulated readout benchmark: the reference's examples/mnist/MCC_reservoir.py topology (Input(784) ->
MCC[Probability, Weight] -> LIFNodes(4000) with a recurrent MCC[Probability, Weight]) plus a readout to 10 LIF neurons
that learns with MCC_learning.MSTDP (B = 32, 128) or MSTDPET (B = 1) on an MCC[Weight], T = 250, inputs resident on the
device.  Beside it, in the same process and alternated window by window, the twin whose readout is a Connection with
learning.MSTDP / MSTDPET and the same weights.  One JSON line per configuration.

    python bench_mcc_reward.py [--steps K] [--warmup W] [--configs MSTDP:32,MSTDP:128,MSTDPET:1]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events).  The
learning phase's share is the phase-3 cycles of one extra window per arm run with SNN_B200_GPROF=1 (the kernel's
per-phase clock64 counters, mean over CTAs), over the cycles of all per-step phases.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import tempfile

import torch

from bench_sparse import device_info
from bindsnet_b200 import _backend
from bindsnet_b200 import learning as L
from bindsnet_b200.learning import MCC_learning
from bindsnet_b200.network import Network, nodes, topology
from bindsnet_b200.network.topology_features import Probability, Weight

T, N_IN, N_RES = 250, 784, 4000
PHASES = ("phase1", "barrierA", "phase2", "barrierB", "phase3", "phase3conv", "barrierC")


def build(rule: str, batch: int, mcc: bool, device, seed: int = 0):
    """The input and recurrent pipelines of bench_mcc_features.py; readout weights uniform in [0, 0.5)."""
    g = torch.Generator().manual_seed(seed)   # built on the host, then moved: both arms hold the same values
    w_in = torch.rand(N_IN, N_RES, generator=g)
    w_rec = (torch.rand(N_RES, N_RES, generator=g) - 0.5) * (8.0 / N_RES ** 0.5)
    p_in = torch.rand(N_IN, N_RES, generator=g)
    p_rec = torch.rand(N_RES, N_RES, generator=g)
    w_out = 0.5 * torch.rand(N_RES, 10, generator=g)
    x = (torch.rand(T, batch, N_IN, generator=g) < 0.05).to(torch.uint8).to(device)
    net = Network(dt=1.0, batch_size=batch, learning=True)
    X, R, O = nodes.Input(N_IN), nodes.LIFNodes(N_RES, thresh=-52.0), nodes.LIFNodes(10, thresh=-55.0)
    net.add_layer(X, "X"); net.add_layer(R, "R"); net.add_layer(O, "O")
    net.add_connection(topology.MulticompartmentConnection(X, R, pipeline=[Probability("p_in", p_in), Weight("w_in", w_in)]), "X", "R")
    net.add_connection(topology.MulticompartmentConnection(R, R, pipeline=[Probability("p_rec", p_rec), Weight("w_rec", w_rec)]), "R", "R")
    nu = (1e-3, 1e-3)
    if mcc:
        readout = topology.MulticompartmentConnection(R, O, pipeline=[
            Weight("w_out", w_out, range=[-1.0, 1.0], learning_rule=getattr(MCC_learning, rule), nu=nu, reduction=torch.sum)])
    else:
        readout = topology.Connection(R, O, w=w_out, update_rule=getattr(L, rule), nu=nu, reduction=torch.sum, wmin=-1.0, wmax=1.0)
    net.add_connection(readout, "R", "O")
    net.to(device)
    return net, {"X": x}


def _window(net, inputs, k: int) -> float:
    _backend.kernel_events = []
    net.run(inputs=inputs, time=T, one_spike_seed=k, reward=1.0 if k % 2 else -0.5)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def _learning_share(net, inputs) -> float:
    """Phase-3 cycles per step over the cycles of all per-step phases, one window with SNN_B200_GPROF=1."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        os.environ["SNN_B200_GPROF"] = "1"
        try:
            _window(net, inputs, 0)
        finally:
            os.environ.pop("SNN_B200_GPROF", None)
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        text = f.read()
    mean = {m.group(1): float(m.group(3)) for m in re.finditer(r"\]\s+(\S+)\s+(\S+)\s+(\S+)\s+(\S+)\s*$", text, re.M)}
    if "phase3" not in mean:
        raise RuntimeError("SNN_B200_GPROF printed no phase counters:\n" + text[-2000:])
    return mean["phase3"] / sum(mean[p] for p in PHASES)


def measure(rule: str, batch: int, steps: int, warmup: int) -> dict:
    dev = torch.device("cuda")
    nets = {k: build(rule, batch, k == "mcc", dev) for k in ("mcc", "dense")}
    for i in range(warmup):
        for net, inputs in nets.values():
            _window(net, inputs, i)
    ms = {k: [] for k in nets}
    for i in range(steps):   # alternated: both arms see the same clocks and the same neighbours on the host
        for k, (net, inputs) in nets.items():
            ms[k].append(_window(net, inputs, i))
    for net, _ in nets.values():
        net.check_errors()
    line = {"rule": rule, "N": N_RES, "B": batch, "T": T, **device_info()}
    for k, v in ms.items():
        line.update({f"{k}_ms_per_window": sum(v) / len(v), f"{k}_ms_min": min(v), f"{k}_ms_max": max(v)})
    line["mcc_over_dense"] = line["mcc_ms_per_window"] / line["dense_ms_per_window"]
    for k, (net, inputs) in nets.items():
        line[f"{k}_learning_phase_share"] = _learning_share(net, inputs)
    del nets
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--configs", default="MSTDP:32,MSTDP:128,MSTDPET:1")
    a = ap.parse_args()
    for item in a.configs.split(","):
        rule, b = item.split(":")
        print(json.dumps(measure(rule, int(b), a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
