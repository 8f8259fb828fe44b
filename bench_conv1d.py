"""Conv1dConnection benchmark, two networks, each beside its Conv2dConnection twin (kernel (1, k) over [C, 1, L]
populations, the same weights and spikes), alternated window by window in the same process:
  example  the reference's examples/mnist/conv1d_MNIST.py: Input [1, 784] -> Conv1dConnection (kernel 56, stride 28, 25
           filters, PostPre nu (1e-4, 1e-2), norm 0.4 * 56, wmax 1) -> DiehlAndCookNodes [25, 27] with the example's -100
           recurrent inhibition
  long     Input [4, 4096] -> Conv1dConnection (kernel 9, stride 1, padding 4, 32 filters, PostPre) -> LIFNodes [32, 4096]
at B = 1 and B = 128, T = 250, seeded Bernoulli input spikes resident on the device.  One JSON line per network and batch
size with the median / min / max kernel time per window of each arm over ``--steps`` windows after ``--warmup`` windows,
the learning phase's share of each arm's per-step cycles, and the device name and power limit read in the same run.

    python bench_conv1d.py [--steps K] [--warmup W] [--configs example:1,example:128,long:1,long:128]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events).  The
learning phase's share is the cycles from the end of the step's neuron update to the barrier that closes the learning
phase, from one extra window per arm run with SNN_B200_GPROF=1 (the kernel's per-phase clock64 counters, mean over CTAs),
over the cycles of all per-step phases.  Each window's time also goes to stderr as it is measured.  Nothing is written
to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import sys
import tempfile

import torch

from bench_sparse import device_info
from bindsnet_b200 import _backend
from bindsnet_b200.learning import PostPre
from bindsnet_b200.network import Network, nodes, topology

T = 250
PHASES = ("phase1", "barrierA", "phase2", "barrierB", "phase3", "phase3conv", "barrierC")
NETS = {   # name: (C_in, L_in, kernel, stride, padding, filters, rate, nu, norm)
    "example": (1, 784, 56, 28, 0, 25, 0.05, (1e-4, 1e-2), 0.4 * 56),
    "long": (4, 4096, 9, 1, 4, 32, 0.02, (1e-4, 1e-3), 0.4 * 36),
}


def build(name: str, batch: int, twin: bool, device, seed: int = 0):
    cin, L_in, k, s, p, F_, rate, nu, norm = NETS[name]
    L = (L_in - k + 2 * p) // s + 1
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(F_, cin, k, generator=g)
    x = (torch.rand(T, batch, cin, L_in, generator=g) < rate).to(torch.uint8)
    net = Network(dt=1.0, batch_size=batch, learning=True)
    X = nodes.Input(shape=[cin, 1, L_in] if twin else [cin, L_in], traces=True)
    shape = [F_, 1, L] if twin else [F_, L]
    Y = nodes.DiehlAndCookNodes(shape=shape, traces=True, one_spike=False) if name == "example" else \
        nodes.LIFNodes(shape=shape, traces=True, thresh=-60.0, refrac=2)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    kw = dict(update_rule=PostPre, nu=list(nu), norm=norm, wmax=1.0, reduction=None if batch == 1 else torch.sum)
    if name == "long":
        kw["wmin"] = 0.0
    if twin:
        conv = topology.Conv2dConnection(X, Y, kernel_size=(1, k), stride=(1, s), padding=(0, p), w=w.unsqueeze(2), **kw)
    else:
        conv = topology.Conv1dConnection(X, Y, kernel_size=k, stride=s, padding=p, w=w, **kw)
    net.add_connection(conv, "X", "Y")
    if name == "example":
        inh = torch.zeros(F_, L, F_, L)
        for f1 in range(F_):
            for f2 in range(F_):
                if f1 != f2:
                    inh[f1, torch.arange(L), f2, torch.arange(L)] = -100.0
        net.add_connection(topology.Connection(Y, Y, w=inh.view(Y.n, Y.n)), "Y", "Y")
    net.to(device)
    x = x.to(device)
    return net, {"X": x.view(T, batch, cin, 1, L_in) if twin else x}


def _window(net, inputs) -> float:
    _backend.kernel_events = []
    net.run(inputs=inputs, time=T)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def _learning_share(net, inputs) -> float:
    """Cycles of the learning phase per step (its barrier included) over the cycles of all per-step phases, one window
    with SNN_B200_GPROF=1."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        os.environ["SNN_B200_GPROF"] = "1"
        try:
            _window(net, inputs)
        finally:
            os.environ.pop("SNN_B200_GPROF", None)
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        text = f.read()
    mean = {m.group(1): float(m.group(3)) for m in re.finditer(r"\]\s+(\S+)\s+(\S+)\s+(\S+)\s+(\S+)\s*$", text, re.M)}
    if "phase3conv" not in mean:
        raise RuntimeError("SNN_B200_GPROF printed no phase counters:\n" + text[-2000:])
    # the CTAs without learning work wait for the busy ones at the barrier that closes the learning phase: its cycles
    # are part of the phase's wall time
    return sum(mean[p] for p in ("phase3", "phase3conv", "barrierC")) / sum(mean[p] for p in PHASES)


def measure(name: str, batch: int, steps: int, warmup: int) -> dict:
    dev = torch.device("cuda")
    arms = {"conv1d": build(name, batch, False, dev), "conv2d_twin": build(name, batch, True, dev)}
    for _ in range(warmup):
        for net, inputs in arms.values():
            net.reset_state_variables()
            _window(net, inputs)
    ms = {k: [] for k in arms}
    for i in range(steps):   # alternated: both arms see the same clocks and the same neighbours on the host
        for k, (net, inputs) in arms.items():
            net.reset_state_variables()
            ms[k].append(_window(net, inputs))
            print(f"{name} B={batch} {k} window {i}: {ms[k][-1]:.2f} ms", file=sys.stderr, flush=True)
    share = {}
    for k, (net, inputs) in arms.items():
        net.check_errors()
        net.reset_state_variables()
        share[k] = _learning_share(net, inputs)
    cin, L_in, k_, s, p, F_, rate, nu, norm = NETS[name]
    line = {"bench": "conv1d", "net": name, "B": batch, "T": T, "input": [cin, L_in], "kernel": k_, "stride": s, "padding": p,
            "filters": F_, "windows": steps, **device_info()}
    for k in arms:
        line[f"{k}_ms_median"] = statistics.median(ms[k])
        line[f"{k}_ms_min"], line[f"{k}_ms_max"] = min(ms[k]), max(ms[k])
        line[f"{k}_learning_share"] = share[k]
    line["conv2d_twin_over_conv1d"] = line["conv2d_twin_ms_median"] / line["conv1d_ms_median"]
    del arms
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--configs", default="example:1,example:128,long:1,long:128")
    a = ap.parse_args()
    for cfg in a.configs.split(","):
        name, batch = cfg.split(":")
        print(json.dumps(measure(name, int(batch), a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
