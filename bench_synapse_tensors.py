"""Per-synapse bounds and rates benchmark: Input(784) -> LIFNodes(4000) with PostPre and a per-target nu ([4000]), plus a
recurrent 4000 x 4000 WeightDependentPostPre Connection with sign bounds per source row ([4000, 1]: 20 % inhibitory
sources in [-1, 0], the others in [0, 1]), seeded Poisson input resident on the device, T = 250, B = 32 and 128.

Windows alternate among four networks with the same weights and spikes:
  row        the workload: per-row bounds, per-target nu
  full       the same bounds materialised as [4000, 4000] tensors (PostPre's nu must broadcast to [1, 4000])
  scalar     scalar bounds [-1, 1] and a scalar nu (the network the tensors extend)
  constant   the scalar network with its bounds and nu as constant tensors of the same values
so that "row" vs "full" shows the cost of reading a materialised tensor and "scalar" vs "constant" the cost of the
tensor path itself.  One JSON line per batch size with the median / min / max kernel time per window of each, and the
device name and power limit read in the same run.

    python bench_synapse_tensors.py [--steps K] [--warmup W]

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
from bindsnet_b200.learning import PostPre, WeightDependentPostPre
from bindsnet_b200.network import Network, nodes, topology

T, N, N_IN, FRAC_INH = 250, 4000, 784, 0.2
VARIANTS = ("row", "full", "scalar", "constant")


def build(variant: str, batch: int, device, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    net = Network(dt=1.0, batch_size=batch, learning=True)
    X = nodes.Input(N_IN, traces=True)
    Y = nodes.LIFNodes(N, traces=True, thresh=-52.0, refrac=5)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    nu_t = 1e-4 * (0.5 + torch.rand(N, generator=g))
    w_in = 0.3 * torch.rand(N_IN, N, generator=g)
    inh = torch.rand(N, 1, generator=g) < FRAC_INH
    lo = torch.where(inh, torch.full((N, 1), -1.0), torch.zeros(N, 1))
    hi = torch.where(inh, torch.zeros(N, 1), torch.ones(N, 1))
    w_r = torch.where(inh, -torch.rand(N, N, generator=g), torch.rand(N, N, generator=g)) * (2.0 / N)
    rate = 0.02 * torch.rand(N_IN, generator=g)
    x = (torch.rand(T, batch, N_IN, generator=g) < rate).to(torch.uint8)
    if variant == "row":
        nu, lo_r, hi_r = (nu_t, nu_t.clone()), lo, hi
    elif variant == "full":
        nu = (nu_t, nu_t.clone())
        lo_r, hi_r = lo.expand(N, N).contiguous(), hi.expand(N, N).contiguous()
    elif variant == "scalar":
        nu, lo_r, hi_r = (1e-4, 1e-4), -1.0, 1.0
    else:
        nu, lo_r, hi_r = (torch.full((N,), 1e-4), torch.full((N,), 1e-4)), torch.full((N, N), -1.0), torch.full((N, 1), 1.0)
    xy = topology.Connection(X, Y, w=w_in, update_rule=PostPre, nu=nu, reduction=torch.sum, wmin=0.0, wmax=1.0)
    yy = topology.Connection(Y, Y, w=w_r, wmin=lo_r, wmax=hi_r, update_rule=WeightDependentPostPre, nu=(1e-3, 1e-3),
                             reduction=torch.sum)
    net.add_connection(xy, "X", "Y")
    net.add_connection(yy, "Y", "Y")
    net.to(device)
    if isinstance(nu[0], torch.Tensor):   # a rule is not a Module: Network.to leaves its nu where it is
        xy.update_rule.nu = xy.update_rule.nu.to(device)
    return net, {"X": x.to(device)}


def _window(net, inputs) -> float:
    _backend.kernel_events = []
    net.run(inputs=inputs, time=T)
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in _backend.kernel_events)
    _backend.kernel_events = None
    return ms


def measure(batch: int, steps: int, warmup: int) -> dict:
    dev = torch.device("cuda")
    nets = {v: build(v, batch, dev) for v in VARIANTS}
    ms = {v: [] for v in VARIANTS}
    for k in range(warmup + steps):
        for v in VARIANTS:   # alternate window by window
            net, inputs = nets[v]
            net.reset_state_variables()
            t = _window(net, inputs)
            if k >= warmup:
                ms[v].append(t)
    spikes = {}
    for v, (net, _) in nets.items():
        net.check_errors()
        assert _backend.last_tier == 1
        spikes[v] = int(net.layers["Y"].s.sum())
    med = {v: statistics.median(ms[v]) for v in VARIANTS}
    line = {"bench": "synapse_tensors", "B": batch, "N": N, "n_in": N_IN, "T": T, "frac_inh": FRAC_INH, "windows": steps,
            **device_info(), **{f"ms_median_{v}": med[v] for v in VARIANTS},
            **{f"ms_min_{v}": min(ms[v]) for v in VARIANTS}, **{f"ms_max_{v}": max(ms[v]) for v in VARIANTS},
            "row_over_full": med["row"] / med["full"], "constant_over_scalar": med["constant"] / med["scalar"],
            "last_step_spikes": spikes}
    del nets
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    for batch in (32, 128):
        print(json.dumps(measure(batch, a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
