"""Reservoir benchmark of SparseConnection: Input(784) -> dense Connection -> LIFNodes(N) with a recurrent
SparseConnection of density p, B = 32, T = 250, learning off, inputs resident on the device.  One JSON line per
configuration, with the same network's recurrent matrix as a dense Connection for comparison where it fits.

    python bench_sparse.py [--steps K] [--warmup W] [--configs 8000:0.01,32000:0.05]

Kernel time per window comes from CUDA events around each window's launch (bindsnet_b200._backend.kernel_events).  The
algorithmic bytes per step are computed from the run's own spike raster: the stored entries of the rows that spiked
(8 B each: int32 column + fp32 value) plus the state the step reads and writes.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import subprocess

import torch

from bindsnet_b200 import _backend
from bindsnet_b200.network import Network, monitors, nodes, topology

B, T, N_IN = 32, 250, 784


def build_reservoir(n: int, p: float, batch: int, steps: int, device, seed: int = 0, dense: bool = False):
    """The pattern is stratified: row i holds one entry in each of k = p * n equal column ranges (a random column of the
    range), so rows come out sorted and duplicate-free without a sort of the whole pattern.  Mixed-sign values, scaled
    by 1 / sqrt(k)."""
    g = torch.Generator(device=device).manual_seed(seed)
    k = max(1, int(round(p * n)))
    stride = n // k
    w_in = 0.6 * torch.rand(N_IN, n, generator=g, device=device)
    rows, cols = [], []
    for r0 in range(0, n, 8192):
        r1 = min(n, r0 + 8192)
        u = torch.randint(0, stride, (r1 - r0, k), generator=g, device=device)
        cols.append((torch.arange(k, device=device) * stride + u).reshape(-1))
        rows.append(torch.arange(r0, r1, device=device).repeat_interleave(k))
    idx = torch.stack([torch.cat(rows), torch.cat(cols)])
    del rows, cols
    val = (torch.rand(idx.shape[1], generator=g, device=device) - 0.55) * (40.0 / k ** 0.5)
    w = torch.sparse_coo_tensor(idx, val, (n, n), is_coalesced=True)
    x = (torch.rand(steps, batch, N_IN, generator=g, device=device) < 0.05).to(torch.uint8)
    net = Network(dt=1.0, batch_size=batch, learning=False)
    X, Y = nodes.Input(N_IN), nodes.LIFNodes(n, thresh=-52.0, refrac=5, tc_decay=20.0)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    net.add_connection(topology.Connection(X, Y, w=w_in), "X", "Y")
    if dense:   # assigned after construction: Connection's constructor would hold a second dense copy
        rec = topology.Connection(Y, Y, w=torch.zeros(1, 1))
        rec.w = torch.nn.Parameter(w.to_dense(), requires_grad=False)
        net.add_connection(rec, "Y", "Y")
    else:
        net.add_connection(topology.SparseConnection(Y, Y, w=w), "Y", "Y")
    del w, idx, val
    net.to(device)
    return net, {"X": x}


def _time_windows(net, inputs, steps: int, warmup: int):
    for _ in range(warmup):
        net.run(inputs=inputs, time=T)
    torch.cuda.synchronize()
    _backend.kernel_events = []
    for _ in range(steps):
        net.run(inputs=inputs, time=T)
    torch.cuda.synchronize()
    net.check_errors()
    ms = [a.elapsed_time(b) for a, b in _backend.kernel_events]
    _backend.kernel_events = None
    return ms


def device_info():
    idx = torch.cuda.current_device()
    power = None
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        pass
    return {"device": torch.cuda.get_device_name(idx), "power_limit_w": power}


def measure(n: int, p: float, steps: int, warmup: int) -> dict:
    dev = torch.device("cuda")
    k = max(1, int(round(p * n)))
    nnz = n * k
    line = {"N": n, "p": p, "B": B, "T": T, "nnz": nnz, **device_info()}
    try:
        net, inputs = build_reservoir(n, p, B, T, dev)
    except torch.OutOfMemoryError:
        torch.cuda.empty_cache()
        return {**line, "sparse": "does not fit"}
    ms = _time_windows(net, inputs, steps, warmup)
    # one more window with a spike raster: activity and the bytes the gather had to read
    mon = monitors.Monitor(net.layers["Y"], ["s"], time=T, device=dev)
    net.add_monitor(mon, "Ys")
    net.run(inputs=inputs, time=T)
    s = mon.get("s").reshape(T, B, n).to(dev)
    csr = net.connections[("Y", "Y")]._b200_csr
    rowlen = (csr[1][1:] - csr[1][:-1]).float()
    spikes = float(s.sum()) / T
    entries = sum(float((s[t0:t0 + 25].float() @ rowlen).sum()) for t0 in range(0, T, 25)) / T
    state = B * n * (4 + 4 + 4 + 1) * 2          # v, refrac_count, input sum read / written; spikes
    mean_ms = sum(ms) / len(ms)
    line.update({"mean_spikes_per_step": spikes, "mean_spikes_per_sample_step": spikes / B,
                 "sparse_ms_per_window": mean_ms, "sparse_ms_min": min(ms), "sparse_ms_max": max(ms),
                 "sparse_sample_timesteps_per_s": B * T / (mean_ms / 1e3),
                 "algorithmic_bytes_per_step": entries * 8 + state,
                 "algorithmic_gb_per_s": (entries * 8 + state) * T / (mean_ms / 1e3) / 1e9})
    del net, inputs, s, mon
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if 4.0 * n * n * 1.2 > free:
        line["dense"] = "does not fit"
        return line
    try:
        net, inputs = build_reservoir(n, p, B, T, dev, dense=True)
        dms = _time_windows(net, inputs, steps, warmup)
        line.update({"dense_ms_per_window": sum(dms) / len(dms), "dense_ms_min": min(dms), "dense_ms_max": max(dms),
                     "dense_sample_timesteps_per_s": B * T / (sum(dms) / len(dms) / 1e3)})
        del net, inputs
    except torch.OutOfMemoryError:
        line["dense"] = "does not fit"
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--configs", default="8000:0.01,8000:0.05,32000:0.01,32000:0.05,100000:0.01,100000:0.05,150000:0.01,150000:0.05")
    a = ap.parse_args()
    for item in a.configs.split(","):
        n, p = item.split(":")
        print(json.dumps(measure(int(n), float(p), a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
